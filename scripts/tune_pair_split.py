"""Sweep the per-tile cost weights that split the SMs between the policy and value-function tile
lists of the paired tensor-core launches (IMPALA_PAIR_W_FWD / IMPALA_PAIR_W_BWD, per cent of the
value-function tile cost) and print the L2-cold kernel times at the c4 shape.

    python scripts/tune_pair_split.py [--config c4] [--weights 100,115,127]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402

CFG = {"c4": dict(T=20, B=4096, O=24, A=4, H=256), "c3": dict(T=20, B=1024, O=24, A=4, H=256)}
ap = argparse.ArgumentParser()
ap.add_argument("--config", default="c4")
ap.add_argument("--weights", default="100,115,127,140,150,160,175,190,210", help="comma-separated weights to sweep")
args = ap.parse_args()
w = CFG[args.config]
hp = default_hparams(batch_size=w["B"], max_timesteps=w["T"])
eng = LearnerEngine(w["T"], w["B"], w["O"], w["A"], w["H"], w["H"], hp, use_graph=False)
eng.load_state(synth.init_params(0, w["O"], w["A"], w["H"]))
eng.load_device_batch(synth.make_batch(1, w["T"], w["B"], w["O"], w["A"]))
eng.step()
eng.synchronize()
buf = torch.empty(256 << 20, dtype=torch.uint8, device=eng.dev)
for wt in (int(x) for x in args.weights.split(",")):
    os.environ["IMPALA_PAIR_W_FWD"] = os.environ["IMPALA_PAIR_W_BWD"] = str(wt)
    with torch.cuda.stream(eng.stream):
        k = bench.kernel_breakdown(eng, buf.zero_, iters=15)
    print(f"W={wt}: fwd_pair {k['mlp_forward_pair(policy+value_fn)']['us']:.2f} us  "
          f"bwd_pair {k['mlp_backward_pair(policy+value_fn)']['us']:.2f} us  "
          f"(singles: fwd {k['mlp_forward(policy)']['us']:.1f}+{k['mlp_forward(value_fn)']['us']:.1f}, "
          f"bwd {k['mlp_backward(policy)']['us']:.1f}+{k['mlp_backward(value_fn)']['us']:.1f})", flush=True)
print("TUNE_DONE")
