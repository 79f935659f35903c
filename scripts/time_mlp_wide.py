"""Wide tensor-core MLP kernels (two K atoms, hidden layer in passes) against the FP32 FFMA kernels on the same inputs:
max abs difference and CUDA-event time of impala_mlp_forward / impala_mlp_backward per network.

    python scripts/time_mlp_wide.py [--M 819200] [--O 64] [--H 512] [--reps 5]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from torched_impala_b200 import ops, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--M", type=int, default=100 * 8192)
ap.add_argument("--O", type=int, default=64)
ap.add_argument("--H", type=int, default=512)
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()
M, O, H = a.M, a.O, a.H
rng = np.random.default_rng(0)
x = torch.from_numpy(rng.standard_normal((M, O), dtype=np.float32)).cuda()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timed(fn):
    ts = []
    out = None
    for i in range(a.reps + 1):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        if i:
            ts.append(e0.elapsed_time(e1) * 1e3)
    return out, statistics.median(ts)


for N2 in (4, 1):
    p = ops.pack_params(synth.init_params(3, O, N2, H)["policy"])
    dout = torch.from_numpy((rng.standard_normal((M, N2), dtype=np.float32) / M).astype(np.float32)).cuda()
    res = {}
    for tcw in ("1", "0"):
        os.environ["IMPALA_MLP_TCW"] = tcw
        out, t_f = timed(lambda: ops.mlp_forward(x, p, O, H, N2))
        grad, t_b = timed(lambda: ops.mlp_backward(x, p, dout, O, H, N2))
        res[tcw] = (out, grad, t_f, t_b)
    fl_f = 2.0 * M * (O * H + H * N2)
    fl_b = 2.0 * M * (O * H + 2 * H * N2)  # algorithmic (no recompute counted), as DESIGN section 4
    d_out = float((res["1"][0] - res["0"][0]).abs().max())
    g1, g0 = res["1"][1], res["0"][1]
    d_grad = float((g1 - g0).abs().max() / g0.abs().max())
    print(f"M={M} O={O} H={H} N2={N2}: fwd tcw {res['1'][2]:.0f} us ({fl_f / res['1'][2] * 1e-6:.1f} TF/s) vs fp32 "
          f"{res['0'][2]:.0f} us; bwd tcw {res['1'][3]:.0f} us ({fl_b / res['1'][3] * 1e-6:.1f} TF/s) vs fp32 {res['0'][3]:.0f} us; "
          f"max|out diff| {d_out:.2e}, max grad diff / max|grad| {d_grad:.2e}", flush=True)
