"""First-light check of the wgmma forward: compare against the float64 oracle and the FP32 kernel."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import impala_oracle as orc  # noqa: E402
from torched_impala_b200 import ops, synth  # noqa: E402

PKEYS = ops.PKEYS
for (M, O, H, N2) in [(128, 24, 256, 4), (128, 4, 32, 2), (300, 24, 256, 1), (86016, 24, 256, 1),
                      (81920, 24, 256, 4), (1000, 8, 64, 3), (5000, 28, 128, 4)]:
    rng = np.random.default_rng(M + O)
    p = synth.init_params(M, O, N2, H)["policy"]
    x = rng.standard_normal((M, O), dtype=np.float32)
    want, _ = orc.mlp_forward(x.astype(np.float64), *[p[k].astype(np.float64) for k in PKEYS])
    xd, pd = torch.from_numpy(x).cuda(), ops.pack_params(p)
    res = {}
    for tc in ("0", "1"):
        os.environ["IMPALA_MLP_TC"] = tc
        got = ops.mlp_forward(xd, pd, O, H, N2)
        torch.cuda.synchronize()
        res[tc] = np.abs(got.cpu().numpy() - want).max()
    print(f"M={M} O={O} H={H} N2={N2}: max|err| fp32={res['0']:.3e} tc={res['1']:.3e}", flush=True)
print("TC_FWD_DONE")
