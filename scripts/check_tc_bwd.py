"""First-light check of the wgmma backward against the float64 oracle and the FP32 kernel."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import impala_oracle as orc  # noqa: E402
from torched_impala_b200 import ops, synth  # noqa: E402

PKEYS = ops.PKEYS


def rel(got, want):
    return float(np.abs(got - want).max() / max(1e-30, np.abs(want).max()))


for (M, O, H, N2) in [(32, 24, 256, 4), (64, 24, 128, 4), (96, 4, 128, 1), (1000, 24, 256, 1),
                      (4100, 8, 256, 3), (86016, 24, 256, 1), (81920, 24, 256, 4)]:
    rng = np.random.default_rng(M + O)
    p = synth.init_params(M, O, N2, H)["policy"]
    x = rng.standard_normal((M, O), dtype=np.float32)
    dout = (rng.standard_normal((M, N2), dtype=np.float32) / M).astype(np.float32)
    p64 = [p[k].astype(np.float64) for k in PKEYS]
    _, pre = orc.mlp_forward(x.astype(np.float64), *p64)
    want = orc.mlp_backward(x.astype(np.float64), pre, p64[2], dout.astype(np.float64))
    xd, pd, dd = torch.from_numpy(x).cuda(), ops.pack_params(p), torch.from_numpy(dout).cuda()
    line = f"M={M} O={O} H={H} N2={N2}:"
    for tc in ("0", "1"):
        os.environ["IMPALA_MLP_TC"] = tc
        flat = ops.mlp_backward(xd, pd, dd, O, H, N2)
        torch.cuda.synchronize()
        got = ops.unpack_grad(flat, O, H, N2)
        line += f" tc={tc} " + " ".join(f"{k.split('.')[1]}{k.split('.')[2][0]}={rel(got[k], w):.1e}"
                                        for k, w in zip(PKEYS, want))
    print(line, flush=True)
print("TC_BWD_DONE")
