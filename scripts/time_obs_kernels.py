"""Per-kernel times of the K-streamed wide-observation MLP kernels (mlp_obs_tc.cu) at a learner shape.

Both networks of one step (policy: T*B rows, N2 = A; value function: (T+1)*B rows, N2 = 1) run their forward and
backward through the C ABI with L2 flushed before each call; torch.profiler (CUDA activities) gives the time of
every kernel.  Each kernel is reported against the H100 SXM data-sheet peak that bounds it: 495 TFLOP/s dense
TF32 for the tensor-core kernels (algorithmic = the fp32 FLOPs of the math, executed = what the tensor cores
issue: x3 for 3xTF32, K padded to whole chunks, the backward's recompute); the float64 reduction of the
partial rows is a memory / latency kernel.  --obs-dtype uint8 runs the byte form (impala_mlp_{forward,backward}_u8
on 0..255 observations: 2 of the 3 products per GEMM remain).  Run on the GPU: there is no CPU path.
"""
import argparse
import collections
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from torched_impala_b200 import _cabi, ops, synth  # noqa: E402

CFG = {"ram4": dict(T=20, B=4096, O=512, A=18, H=256), "minatar": dict(T=20, B=4096, O=400, A=6, H=256)}
PEAK_TF32 = 495e12
ap = argparse.ArgumentParser()
ap.add_argument("--config", default="ram4", choices=sorted(CFG))
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--obs-dtype", default="float32", choices=["float32", "uint8"])
a = ap.parse_args()
w = CFG[a.config]
T, B, O, A, H = w["T"], w["B"], w["O"], w["A"], w["H"]
lib = _cabi.lib()
rng = np.random.default_rng(0)
U8 = a.obs_dtype == "uint8"
if U8:
    obs = torch.from_numpy(rng.integers(0, 256, ((T + 1) * B, O), dtype=np.uint8)).cuda()
else:
    obs = torch.from_numpy(rng.random(((T + 1) * B, O), dtype=np.float32)).cuda()
fwd_fn = lib.impala_mlp_forward_u8 if U8 else lib.impala_mlp_forward
bwd_fn = lib.impala_mlp_backward_u8 if U8 else lib.impala_mlp_backward
SPLIT = 2 if U8 else 3  # products per GEMM: x_lo = 0 drops one for byte observations
nets = []
for M, N2 in ((T * B, A), ((T + 1) * B, 1)):
    params = ops.pack_params(synth.init_params(1, O, N2, H)["policy"])
    out = torch.empty(M * N2, dtype=torch.float32, device="cuda")
    dout = torch.from_numpy(rng.standard_normal((M, N2), dtype=np.float32) / M).cuda()
    nbytes = int(lib.impala_mlp_backward_workspace(M, O, H, N2))
    if nbytes < 0:
        _cabi.check(nbytes, "impala_mlp_backward_workspace")
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    grad = torch.empty(_cabi.param_layout(O, H, N2)[1], dtype=torch.float64, device="cuda")
    nets.append((M, N2, params, out, dout, ws, grad))
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def run_once():
    for M, N2, params, out, dout, ws, grad in nets:
        flush.zero_()
        _cabi.check(fwd_fn(ops._p(obs), ops._p(params), ops._p(out), M, O, H, N2, ops._st()), "fwd")
        flush.zero_()
        _cabi.check(bwd_fn(ops._p(obs), ops._p(params), ops._p(dout), ops._p(grad), ops._p(ws),
                           ws.numel(), M, O, H, N2, ops._st()), "bwd")


for _ in range(3):
    run_once()
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(a.iters):
        run_once()
    torch.cuda.synchronize()
times = collections.defaultdict(list)
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA and ("obs" in ev.name or "reduce_partials" in ev.name):
        times[ev.name].append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)


def up(x, m):
    return -(-x // m) * m


def is_vf(name):  # the one-output instantiation (value function)
    return re.search(r"<1[,>]", name) is not None or "ILi1E" in name


def work(name):
    """(algorithmic FLOPs, executed FLOPs) of one step's launches, summed over the two networks."""
    alg = exe = 0
    for M, N2, *_ in nets:
        Mp = up(M, 64)
        if "fwd_obs" in name and is_vf(name) == (N2 == 1):
            alg += 2 * M * O * H + 2 * M * H * N2
            exe += SPLIT * 2 * Mp * up(O, 32) * H
        elif "pre_kernel" in name and is_vf(name) == (N2 == 1):
            alg += 4 * M * H * N2  # dh and dW2; the recompute is not algorithmic
            exe += SPLIT * 2 * Mp * up(O, 32) * H
        elif "dw1_kernel" in name:
            alg += 2 * M * O * H
            exe += SPLIT * 2 * Mp * up(O, 64) * H
    return alg, exe


dev = torch.cuda.get_device_name()
print(f"{a.config} {w} obs {a.obs_dtype} on {dev}, L2 flushed before each C-ABI call, {a.iters} iterations")
for name, ts in sorted(times.items()):
    n_launch = len(ts) / a.iters  # launches of this kernel per iteration (one per network where both use it)
    us = float(np.mean(ts)) * n_launch  # per iteration
    alg, exe = work(name)
    short = re.search(r"(mlp_\w+|reduce_partials_kernel)(<[^>]*>)?", name).group(0)
    if exe:
        print(f"  {short:40s} {us:9.1f} us/step  algorithmic {alg / us / 1e6:6.1f} TFLOP/s  executed {exe / us / 1e6:6.1f}"
              f" TFLOP/s = {exe / us / 1e6 / (PEAK_TF32 / 1e12):.2f} of the TF32 peak (bound: tensor)")
    else:
        print(f"  {short:40s} {us:9.1f} us/step  (bound: HBM / latency)")
