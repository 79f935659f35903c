"""GPU: corners of the MLP route table (csrc/mlp.cu) that the shape lists of the other MLP tests do not reach.

Every case names the route row its forward and its backward take, and that is asserted once from the launched
kernel names; then every output and gradient entry is held to its float64 error bound (tests/mlp_bounds.py):

- Wide at H from 640 to 4096 (several 64-, 128- and 256-unit passes per CTA);
- M in {1, 31, 32, 33, 63, 64, 65} on Narrow, Wide at 1, 2 and 4 K atoms, Obs and FP32: the 32- and 64-row tiles;
- the FP32 backward at 32 * 1024 + 1 rows: more 32-row tiles than kMaxParts = 1024 partial rows, so the workspace
  is sized by the cap and every CTA runs several tiles;
- N2 in {1, 2, 4, 5, 16, 17, 32} at each K-atom count, O from 4 to 1024;
- pointers the tensor-core kernels cannot take: x at +1 float (FP32), dout at +1 float or grad at +1 double on
  the c4 backward shape (Wide instead of Narrow), byte rows at +4 bytes and rows of 132 bytes (4- but not
  16-byte aligned, still Obs);
- raw 0..255 byte rows through the byte entry points, and rows of zeros against b1 entries that are exactly 0,
  whose ReLU derivative must be torch's relu'(0) = 0.

Outputs past M rows stay NaN, the backward workspace is NaN past its control header, and a second call gives
the same bits.
"""
import re
import zlib
from typing import NamedTuple

import numpy as np
import pytest
import torch

from mlp_bounds import check_backward, check_forward
from test_gpu_mlp_routes import _has, _kernel_names, _ours
from torched_impala_b200 import _cabi, synth

pytestmark = pytest.mark.gpu

WS_HEADER = 256


class Case(NamedTuple):
    M: int
    O: int
    H: int
    N2: int
    fwd: str | None  # route row of the forward: narrow, wide1, wide2, wide4, obs, fp32 (None: not run)
    bwd: str | None  # ... of the backward
    kind: str = "normal"  # normal | bytes (uint8 0..255, byte entry points) | zeros (zero rows, zero b1 entries)
    x_off: int = 0  # x at this many elements past an aligned buffer
    dout_off: int = 0
    grad_off: int = 0


CASES = {}
# Wide at large H: (M, O, H, N2) -> K atoms
for M, O, H, N2, ka in [(2049, 128, 4096, 32, 4), (3001, 64, 2048, 16, 2), (1000, 32, 1536, 4, 1),
                        (777, 128, 640, 18, 4), (777, 24, 1152, 1, 1)]:
    CASES[f"wide_h{H}_{M}x{O}x{N2}"] = Case(M, O, H, N2, f"wide{ka}", f"wide{ka}")
# 32- and 64-row tile edges on every row of the route
EDGE_SHAPES = {"narrow": (24, 256, 4, "normal"), "wide1": (32, 512, 4, "normal"), "wide2": (64, 256, 16, "normal"),
               "wide4": (128, 256, 18, "normal"), "obs": (256, 128, 3, "bytes"), "fp32": (30, 96, 5, "normal")}
for M in (1, 31, 32, 33, 63, 64, 65):
    for route, (O, H, N2, kind) in EDGE_SHAPES.items():
        CASES[f"{route}_m{M}"] = Case(M, O, H, N2, route, route, kind)
# persistent FP32 CTAs over more tiles than partial rows
CASES["fp32_m32769"] = Case(32 * 1024 + 1, 30, 96, 5, None, "fp32")
# outputs at one, two and four K atoms (the backward takes four K atoms above 16 outputs)
for O, ka in ((32, 1), (64, 2), (128, 4)):
    for N2 in (1, 2, 4, 5, 16, 17, 32):
        CASES[f"n{N2}_o{O}"] = Case(1000, O, 256, N2, f"wide{ka}", f"wide{ka if N2 <= 16 else 4}")
# observation widths
for O, route in ((4, "narrow"), (28, "narrow"), (32, "wide1"), (36, "wide2"), (64, "wide2"), (68, "wide4"),
                 (128, "wide4"), (132, "obs"), (1020, "obs"), (1024, "obs")):
    CASES[f"o{O}"] = Case(777, O, 256, 4, route, route)
# misaligned pointers
CASES["x_off1"] = Case(4097, 24, 256, 4, "fp32", "fp32", x_off=1)
CASES["c4_dout_off1"] = Case(4097, 24, 256, 4, None, "wide1", dout_off=1)
CASES["c4_grad_off1"] = Case(4097, 24, 256, 4, None, "wide1", grad_off=1)
CASES["u8_x_off4"] = Case(1000, 512, 256, 6, "obs", "obs", "bytes", x_off=4)
CASES["u8_o132"] = Case(333, 132, 128, 3, "obs", "obs", "bytes")
# raw bytes and exact zeros
CASES["u8_ram4"] = Case(4096, 512, 256, 18, "obs", "obs", "bytes")
for route, (O, H, N2) in {"narrow": (24, 256, 4), "wide1": (32, 512, 4), "wide4": (128, 256, 18),
                          "obs": (512, 256, 6), "fp32": (30, 96, 5)}.items():
    CASES[f"zeros_{route}"] = Case(1000, O, H, N2, route, route, "zeros")

FORWARD_CASES = {k: c for k, c in CASES.items() if c.fwd}
BACKWARD_CASES = {k: c for k, c in CASES.items() if c.bwd}


def make_case(c: Case):
    """Seeded (x, params, dout) of a case: x float32 or uint8 (M, O)."""
    rng = np.random.default_rng(zlib.crc32(repr(c[:4] + (c.kind,)).encode()))
    p = synth.init_params(c.M + c.O, c.O, c.N2, c.H)["policy"]
    if c.kind == "bytes":
        x = rng.integers(0, 256, (c.M, c.O), dtype=np.uint8)
    else:
        x = rng.standard_normal((c.M, c.O), dtype=np.float32)
    if c.kind == "zeros":
        x[::3] = 0.0
        p["model.0.bias"][::4] = 0.0
    dout = (rng.standard_normal((c.M, c.N2), dtype=np.float32) / c.M).astype(np.float32)
    return x, p, dout


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def _at(a, off, dtype=None):
    """A device copy of `a` that starts `off` elements into a buffer of the allocator's alignment."""
    t = torch.from_numpy(np.ascontiguousarray(a)).reshape(-1)
    buf = torch.zeros(t.numel() + max(off, 1), dtype=t.dtype, device="cuda")
    buf[off:off + t.numel()] = t.cuda()
    return buf[off:off + t.numel()]


def run_forward(ops, c, x, params):
    """The forward entry point (byte rows: the byte one) into an output NaN-filled past M rows."""
    M, O, H, N2 = c[:4]
    out = torch.full(((M + 64) * N2,), float("nan"), dtype=torch.float32, device="cuda")
    fn = _cabi.lib().impala_mlp_forward_u8 if x.dtype == torch.uint8 else _cabi.lib().impala_mlp_forward
    _cabi.check(fn(ops._p(x), ops._p(params), ops._p(out), M, O, H, N2, ops._st()), "mlp forward")
    torch.cuda.synchronize()
    assert torch.isnan(out[M * N2:]).all(), "rows past M were written"
    return out[: M * N2].view(M, N2)


def run_backward(ops, c, x, params, dout):
    """The backward entry point with the workspace NaN past its control header, the gradient at c.grad_off
    doubles into a NaN-filled buffer."""
    M, O, H, N2 = c[:4]
    lib = _cabi.lib()
    nbytes = int(lib.impala_mlp_backward_workspace(M, O, H, N2))
    assert nbytes > WS_HEADER, nbytes
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    ws[:WS_HEADER] = 0
    total = _cabi.param_layout(O, H, N2)[1]
    grad = torch.full((total + 1,), float("nan"), dtype=torch.float64, device="cuda")[c.grad_off:c.grad_off + total]
    fn = lib.impala_mlp_backward_u8 if x.dtype == torch.uint8 else lib.impala_mlp_backward
    _cabi.check(fn(ops._p(x), ops._p(params), ops._p(dout), ops._p(grad), ops._p(ws), nbytes, M, O, H, N2, ops._st()),
                "mlp backward")
    torch.cuda.synchronize()
    return grad


def _routes(names):
    """Route rows named by the launched kernels: narrow (the in-kernel-reduced block backward), tc1 / tc2 / tc4
    (tensor-core forward or wide backward at that many K atoms), obs, fp32, and reduce."""
    mine = {n for n in names if _ours(n)}
    got = set()
    for n in mine:
        if _has({n}, "mlp_fwd_tc_kernel") or _has({n}, "mlp_bwd_tcw_kernel"):
            m = re.search(r"<\s*\d+\s*,\s*(\d+)\s*>", n) or re.search(r"ILi\d+ELi(\d+)E", n)
            got.add(f"tc{m.group(1)}")
        elif _has({n}, "mlp_bwd_tc_kernel"):
            got.add("narrow")
        elif "_obs_" in n:
            got.add("obs")
        elif _has({n}, "mlp_fwd_kernel") or _has({n}, "mlp_bwd_kernel"):
            got.add("fp32")
        elif "reduce_partials" in n:
            got.add("reduce")
        else:
            got.add(n)
    return got


def _want(route, bwd):
    fam = {"narrow": "tc1", "wide1": "tc1", "wide2": "tc2", "wide4": "tc4", "obs": "obs", "fp32": "fp32"}[route]
    if not bwd:
        return {fam}
    return {"narrow"} if route == "narrow" else {fam, "reduce"}


def _inputs(c):
    x, p, dout = make_case(c)
    return x, p, dout, _at(x, c.x_off), _at(dout, c.dout_off)


@pytest.mark.parametrize("name", list(FORWARD_CASES))
def test_forward_corner(ops, name):
    c = FORWARD_CASES[name]
    x, p, _, xd, _ = _inputs(c)
    params = ops.pack_params(p)
    assert _routes(_kernel_names(lambda: run_forward(ops, c, xd, params), tries=6)) == _want(c.fwd, False), name
    got = run_forward(ops, c, xd, params)
    check_forward(got, x, p, f"corner fwd {name} [{c.fwd}]", scaled=True)  # raw byte rows: outputs of order 1e2
    assert torch.equal(got, run_forward(ops, c, xd, params))


@pytest.mark.parametrize("name", list(BACKWARD_CASES))
def test_backward_corner(ops, name):
    c = BACKWARD_CASES[name]
    x, p, dout, xd, dd = _inputs(c)
    params = ops.pack_params(p)
    assert _routes(_kernel_names(lambda: run_backward(ops, c, xd, params, dd), tries=6)) == _want(c.bwd, True), name
    got = run_backward(ops, c, xd, params, dd)
    check_backward(got, x, p, dout, f"corner bwd {name} [{c.bwd}]")
    assert torch.equal(got, run_backward(ops, c, xd, params, dd))
