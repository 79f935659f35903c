"""GPU: the narrow tensor-core backward (one 64-unit hidden block per CTA, independent warpgroups).

Each CTA of `mlp_bwd_tc_pair_kernel` / `mlp_bwd_tc_kernel` owns one hidden block of one network and
writes only that block's entries of its partial row.  These cases pin what that layout has to get
right: every entry of the summed rows written exactly once (the workspace is filled with NaN before
the launch, so an entry no CTA writes shows), CTAs and warpgroups that get no tile, hidden widths
that differ between the two networks (different numbers of CTA groups per network), a ragged last
tile, and a reduction that is bitwise reproducible from launch to launch.  Every gradient entry is held to
its float64 error bound (tests/mlp_bounds.py).
"""
import numpy as np
import pytest
import torch

from mlp_bounds import check_backward
from torched_impala_b200 import _cabi, ops, synth

pytestmark = pytest.mark.gpu

WS_HEADER = 256  # control words at the start of a backward workspace (zero-filled once)


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")


def _workspace(M, O, H, N2):
    """A backward workspace with zeroed control words and NaN everywhere else."""
    nbytes = int(_cabi.lib().impala_mlp_backward_workspace(M, O, H, N2))
    assert nbytes > WS_HEADER
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    ws[:WS_HEADER] = 0
    return ws


def _pair(x, pp, pv, dlog, dv, M_pi, M_vf, O, H_pi, H_vf, A, ws_pi, ws_vf):
    g_pi = torch.empty(_cabi.param_layout(O, H_pi, A)[1], dtype=torch.float64, device="cuda")
    g_vf = torch.empty(_cabi.param_layout(O, H_vf, 1)[1], dtype=torch.float64, device="cuda")
    p = ops._p
    _cabi.check(_cabi.lib().impala_mlp_backward_pair(
        p(x), p(pp), p(pv), p(dlog), p(dv), p(g_pi), p(g_vf), p(ws_pi), ws_pi.numel(), p(ws_vf), ws_vf.numel(),
        M_pi, M_vf, O, H_pi, H_vf, A, ops._st()), "impala_mlp_backward_pair")
    return g_pi, g_vf


def _single(x, params, dout, M, O, H, N2, ws):
    grad = torch.empty(_cabi.param_layout(O, H, N2)[1], dtype=torch.float64, device="cuda")
    p = ops._p
    _cabi.check(_cabi.lib().impala_mlp_backward(p(x), p(params), p(dout), p(grad), p(ws), ws.numel(), M, O, H, N2,
                                                ops._st()), "impala_mlp_backward")
    return grad


PAIR_SHAPES = [
    # (T, B, O, H_pi, H_vf, A): M_pi = T*B, M_vf = (T+1)*B
    (5, 7, 8, 128, 256, 2),      # one tile per network: most warpgroups idle; 2 + 4 hidden blocks
    (3, 50, 28, 256, 128, 3),    # H_pi > H_vf, three tiles each
    (7, 129, 12, 128, 256, 4),   # H_pi < H_vf, ragged last tile (903 / 1032 rows)
    (4, 2049, 24, 256, 256, 4),  # more tiles than CTAs of a group, odd tail (8196 / 10245 rows)
    (20, 4096, 24, 256, 256, 4),  # the benchmark's shape
]


def pair_cases(T, B, O, H_pi, H_vf, A):
    """(x, params, dout) of the policy and of the value network, seeded as test_pair_against_oracle."""
    rng = np.random.default_rng(11 * T + B + O + H_pi)
    M_pi, M_vf = T * B, (T + 1) * B
    p_pi = synth.init_params(3, O, A, H_pi)["policy"]
    p_vf = synth.init_params(4, O, 1, H_vf)["policy"]
    x = rng.standard_normal((M_vf, O), dtype=np.float32)
    dlog = (rng.standard_normal((M_pi, A), dtype=np.float32) / M_pi).astype(np.float32)
    dv = (rng.standard_normal((M_vf,), dtype=np.float32) / M_vf).astype(np.float32)
    return (x[:M_pi], p_pi, dlog), (x, p_vf, dv.reshape(-1, 1))


@pytest.mark.parametrize("T,B,O,H_pi,H_vf,A", PAIR_SHAPES)
def test_pair_against_oracle(T, B, O, H_pi, H_vf, A):
    """Both networks' gradients, every entry within its float64 error bound (tests/mlp_bounds.py) and pad
    entries exactly zero."""
    (_, p_pi, dlog), (x, p_vf, dv) = pair_cases(T, B, O, H_pi, H_vf, A)
    M_pi, M_vf = T * B, (T + 1) * B
    xd, dlogd, dvd = (torch.from_numpy(a).cuda() for a in (x, dlog, dv.reshape(-1)))
    g_pi, g_vf = _pair(xd, ops.pack_params(p_pi), ops.pack_params(p_vf), dlogd, dvd, M_pi, M_vf, O, H_pi, H_vf, A,
                       _workspace(M_pi, O, H_pi, A), _workspace(M_vf, O, H_vf, 1))
    check_backward(g_pi, x[:M_pi], p_pi, dlog, f"pair policy {T},{B},{O},{H_pi},{A}")
    check_backward(g_vf, x, p_vf, dv, f"pair value {T},{B},{O},{H_vf}")


SINGLE_SHAPES = [
    # (M, O, H, N2)
    (5, 8, 256, 4), (64, 24, 128, 1), (65, 24, 256, 3), (6401, 28, 128, 4), (86017, 24, 256, 1),
]


def single_case(M, O, H, N2):
    rng = np.random.default_rng(5 * M + O + H + N2)
    p = synth.init_params(M + 2, O, N2, H)["policy"]
    x = rng.standard_normal((M, O), dtype=np.float32)
    return x, p, (rng.standard_normal((M, N2), dtype=np.float32) / M).astype(np.float32)


@pytest.mark.parametrize("M,O,H,N2", SINGLE_SHAPES)
def test_single_against_oracle(M, O, H, N2):
    x, p, dout = single_case(M, O, H, N2)
    grad = _single(torch.from_numpy(x).cuda(), ops.pack_params(p), torch.from_numpy(dout).cuda(), M, O, H, N2,
                   _workspace(M, O, H, N2))
    check_backward(grad, x, p, dout, f"single {M},{O},{H},{N2}")


def test_pair_is_bitwise_reproducible_at_c4():
    """Two consecutive launches on the same workspaces (the grid barrier re-arms itself) give the same
    bits: the partial rows are summed in a fixed order."""
    T, B, O, H, A = 20, 4096, 24, 256, 4
    M_pi, M_vf = T * B, (T + 1) * B
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(M_vf, O, device="cuda", generator=g)
    dlog = torch.randn(M_pi, A, device="cuda", generator=g) / M_pi
    dv = torch.randn(M_vf, device="cuda", generator=g) / M_vf
    pp = ops.pack_params(synth.init_params(1, O, A, H)["policy"])
    pv = ops.pack_params(synth.init_params(2, O, 1, H)["policy"])
    ws_pi, ws_vf = _workspace(M_pi, O, H, A), _workspace(M_vf, O, H, 1)
    first = _pair(x, pp, pv, dlog, dv, M_pi, M_vf, O, H, H, A, ws_pi, ws_vf)
    second = _pair(x, pp, pv, dlog, dv, M_pi, M_vf, O, H, H, A, ws_pi, ws_vf)
    for a, b in zip(first, second):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)
