"""GPU: the tensor-core forward with the x tile held in registers (one K atom, O <= 32).

Each thread of `mlp_fwd_tc_pair_kernel` / `mlp_fwd_tc_kernel<NP, 1>` loads the x elements of its own
wgmma A-fragment slots straight from global memory: features 8 kk + q and 8 kk + q + 4 of two rows.
These cases pin what that mapping has to get right: a partial last K step and zero-filled features
for every observation width up to 32, ragged tiles and warpgroups without a tile, every hidden width
the narrow and wide kernels take at one K atom, every output count the register path serves, and
rows beyond M left untouched (the output buffer is over-allocated and NaN-filled).  The two-atom
widths (40, 48, 64), which stage the tile in shared memory, share the batched weight staging and
run beside them.  Everything is held against the float64 oracle at the forward's 1e-5 tolerance.
"""
import numpy as np
import pytest
import torch

from conftest import PKEYS
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, ops, synth

pytestmark = pytest.mark.gpu

ATOL = 1e-5
PAD_ROWS = 37  # sentinel rows past M in every output buffer


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")


def _oracle(x, p):
    want, _ = orc.mlp_forward(x.astype(np.float64), *[p[k].astype(np.float64) for k in PKEYS])
    return want


def _forward_padded(x, params, M, O, H, N2):
    """impala_mlp_forward into a NaN-filled buffer of M + PAD_ROWS rows."""
    out = torch.full((M + PAD_ROWS, N2), float("nan"), dtype=torch.float32, device="cuda")
    _cabi.check(_cabi.lib().impala_mlp_forward(ops._p(x), ops._p(params), ops._p(out), M, O, H, N2, ops._st()),
                "impala_mlp_forward")
    return out.cpu().numpy()


def _check(got, want, M):
    assert np.isfinite(got[:M]).all()
    assert np.abs(got[:M] - want).max() < ATOL, float(np.abs(got[:M] - want).max())
    assert np.isnan(got[M:]).all(), "a row past M was written"


SHAPES = [
    # (M, O, H, N2)
    # every observation width: partial last K step (O % 8 = 4), 1..8 K steps, zero-filled features
    (1000, 4, 256, 4), (1000, 8, 256, 4), (1000, 12, 256, 4), (1000, 20, 256, 4), (1000, 24, 256, 4),
    (1000, 28, 256, 4), (1000, 32, 256, 4), (1000, 40, 256, 4), (1000, 64, 256, 4), (1000, 40, 512, 1),
    # ragged M: fewer rows than a tile, M % 64 in {1, 63}, more warpgroups than tiles
    (5, 24, 256, 4), (63, 24, 128, 1), (129, 24, 256, 3), (191, 12, 256, 4), (4097, 64, 512, 4),
    # hidden widths: narrow path (O <= 28), and passes at one K atom on the wide path (O <= 32)
    (777, 24, 32, 4), (777, 24, 96, 1), (777, 20, 384, 4), (777, 32, 512, 3), (777, 8, 384, 1),
    # output counts: 1, 3, 4 (narrow / wide), 17 and 32 (17..32 outputs at one and two K atoms)
    (700, 24, 256, 1), (700, 24, 256, 3), (700, 24, 128, 17), (700, 32, 256, 32), (700, 64, 256, 17),
    (700, 48, 128, 32),
]


@pytest.mark.parametrize("M,O,H,N2", SHAPES)
def test_forward_against_oracle(M, O, H, N2):
    rng = np.random.default_rng(3 * M + 5 * O + H + N2)
    p = synth.init_params(M + O, O, N2, H)["policy"]
    x = rng.standard_normal((M, O), dtype=np.float32)
    got = _forward_padded(torch.from_numpy(x).cuda(), ops.pack_params(p), M, O, H, N2)
    _check(got, _oracle(x, p), M)


PAIR_SHAPES = [
    # (T, B, O, H_pi, H_vf, A): M_pi = T*B, M_vf = (T+1)*B
    (20, 4096, 24, 256, 256, 4),  # the benchmark's shape
    (5, 7, 8, 128, 256, 2),       # H_vf > H_pi: the launch's shared memory is sized by the value network
    (7, 129, 20, 256, 96, 3),     # H_pi > H_vf, an odd number of 32-unit slices, ragged last tile
]


@pytest.mark.parametrize("T,B,O,H_pi,H_vf,A", PAIR_SHAPES)
def test_pair_against_oracle_and_bitwise_reproducible(T, B, O, H_pi, H_vf, A):
    """The forward pair (both networks through one kernel body): both networks against the oracle, rows
    past M untouched, and two launches give the same bits."""
    M_pi, M_vf = T * B, (T + 1) * B
    rng = np.random.default_rng(2024 + T + H_vf)
    p_pi = synth.init_params(1, O, A, H_pi)["policy"]
    p_vf = synth.init_params(2, O, 1, H_vf)["policy"]
    x = rng.standard_normal((M_vf, O), dtype=np.float32)
    xd, pp, pv = torch.from_numpy(x).cuda(), ops.pack_params(p_pi), ops.pack_params(p_vf)

    def launch():
        logits = torch.full((M_pi + PAD_ROWS, A), float("nan"), dtype=torch.float32, device="cuda")
        values = torch.full((M_vf + PAD_ROWS,), float("nan"), dtype=torch.float32, device="cuda")
        _cabi.check(_cabi.lib().impala_mlp_forward_pair(ops._p(xd), ops._p(pp), ops._p(pv), ops._p(logits),
                                                        ops._p(values), M_pi, M_vf, O, H_pi, H_vf, A, ops._st()),
                    "impala_mlp_forward_pair")
        return logits, values

    first, second = launch(), launch()
    for a, b, M in zip(first, second, (M_pi, M_vf)):
        assert torch.equal(a[:M], b[:M])  # the NaN sentinel rows are checked below
    logits, values = (t.cpu().numpy() for t in first)
    _check(logits, _oracle(x[:M_pi], p_pi), M_pi)
    _check(values.reshape(-1, 1), _oracle(x, p_vf), M_vf)
