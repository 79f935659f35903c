"""CPU: the optimizer and the peer-memory gradient exchange without a device - the C entry points' argument
checks (all of them come before any launch), the oracle's clip coefficient against torch.nn.utils.clip_grad_norm_
(finite, infinite and NaN gradients) and the ptxas report of the three kernels in optim.cu."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi

BAD_ARG = -1


def _buf(nbytes=4096, offset=0):
    """Host memory the checks may look at but no kernel ever reads: a 16-byte aligned address + offset."""
    raw = np.zeros(nbytes + 64, np.uint8)
    base = (raw.ctypes.data + 15) // 16 * 16
    _buf.keep.append(raw)
    return C.c_void_p(base + offset)


_buf.keep = []


def test_clip_adam_refuses_bad_arguments():
    lib = _cabi.lib()
    p = _buf()
    hp = (10.0, 1e-3, 0.9, 0.999, 1e-8)

    def rc(params=p, grad=p, m=p, v=p, state=p, n_policy=3, n_total=7):
        return lib.impala_clip_adam(params, grad, m, v, state, n_policy, n_total, *hp, None, None)

    for name in ("params", "grad", "m", "v", "state"):
        assert rc(**{name: None}) == BAD_ARG, name
    for n_policy, n_total in ((-1, 7), (8, 7), (0, 0), (0, -3)):
        assert rc(n_policy=n_policy, n_total=n_total) == BAD_ARG, (n_policy, n_total)


def test_peer_push_refuses_bad_arguments():
    lib = _cabi.lib()
    p = _buf()
    n = 100

    def rc(local=p, n=n, gather=p, seq=p, slot=n, buf=2 * n, rank=0, world=2):
        return lib.impala_peer_push(local, n, gather, seq, slot, buf, rank, world, None)

    for name in ("local", "gather", "seq"):
        assert rc(**{name: None}) == BAD_ARG, name
    for kw in (dict(n=0), dict(world=0), dict(world=9, buf=9 * n), dict(rank=2), dict(rank=-1),
               dict(rank=8, world=8, buf=8 * n), dict(slot=n - 1), dict(buf=2 * n - 1),
               dict(world=8, buf=8 * n - 1)):
        assert rc(**kw) == BAD_ARG, kw


def test_gather_clip_adam_refuses_bad_arguments():
    lib = _cabi.lib()
    p = _buf()
    n_total, n_extra = 100, 4
    slot = n_total + n_extra
    hp = (10.0, 1e-3, 0.9, 0.999, 1e-8)

    def rc(params=p, reduced=p, gather=p, seq=p, slot=slot, buf=2 * slot, world=2, n_extra=n_extra, m=p, v=p,
           state=p, n_policy=40, n_total=n_total):
        return lib.impala_gather_clip_adam(params, reduced, gather, seq, slot, buf, world, n_extra, m, v, state,
                                           n_policy, n_total, *hp, None, None, 1.0, None)

    for name in ("params", "reduced", "gather", "seq", "m", "v", "state"):
        assert rc(**{name: None}) == BAD_ARG, name
    for kw in (dict(n_policy=-1), dict(n_policy=n_total + 1), dict(n_total=0, n_policy=0), dict(world=0),
               dict(world=9, buf=9 * slot), dict(n_extra=-1), dict(n_extra=1025, slot=n_total + 1025),
               dict(slot=slot - 1), dict(buf=2 * slot - 1), dict(world=8, buf=8 * slot - 1),
               dict(gather=_buf(offset=8)), dict(gather=_buf(offset=4))):
        assert rc(**kw) == BAD_ARG, kw


def test_backward_pair_push_refuses_bad_arguments():
    lib = _cabi.lib()
    p = _buf()
    T, B, O, H, A = 5, 8, 24, 256, 4  # a shape the fused push takes (Narrow tensor-core plans)
    M_pi, M_vf = T * B, (T + 1) * B
    assert lib.impala_mlp_backward_pair_push_supported(M_pi, M_vf, O, H, H, A) == 1
    n = _cabi.param_layout(O, H, A)[1] + _cabi.param_layout(O, H, 1)[1]
    n_extra = 4
    slot = n + n_extra
    big = 1 << 40

    def rc(x=p, pp=p, pv=p, dl=p, dv=p, ws_pi=p, ws_vf=p, extra=p, n_extra=n_extra, gather=p, seq=p, slot=slot,
           buf=2 * slot, rank=0, world=2, A=A):
        return lib.impala_mlp_backward_pair_push(x, pp, pv, dl, dv, ws_pi, big, ws_vf, big, M_pi, M_vf, O, H, H, A,
                                                 extra, n_extra, gather, seq, slot, buf, rank, world, None)

    for name in ("x", "pp", "pv", "dl", "dv", "ws_pi", "ws_vf", "extra", "gather", "seq"):
        assert rc(**{name: None}) == BAD_ARG, name
    for kw in (dict(world=0), dict(world=9, buf=9 * slot), dict(rank=2), dict(rank=-1),
               dict(rank=8, world=8, buf=8 * slot), dict(n_extra=-1), dict(n_extra=33, slot=n + 33),
               dict(slot=slot - 1), dict(buf=2 * slot - 1), dict(world=8, buf=8 * slot - 1)):
        assert rc(**kw) == BAD_ARG, kw
    # shapes outside the fused kernel are unsupported, not bad arguments
    assert rc(A=6) == -2 and rc(x=_buf(offset=4)) == -2


def _torch_clip(grads, max_norm):
    ts = [torch.tensor(g, dtype=torch.float64, requires_grad=True) for g in grads]
    for t, g in zip(ts, grads):
        t.grad = torch.tensor(g, dtype=torch.float64)
    norm = torch.nn.utils.clip_grad_norm_(ts, max_norm)
    return [t.grad.numpy() for t in ts], float(norm)


@pytest.mark.parametrize("case", ["below", "above", "zero", "inf", "nan", "nan_and_inf"])
def test_oracle_clip_coef_matches_torch(case):
    rng = np.random.default_rng(3)
    grads = [rng.standard_normal(7), rng.standard_normal((3, 4))]
    max_norm = {"below": 100.0, "above": 0.5}.get(case, 1.0)
    if case == "zero":
        grads = [np.zeros(7), np.zeros((3, 4))]
    if case in ("inf", "nan_and_inf"):
        grads[1][1, 2] = np.inf
    if case in ("nan", "nan_and_inf"):
        grads[0][4] = np.nan
    want, want_norm = _torch_clip(grads, max_norm)
    coef, norm = orc.clip_coef(grads, max_norm)
    assert (math.isnan(norm) and math.isnan(want_norm)) or norm == pytest.approx(want_norm, rel=1e-12), (norm, want_norm)
    for g, w in zip(grads, want):
        with np.errstate(invalid="ignore"):  # inf * 0 is the NaN torch produces as well
            np.testing.assert_allclose(g * coef, w, rtol=1e-12, atol=0, equal_nan=True)
    if case == "nan":  # torch: every gradient of the group becomes NaN (clamp keeps the NaN coefficient)
        assert all(np.isnan(w).all() for w in want) and math.isnan(coef)
    if case == "inf":  # coefficient 0: finite entries become 0, the infinite one NaN
        assert coef == 0.0 and np.isnan(want[1][1, 2]) and (np.delete(want[1].ravel(), 6) == 0).all()
    if case == "below":
        assert coef == 1.0


def test_optim_kernels_have_no_spills_or_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.fail("nvcc not found")
    src = os.path.join(os.path.dirname(_cabi.__file__), "csrc", "optim.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", src, "-o", str(tmp_path / "optim.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    blocks = re.split(r"Compiling entry function", res.stderr)[1:]
    # mangled names carry the identifier's length: 16clip_adam_kernel is not a suffix of 23gather_clip_adam_kernel
    for name in ("16clip_adam_kernel", "23gather_clip_adam_kernel", "16peer_push_kernel"):
        mine = [b for b in blocks if name in b.split("'")[1]]
        assert len(mine) == 1, (name, len(mine))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in mine[0], mine[0]
        assert not re.search(r"\d+ bytes lmem", mine[0]) or re.search(r"\b0 bytes lmem", mine[0]), mine[0]
