"""GPU: policies with 5..16 actions (Atari minimal action sets: 6 for Pong, 9 for Ms. Pac-Man) on the
tensor-core MLP kernels.

The forward runs the 16-output epilogue at one, two or four K atoms and the backward the 16-output
layer-2-through-shared-memory kernel at one or two (at four it keeps the 32-output padded kernel).  Both
are held to the float64 error bound of tests/mlp_bounds.py with every logit written (the output starts as NaN), and the whole learner
step - eager engine, byte observations, forked Learner behind a RingQueue - is checked at A = 6 and A = 9.
Which kernels the launches take is checked in test_gpu_mlp_routes.py.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from mlp_bounds import check_backward, check_forward
from oracle.check import first_step_parity
from test_gpu_parity import backward_case, forward_case
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu

REL = 5e-5  # the backward's precision floor here (mlp_bounds.GRAD_REL elsewhere)

SHAPES = [
    # (M, O, H, N2): four K atoms (the 16-output forward replaces one that wrote 4 logits) ...
    (20 * 1024, 128, 256, 6), (5000, 100, 512, 9), (5, 128, 128, 16),
    # ... one K atom, including observation widths the narrow kernels take at <= 4 outputs ...
    (3001, 24, 256, 6), (60001, 28, 128, 5), (1000, 32, 1024, 8), (4097, 4, 128, 7),
    # ... and two
    (777, 64, 512, 16),
]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def forward_into_nan(x, params, M, O, H, N2):
    out = torch.full((M, N2), float("nan"), dtype=torch.float32, device="cuda")
    _cabi.check(_cabi.lib().impala_mlp_forward(_p(x), _p(params), _p(out), M, O, H, N2, _st()), "impala_mlp_forward")
    return out


def backward_into_nan(x, params, dout, M, O, H, N2):
    lib = _cabi.lib()
    nbytes = int(lib.impala_mlp_backward_workspace(M, O, H, N2))
    assert nbytes > 0, nbytes
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    grad = torch.full((_cabi.param_layout(O, H, N2)[1],), float("nan"), dtype=torch.float64, device="cuda")
    _cabi.check(lib.impala_mlp_backward(_p(x), _p(params), _p(dout), _p(grad), _p(ws), nbytes, M, O, H, N2, _st()),
                "impala_mlp_backward")
    return grad


@pytest.mark.parametrize("M,O,H,N2", SHAPES)
def test_forward_matches_oracle(ops, M, O, H, N2):
    x, p = forward_case(M, O, H, N2)
    got = forward_into_nan(dev(x), ops.pack_params(p), M, O, H, N2)
    check_forward(got, x, p, f"fwd {M},{O},{H},{N2}")  # a NaN left in the output fails it


@pytest.mark.parametrize("M,O,H,N2", SHAPES)
def test_backward_matches_oracle(ops, M, O, H, N2):
    """Every entry within its float64 error bound (ReLU ties allowed only in the entries they move); W2, b2 and the
    W1 / b1 rows without a tie within REL of their tensor's largest entry."""
    x, p, dout = backward_case(M, O, H, N2)
    flat = backward_into_nan(dev(x), ops.pack_params(p), dev(dout), M, O, H, N2)
    check_backward(flat, x, p, dout, f"bwd {M},{O},{H},{N2}", rel=REL)


# name: (T, B, O, A, H, ragged)
CASES = {
    "ram_a6": (20, 4096, 128, 6, 256, False),
    "c4a6": (20, 4096, 24, 6, 256, False),
    "ram_a9h512_ragged_B1024": (20, 1024, 128, 9, 512, True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_first_step_matches_oracle(ops, name):
    from test_gpu_wide_shapes import check_engine_mlp, check_grad_end_to_end
    from torched_impala_b200.engine import LearnerEngine

    T, B, O, A, H, ragged = CASES[name]
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(11, O, A, H)
    batch = synth.make_batch(17, T, B, O, A, ragged=ragged)
    eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=False)
    par = first_step_parity(eng, params, batch)
    print(name, json.dumps(par))
    assert par["max_abs_vs"] < 1e-5, par
    assert par["max_abs_pg"] < 1e-5, par
    for k, v in par["scalars"].items():
        assert v["abs_err"] < 1e-5, (k, v)
    check_engine_mlp(eng, params)
    if par["max_rel_grad"] >= 5e-5:
        check_grad_end_to_end(eng, params, batch, hp)
    assert par["max_abs_param_after_1_update"] < 5e-5, par
    assert par["frac_params_off"] < 1e-3, par
    for k in ("norm_policy", "norm_value"):
        assert abs(par[k]["got"] - par[k]["ref"]) < 5e-5 * max(1.0, par[k]["ref"]), par


def _run_engine(obs_dtype, T, B, O, A, H, hp, params, batches):
    from torched_impala_b200.engine import LearnerEngine

    eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=True, obs_dtype=obs_dtype)
    eng.load_state(params)
    scal = []
    for u in range(4):
        b = batches[u % 2]
        eng.fill_host(b if obs_dtype == "uint8" else {**b, "obs": b["obs"].astype(np.float32)}, u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        scal.append(eng.read_scalars())
    eng.synchronize()
    return eng.params.clone(), scal


def test_byte_observations_equal_float_at_ram_a6(ops):
    T, B, O, A, H, _ = CASES["ram_a6"]
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(31, O, A, H)
    batches = [synth.make_batch(50 + i, T, B, O, A, obs_kind="bytes") for i in range(2)]
    p8, s8 = _run_engine("uint8", T, B, O, A, H, hp, params, batches)
    pf, sf = _run_engine("float32", T, B, O, A, H, hp, params, batches)
    assert torch.equal(p8, pf), float((p8 - pf).abs().max())
    assert s8 == sf


def test_learner_process_ring_a6():
    """MlpPolicy(128, 6, 256) / MlpValueFn(128, 256) in a forked Learner behind a RingQueue: the check of
    wide_learner_process_check.py (3 updates on ragged trajectories, policy within 5e-5 of the oracle's) at
    A = 6, in a fresh interpreter (the parent of a forked CUDA process must never have initialised CUDA)."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"import sys; sys.path.insert(0, {here!r}); import wide_learner_process_check as w; w.A = 6; w.main()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "WIDE_LEARNER_OK" in res.stdout
