"""GPU: wide observations (128 < O <= 1024, O % 4 == 0) on the K-streamed tensor-core kernels.

The forward and the two-phase backward (recompute + DP^T, then dW1 = DP^T X) against the float64 oracle,
with N(0, 1), binary {0, 1} (MinAtar) and uniform [0, 1] (Atari RAM / 255) observations; output and
workspace buffers NaN-filled so that an entry no CTA writes shows up; bitwise determinism; the refused
shapes; first-step parity of the whole learner step; graph replay; the forked Learner behind a RingQueue.
Every output and gradient entry is held to its float64 error bound (tests/mlp_bounds.py); the engine checks
are those of test_gpu_wide_shapes.py.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from mlp_bounds import check_backward, check_forward
from oracle.check import first_step_parity
from test_gpu_wide_shapes import check_engine_mlp, check_grad_end_to_end
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu

OBS_SHAPES = [
    # (M, O, H, N2)
    (20 * 1024, 512, 256, 18), (21 * 1024, 512, 256, 1), (5000, 400, 256, 6), (3001, 132, 128, 3),
    (777, 1024, 512, 17), (333, 700, 1024, 4), (5, 1000, 128, 32), (60001, 256, 384, 18),
]
INPUTS = ["normal", "binary", "uniform"]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_x(rng, M, O, kind):
    if kind == "binary":
        return (rng.random((M, O)) < 0.3).astype(np.float32)
    if kind == "uniform":
        return rng.integers(0, 256, (M, O)).astype(np.float32) / np.float32(255)
    return rng.standard_normal((M, O), dtype=np.float32)


def forward_case(M, O, H, N2, kind):
    rng = np.random.default_rng(M + O + H + N2)
    p = synth.init_params(M, O, N2, H)["policy"]
    return make_x(rng, M, O, kind), p


def backward_case(M, O, H, N2, kind):
    rng = np.random.default_rng(7 * M + O + H + N2)
    p = synth.init_params(M + 1, O, N2, H)["policy"]
    x = make_x(rng, M, O, kind)
    return x, p, (rng.standard_normal((M, N2), dtype=np.float32) / M).astype(np.float32)


def forward(ops, x, params, M, O, H, N2):
    """impala_mlp_forward into an output buffer NaN-filled past M rows."""
    out = torch.full(((M + 64) * N2,), float("nan"), dtype=torch.float32, device="cuda")
    _cabi.check(_cabi.lib().impala_mlp_forward(ops._p(x), ops._p(params), ops._p(out), M, O, H, N2, ops._st()),
                "impala_mlp_forward")
    torch.cuda.synchronize()
    assert torch.isnan(out[M * N2:]).all(), "rows past M were written"
    return out[: M * N2].view(M, N2)


def backward(ops, x, params, dout, M, O, H, N2):
    """impala_mlp_backward with the workspace past its control header filled with NaN."""
    lib = _cabi.lib()
    nbytes = int(lib.impala_mlp_backward_workspace(M, O, H, N2))
    assert nbytes > 0, nbytes
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    ws[256:] = 255  # 0xffffffff: a float32 NaN
    grad = torch.empty(_cabi.param_layout(O, H, N2)[1], dtype=torch.float64, device="cuda")
    _cabi.check(lib.impala_mlp_backward(ops._p(x), ops._p(params), ops._p(dout), ops._p(grad), ops._p(ws), nbytes,
                                        M, O, H, N2, ops._st()), "impala_mlp_backward")
    torch.cuda.synchronize()
    return grad


@pytest.mark.parametrize("kind", INPUTS)
@pytest.mark.parametrize("M,O,H,N2", OBS_SHAPES)
def test_obs_mlp_forward(ops, M, O, H, N2, kind):
    x, p = forward_case(M, O, H, N2, kind)
    params, xd = ops.pack_params(p), dev(x)
    got = forward(ops, xd, params, M, O, H, N2)
    check_forward(got, x, p, f"fwd {M},{O},{H},{N2} {kind}")
    assert torch.equal(got, forward(ops, xd, params, M, O, H, N2))  # bitwise reproducible


@pytest.mark.parametrize("kind", INPUTS)
@pytest.mark.parametrize("M,O,H,N2", OBS_SHAPES)
def test_obs_mlp_backward(ops, M, O, H, N2, kind):
    x, p, dout = backward_case(M, O, H, N2, kind)
    params, xd, dd = ops.pack_params(p), dev(x), dev(dout)
    flat = backward(ops, xd, params, dd, M, O, H, N2)
    check_backward(flat, x, p, dout, f"bwd {M},{O},{H},{N2} {kind}")  # also: pad entries exactly zero
    assert torch.equal(flat, backward(ops, xd, params, dd, M, O, H, N2))  # bitwise reproducible


REFUSED = [
    # (O, H, env)
    (130, 256, {}), (1028, 256, {}), (512, 320, {}), (512, 1152, {}),
    (512, 256, {"IMPALA_MLP_TC": "0"}), (512, 256, {"IMPALA_MLP_TCW": "0"}),
]


@pytest.mark.parametrize("O,H,env", REFUSED)
def test_obs_refused_shapes(ops, monkeypatch, O, H, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    M, N2 = 100, 6
    p = synth.init_params(0, O, N2, H)["policy"]
    x = dev(np.zeros((M, O), np.float32))
    with pytest.raises(_cabi.ImpalaCudaError, match="UNSUPPORTED_SHAPE"):
        ops.mlp_forward(x, ops.pack_params(p), O, H, N2)
    with pytest.raises(_cabi.ImpalaCudaError, match="UNSUPPORTED_SHAPE"):
        ops.mlp_backward(x, ops.pack_params(p), dev(np.zeros((M, N2), np.float32)), O, H, N2)


# name: (T, B, O, A, H, ragged) - thresholds of test_gpu_wide_shapes.test_wide_first_step_matches_oracle
CASES = {
    "ram4": (20, 4096, 512, 18, 256, False),
    "minatar_ragged_B1024": (20, 1024, 400, 6, 256, True),
    "O1024_A18_H1024_B1024": (20, 1024, 1024, 18, 1024, False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_obs_first_step_matches_oracle(name):
    from torched_impala_b200.engine import LearnerEngine

    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
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
    if par["max_rel_grad"] < 5e-5:
        assert par["ok"]


def test_obs_graph_replay_equals_eager_at_ram4():
    from torched_impala_b200.engine import LearnerEngine

    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    T, B, O, A, H = 20, 4096, 512, 18, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(5 + i, T, B, O, A) for i in range(2)]
    out = []
    for graph in (False, True):
        eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=graph)
        eng.load_state(params)
        for u in range(4):
            eng.fill_host(batches[u % 2], u % 2)
            eng.ingest(u % 2)
            eng.step(u % 2)
        eng.synchronize()
        out.append(eng.params.clone())
    assert torch.equal(out[0], out[1])


def test_obs_learner_process_ring():
    """MlpPolicy(512, 18, 256) / MlpValueFn(512, 256) in a forked Learner behind a RingQueue."""
    script = os.path.join(os.path.dirname(__file__), "obs_learner_process_check.py")
    res = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "OBS_LEARNER_OK" in res.stdout
