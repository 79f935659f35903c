"""GPU: the off-policy diagnostics of impala_vtrace_loss_diag against the float64 statement in
tests/diagnostics_oracle.py, through every launch shape of the V-trace kernel, the engine, a forked
Learner and (>= 2 devices) the data-parallel all-reduce."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import diagnostics_oracle as dorc
from conftest import PKEYS
from oracle import impala_oracle as orc
from torched_impala_b200 import synth
from torched_impala_b200.engine import LearnerEngine, diagnostic_values
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu

ATOL = 1e-5


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check_against_oracle(got_sums, got_vfl, want_sums, want_vfl, batch, ratio, valid, rho_bar, c_bar):
    """n exact; each clip count off only by steps within 1e-5 relative of its bound; means within 1e-5."""
    assert got_sums[0] == want_sums[0]
    for i, bound in ((2, rho_bar), (3, c_bar)):
        near = int((np.abs(ratio[valid] - bound) <= 1e-5 * bound).sum())
        assert abs(got_sums[i] - want_sums[i]) <= near, (i, got_sums[i], want_sums[i], near)
    got, want = diagnostic_values(got_sums, got_vfl, batch), dorc.derived(want_sums, want_vfl, batch)
    for k in ("log_ratio_mean", "kl_behaviour_current", "value_explained_variance"):
        assert abs(got[k] - want[k]) < ATOL, (k, got[k], want[k])
    n = want_sums[0]
    scale = max(1.0, abs(want_sums[5]) / n)
    assert abs(got_sums[5] - want_sums[5]) / n < ATOL * scale  # mean vs
    assert abs(got_sums[7] - want_sums[7]) / n < ATOL * scale  # mean vs - v


def taken_ratio(cur, beh, actions):
    a = actions.astype(np.int64)[..., None]
    lp = np.take_along_axis(orc.log_softmax(np.asarray(cur, np.float64)), a, -1)[..., 0]
    lq = np.take_along_axis(orc.log_softmax(np.asarray(beh, np.float64)), a, -1)[..., 0]
    return np.exp(lp - lq)


def _launch_shapes():
    out = []
    for A in (2, 4, 6, 9, 18, 32):  # every AP bucket; A = 2, 4, 32 take the 128-bit (VEC) rows, 6, 9, 18 not
        for s in ((1, 2, 5) if A <= 4 else (0,)):  # IMPALA_VTRACE_S applies to AP <= 4
            for cl in (1, 4):
                out.append((A, s, cl))
    return out


@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("T", [20, 100])
@pytest.mark.parametrize("A,S,cluster", _launch_shapes())
def test_kernel_matches_oracle(ops, monkeypatch, A, S, cluster, T, ragged, mode):
    if S:
        monkeypatch.setenv("IMPALA_VTRACE_S", str(S))
    monkeypatch.setenv("IMPALA_VTRACE_CLUSTER", str(cluster))
    B = 77  # three full trajectory groups and a partial one
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9, gamma=0.97)
    b = synth.make_batch(T + A + S, T, B, 3, A, ragged=ragged)
    rng = np.random.default_rng(T * A + S + cluster)
    logits = (b["beh_logits"] + 0.5 * rng.standard_normal((T, B, A))).astype(np.float32)
    v = rng.standard_normal((T + 1, B), dtype=np.float32)
    args = (dev(logits), dev(b["beh_logits"]), dev(b["actions"]), dev(b["rewards"]), dev(b["done"]),
            dev(b["lens"]), dev(v), hp, 1.0 / B)
    res = ops.vtrace_loss_diag(*args, mode=mode)
    plain = ops.vtrace_loss(*args, mode=mode)
    for k in ("vs", "pg_adv", "dlogits", "dv", "scalars"):  # the diag kernel computes what the plain one does
        assert torch.equal(res[k], plain[k]), k
    vs, pg, _ = orc.vtrace(v, logits, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], hp.gamma,
                           hp.rho_bar, hp.c_bar, mode)
    ref = orc.losses(v.astype(np.float64), vs, logits, b["actions"], pg, b["lens"], hp.v_loss_c, hp.policy_loss_c,
                     hp.entropy_c, B)
    want = dorc.diagnostics(v, vs, logits, b["beh_logits"], b["actions"], b["lens"], hp.rho_bar, hp.c_bar)
    valid = np.arange(T)[:, None] < b["lens"][None, :]
    check_against_oracle(res["diag"].cpu().tolist(), float(res["scalars"][0]), want, ref["value_fn_loss"], B,
                         taken_ratio(logits, b["beh_logits"], b["actions"]), valid, hp.rho_bar, hp.c_bar)


@pytest.mark.parametrize("A", [2, 4, 6, 9, 18, 32])
@pytest.mark.parametrize("T", [20, 100])
def test_on_policy_is_exactly_zero(ops, A, T):
    """Behaviour logits == current logits: no log ratio, no KL, nothing clipped at rho_bar = c_bar = 1."""
    B = 64
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=1.0)
    b = synth.make_batch(A + T, T, B, 3, A, ragged=True)
    z = dev(b["beh_logits"])
    res = ops.vtrace_loss_diag(z, z, dev(b["actions"]), dev(b["rewards"]), dev(b["done"]), dev(b["lens"]),
                               dev(np.random.default_rng(A).standard_normal((T + 1, B), dtype=np.float32)), hp, 1.0 / B)
    d = res["diag"].cpu().tolist()
    assert d[0] == int(np.clip(b["lens"], 0, T).sum())
    assert d[1] == 0.0 and d[2] == 0.0 and d[3] == 0.0 and d[4] == 0.0, d


ENGINE_SHAPES = {  # T, B, O, A, H, obs kind
    "c4": (20, 1024, 24, 4, 256, "normal"),
    "ram": (20, 1024, 128, 18, 256, "normal"),
    "minatar": (20, 1024, 400, 6, 256, "planes"),
}


@pytest.mark.parametrize("shape", list(ENGINE_SHAPES))
def test_engine_first_step_and_training_unchanged(shape):
    T, B, O, A, H, kind = ENGINE_SHAPES[shape]
    obs_dtype = "uint8" if kind != "normal" else "float32"
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    params = synth.init_params(5, O, A, H)
    batches = [synth.make_batch(20 + u, T, B, O, A, ragged=(u % 2 == 1), obs_kind=kind) for u in range(5)]
    engines = [LearnerEngine(T, B, O, A, H, H, hp, obs_dtype=obs_dtype, diagnostics=d) for d in (True, False)]
    for e in engines:
        e.load_state(params)
    # first step against the oracle on the float64 forward of the same parameters
    on = engines[0]
    on.load_device_batch(batches[0])
    on.step(0)
    sc = on.read_scalars()
    got = on.comm[on.n_total + 4:on.n_total + 12].cpu().tolist()
    b = batches[0]
    obs = b["obs"].astype(np.float64)
    f64 = {g: [np.asarray(params[g][k], np.float64) for k in PKEYS] for g in ("policy", "value_fn")}
    logits, _ = orc.mlp_forward(obs[:-1], *f64["policy"])
    v = orc.mlp_forward(obs, *f64["value_fn"])[0][..., 0]
    vs, pg, _ = orc.vtrace(v, logits, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], hp.gamma,
                           hp.rho_bar, hp.c_bar)
    ref = orc.losses(v, vs, logits, b["actions"], pg, b["lens"], hp.v_loss_c, hp.policy_loss_c, hp.entropy_c, B)
    want = dorc.diagnostics(v, vs, logits, b["beh_logits"], b["actions"], b["lens"], hp.rho_bar, hp.c_bar)
    valid = np.arange(T)[:, None] < b["lens"][None, :]
    check_against_oracle(got, sc["value_fn_loss"], want, ref["value_fn_loss"], B,
                         taken_ratio(logits, b["beh_logits"], b["actions"]), valid, hp.rho_bar, hp.c_bar)
    for k in ("log_ratio_mean", "rho_clip_fraction", "c_clip_fraction", "kl_behaviour_current",
              "value_explained_variance", "valid_steps"):
        assert k in sc
    # five steps with and without diagnostics: the same parameters, bit for bit
    on.load_state(params)
    on.adam_m.zero_(), on.adam_v.zero_(), on.adam_step.zero_()
    for e in engines:
        for u, bt in enumerate(batches):
            e.fill_host(bt, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
        e.synchronize()
    assert torch.equal(engines[0].params, engines[1].params)
    assert engines[0].launches_per_step == engines[1].launches_per_step


def _run_learner(tmp_path, mode, n_dev):
    script = os.path.join(os.path.dirname(__file__), "diag_learner_process_check.py")
    out = tmp_path / f"weights_{mode}.npz"
    res = subprocess.run([sys.executable, script, str(tmp_path / f"logs_{mode}"), mode, str(out), str(n_dev)],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "DIAG_LEARNER_OK" in res.stdout
    assert ("rho clipped" in res.stdout) == (mode == "on")  # console line at verbose >= 1
    return np.load(out)


@pytest.mark.parametrize("n_dev", [1, 2])
def test_forked_learner_logs_diagnostics(tmp_path, n_dev):
    if torch.cuda.device_count() < n_dev:
        pytest.skip(f"needs at least {n_dev} GPUs")
    on, off = _run_learner(tmp_path, "on", n_dev), _run_learner(tmp_path, "off", n_dev)
    assert set(on.files) == set(off.files)
    for k in on.files:
        assert np.array_equal(on[k], off[k]), k


@pytest.mark.parametrize("allreduce", ["peer", "peer-standalone", "nccl"])
def test_two_rank_sums_match_single_gpu(allreduce):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs (data-parallel path)")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_diag_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240,
                         env=dict(os.environ, IMPALA_ALLREDUCE=allreduce.split("-")[0],
                                  IMPALA_PUSH_FUSED="0" if allreduce == "peer-standalone" else "1"))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_DIAG_OK" in res.stdout
