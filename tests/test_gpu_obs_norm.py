"""GPU: observation normalization (obs_norm).  impala_obs_normalize against the float64 oracle
(tests/obs_norm_oracle.py) for every slab form; the first update of a fresh obs_norm engine bitwise equal to a plain
engine; five updates (two with each other option) equal to a plain engine fed the oracle's normalized rows, with the
statistics against the oracle; the folded policy the actors run; load_state(state()) round trips; launch counts."""
import ctypes as C

import numpy as np
import pytest
import torch

import obs_norm_oracle as onorc
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.engine import LearnerEngine
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return _cabi.lib()


def P(t):
    return C.c_void_p(t.data_ptr())


# (T, B, F, k, dtype): dense float32, bytes at O <= 128 and O > 128, frames of float32 and of bytes
FORMS = {"f32": (5, 37, 24, 1, "float32"), "u8_o100": (5, 37, 100, 1, "uint8"), "u8_o200": (4, 29, 200, 1, "uint8"),
         "frames_f32": (6, 23, 6, 4, "float32"), "frames_u8": (5, 19, 50, 4, "uint8"),
         "c4_rows": (20, 512, 24, 1, "float32")}


@pytest.mark.parametrize("form", list(FORMS))
def test_normalize_kernel_against_oracle(lib, form):
    T, B, F, k, dt = FORMS[form]
    O = F * k
    rng = np.random.default_rng(sum(map(ord, form)))
    lens = rng.integers(0, T + 1, B).astype(np.int32)
    lens[:2] = (0, T)
    if dt == "uint8":
        obs = rng.integers(0, 256, (T + k, B, F), dtype=np.uint8) if k > 1 else \
            rng.integers(0, 256, (T + 1, B, O), dtype=np.uint8)
    else:
        obs = onorc.scaled_obs(7, T + k - 1, B, F, np.full(B, T + k - 1))
    mean, var = rng.uniform(-50, 150, O), 10.0 ** rng.uniform(-3, 3, O)
    mu_f, r_f = onorc.norm_f32(mean, var, 1e-8)
    dev = dict(device="cuda")
    d_obs, d_lens = torch.from_numpy(obs).to(**dev), torch.from_numpy(lens).to(**dev)
    norm = torch.from_numpy(np.concatenate([mu_f, r_f])).to(**dev)
    out = torch.full(((T + 1) * B * O,), float("nan"), **dev)
    sums = torch.zeros(2 * O + 1, dtype=torch.float64, **dev)
    ws = torch.zeros(int(lib.impala_obs_normalize_workspace(T, B, O)), dtype=torch.uint8, **dev)
    code = _cabi.OBS_DTYPES[dt]

    def run():
        _cabi.check(lib.impala_obs_normalize(P(d_obs), code, T, B, F, k, P(d_lens), P(norm), P(out), P(sums), P(ws),
                                             ws.numel(), None), "impala_obs_normalize")
        torch.cuda.synchronize()
        return out.clone(), sums.clone()

    out1, sums1 = run()
    x = onorc.dense_rows(obs, T, k)
    want = onorc.normalize(x, mu_f, r_f).reshape(-1)
    got = out1.cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=2e-7, atol=2e-7 * np.abs(want).max())  # every row is written
    s1, s2, n = onorc.batch_sums(x, lens, T)
    got_s = sums1.cpu().numpy()
    assert got_s[2 * O] == n == np.minimum(lens, T).sum()
    np.testing.assert_allclose(got_s[:O], s1, rtol=1e-12, atol=1e-12 * np.abs(s1).max())
    np.testing.assert_allclose(got_s[O:2 * O], s2, rtol=1e-12, atol=0)
    out2, sums2 = run()  # deterministic: the same bits again (the counters were left zeroed)
    assert torch.equal(out1, out2) and torch.equal(sums1, sums2)
    assert int(ws[:4].view(torch.int32)[0]) == 0


def _hp(T, B):
    return default_hparams(batch_size=B, max_timesteps=T)


def _batch(kind, seed, T, B, O, A, heads=(), frames=1):
    """A ragged batch of `kind` whose float32 observations have the oracle's wide feature scales."""
    if kind == "gaussian":
        batch = synth.make_gaussian_batch(seed, T, B, O, A, ragged=True)
    elif kind == "md_mask":
        batch = synth.make_masked_batch(seed, T, B, O, A, heads, ragged=True)
        batch.pop("legal")
    else:
        batch = synth.make_batch(seed, T, B, O, A, ragged=True, frames=frames,
                                 obs_kind="bytes" if kind == "frames_u8" else "normal")
    batch["lens"][:2] = (0, T)
    if kind != "frames_u8":
        batch["obs"] = onorc.scaled_obs(seed, T, B, O, batch["lens"])
    return batch


# name: (batch kind, engine options, updates)
CASES = {"plain": ("plain", {}, 5), "popart": ("plain", dict(popart=True), 2),
         "shared_torso": ("plain", dict(shared_torso=True), 2),
         "gaussian": ("gaussian", dict(action_dist="gaussian"), 2),
         "md_mask": ("md_mask", dict(action_dist="multi_discrete", action_heads=(3, 3, 2), action_mask=True), 2),
         "frames_u8": ("frames_u8", dict(frames=4, obs_dtype="uint8"), 2)}


@pytest.mark.parametrize("case", list(CASES))
def test_engine_against_plain_engine_on_oracle_rows(lib, case):
    """Update k of an obs_norm engine is a plain engine's update on the oracle's normalized rows."""
    kind, opts, updates = CASES[case]
    T, B, A, H = 6, 48, 4, 64
    O = 200 if kind == "frames_u8" else 24
    H = 256 if O > 128 else H  # the tensor-core shapes of O > 128 features
    A = 8 if kind == "md_mask" else A
    hp = _hp(T, B)
    on = LearnerEngine(T, B, O, A, H, H, hp, obs_norm=True, **opts)
    plain_opts = {k: v for k, v in opts.items() if k not in ("frames", "obs_dtype")}
    plain = LearnerEngine(T, B, O, A, H, H, hp, **plain_opts)
    gauss = kind == "gaussian"
    init = synth.init_params(0, O, 2 * A if gauss else A, H)
    if opts.get("shared_torso"):
        init["value_fn"]["model.0.weight"] = init["policy"]["model.0.weight"]
    on.load_state(init)
    plain.load_state(init)
    run = onorc.Running(O)
    for u in range(updates):
        batch = _batch(kind, 100 + u, T, B, O, A, heads=opts.get("action_heads", ()), frames=opts.get("frames", 1))
        x = onorc.dense_rows(batch["obs"], T, opts.get("frames", 1))
        pb = dict(batch, obs=onorc.normalize(x, *run.f32()))
        for eng, b in ((on, batch), (plain, pb)):
            eng.load_device_batch(b)
            eng.step()
        sc_on, sc_plain = on.read_scalars(), plain.read_scalars()
        run.update(x, batch["lens"], T)
        for name in ("value_fn_loss", "policy_loss", "policy_entropy", "norm_policy", "norm_value"):
            assert sc_on[name] == pytest.approx(sc_plain[name], rel=1e-5, abs=1e-6), (case, u, name)
        s_on, s_plain = on.normalized_state(), plain.normalized_state()
        for grp in s_on:
            for key in s_on[grp]:
                np.testing.assert_allclose(s_on[grp][key].numpy(), s_plain[grp][key].numpy(), rtol=1e-5, atol=1e-6,
                                           err_msg=f"{case} update {u + 1} {grp}.{key}")
        st = on.obs_norm_stats()
        assert st["count"] == run.count
        np.testing.assert_allclose(st["mean"], run.mean, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(st["var"], run.var, rtol=1e-12, atol=1e-300)


def test_replay_against_plain_engine_on_composed_rows(lib):
    """Replay: the normalize launch reads the composed slab, and replayed columns count in the statistics each time
    they are trained on.  Update k equals a plain engine's update on the oracle's normalized rows of the composed
    batch, with the oracle statistics over the composed batches."""
    T, B, O, A, H = 6, 48, 24, 4, 64
    hp = _hp(T, B)
    on = LearnerEngine(T, B, O, A, H, H, hp, obs_norm=True, replay_slabs=2, replay_columns=B // 2)
    plain = LearnerEngine(T, B, O, A, H, H, hp)
    init = synth.init_params(0, O, A, H)
    on.load_state(init)
    plain.load_state(init)
    run = onorc.Running(O)
    replayed = 0
    for u in range(5):
        on.load_device_batch(_batch("plain", 200 + u, T, on.B_fresh, O, A))
        on.step(0)
        on.synchronize()
        composed = {k: v.cpu().numpy().copy() for k, v in on.d_views[0].items()}
        replayed += int((on.replay_plan[on.B_fresh:, 0] >= 0).sum())
        x = onorc.dense_rows(composed["obs"], T)
        plain.load_device_batch(dict(composed, obs=onorc.normalize(x, *run.f32())))
        plain.step(0)
        run.update(x, composed["lens"], T)
        sc_on, sc_plain = on.read_scalars(), plain.read_scalars()
        for name in ("value_fn_loss", "policy_loss", "policy_entropy", "norm_policy", "norm_value"):
            assert sc_on[name] == pytest.approx(sc_plain[name], rel=1e-5, abs=1e-6), (u, name)
        s_on, s_plain = on.normalized_state(), plain.normalized_state()
        for grp in s_on:
            for key in s_on[grp]:
                np.testing.assert_allclose(s_on[grp][key].numpy(), s_plain[grp][key].numpy(), rtol=1e-5, atol=1e-6,
                                           err_msg=f"replay update {u + 1} {grp}.{key}")
        st = on.obs_norm_stats()
        assert st["count"] == run.count
        np.testing.assert_allclose(st["mean"], run.mean, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(st["var"], run.var, rtol=1e-12, atol=1e-300)
    assert replayed > 0  # replayed columns were trained on, and counted
    fresh = sum(int(np.minimum(_batch("plain", 200 + u, T, on.B_fresh, O, A)["lens"], T).sum()) for u in range(5))
    assert run.count > fresh


def test_first_update_is_bitwise_the_plain_engine(lib):
    """Fresh statistics (mean 0, sigma rounding to 1.0f): the normalized rows are the raw ones."""
    T, B, O, A, H = 20, 256, 24, 4, 256
    hp = _hp(T, B)
    batch = synth.make_batch(3, T, B, O, A, ragged=True)
    engines = [LearnerEngine(T, B, O, A, H, H, hp, obs_norm=on) for on in (False, True)]
    for eng in engines:
        eng.load_state(synth.init_params(0, O, A, H))
        eng.load_device_batch(batch)
        eng.step()
        eng.synchronize()
    a, b = engines
    assert torch.equal(a.params, b.params)
    assert torch.equal(a.comm[:a.n_total + a.n_extra], b.comm[:b.n_total + b.n_extra])  # gradient and scalars
    assert a.read_scalars() == b.read_scalars()


def test_published_policy_on_raw_rows_matches_engine_logits(lib):
    T, B, O, A, H = 6, 40, 24, 4, 64
    eng = LearnerEngine(T, B, O, A, H, H, _hp(T, B), obs_norm=True)
    eng.load_state(synth.init_params(0, O, A, H))
    batch = synth.make_batch(1, T, B, O, A, ragged=True)
    batch["obs"] = (batch["obs"] * np.linspace(0.5, 3.0, O) + np.linspace(-5.0, 5.0, O)).astype(np.float32)
    eng.load_device_batch(batch)
    eng.step()
    eng.forward_backward_only()  # logits of the updated network on rows normalized by the updated statistics
    eng.synchronize()
    sd = eng.state()["policy"]
    x = batch["obs"][:T].reshape(-1, O).astype(np.float64)
    h = np.maximum(x @ sd["model.0.weight"].numpy().T + sd["model.0.bias"].numpy(), 0.0)
    want = h @ sd["model.3.weight"].numpy().T + sd["model.3.bias"].numpy()
    got = eng.logits.cpu().numpy().reshape(-1, A).astype(np.float64)
    valid = onorc.valid_rows(batch["lens"], T)[:T].reshape(-1)
    np.testing.assert_allclose(got[valid], want[valid], rtol=1e-4, atol=1e-4 * np.abs(want).max())


@pytest.mark.parametrize("opts", [{}, dict(shared_torso=True, popart=True)])
def test_state_round_trip(lib, opts):
    T, B, O, A, H = 6, 40, 24, 4, 64
    hp = _hp(T, B)
    eng = LearnerEngine(T, B, O, A, H, H, hp, obs_norm=True, **opts)
    init = synth.init_params(0, O, A, H)
    if opts.get("shared_torso"):
        init["value_fn"]["model.0.weight"] = init["policy"]["model.0.weight"]
    eng.load_state(init)
    for u in range(2):  # moderate feature scales: a float32 folded b1' cancels W1' x by the scales' ratio
        batch = synth.make_batch(10 + u, T, B, O, A, ragged=True)
        batch["obs"] = (batch["obs"] * np.linspace(0.5, 3.0, O) + np.linspace(-5.0, 5.0, O)).astype(np.float32)
        eng.load_device_batch(batch)
        eng.step()
    st, trained = eng.obs_norm_stats(), eng.normalized_state()
    pop = eng.popart_stats() if opts.get("popart") else None
    other = LearnerEngine(T, B, O, A, H, H, hp, obs_norm=True, **opts)
    other.load_state(eng.state(), popart=pop, obs_norm=st)
    st2 = other.obs_norm_stats()
    assert st2["count"] == st["count"]
    assert (st2["mean"] == st["mean"]).all() and (st2["var"] == st["var"]).all()
    for grp, d in other.normalized_state().items():
        for key, t in d.items():
            np.testing.assert_allclose(t.numpy(), trained[grp][key].numpy(), rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError, match="obs_norm=False"):
        LearnerEngine(T, B, O, A, H, H, hp).load_state(eng.state(), obs_norm=st)


# (obs_dtype, frames, O, launches added): +2 for a float32 dense slab, +1 where the normalize launch replaces the
# widening (bytes, O <= 128) or the unstacking launch
LAUNCHES = [("float32", 1, 24, 2), ("uint8", 1, 128, 1), ("float32", 4, 24, 1), ("uint8", 4, 128, 1)]


@pytest.mark.parametrize("dt,frames,O,added", LAUNCHES)
def test_launch_count(lib, dt, frames, O, added):
    T, B, A, H = 6, 40, 4, 64
    counts = []
    for on in (False, True):
        eng = LearnerEngine(T, B, O, A, H, H, _hp(T, B), obs_dtype=dt, frames=frames, obs_norm=on)
        eng.load_state(synth.init_params(0, O, A, H))
        eng.load_device_batch(synth.make_batch(1, T, B, O, A, frames=frames,
                                               obs_kind="bytes" if dt == "uint8" else "normal"))
        for _ in range(3):  # eager, then the captured graph
            eng.step()
        eng.synchronize()
        counts.append(eng.launches_per_step)
    assert counts[1] == counts[0] + added


# --------------------------------------------------------------------------------------- forked Learner
def test_forked_learner_obs_norm(tmp_path):
    """Forked Learner(obs_norm=True) behind a RingQueue (tests/obs_norm_learner_process_check.py): the published and
    checkpointed modules equal the folded state of an engine run on the same batches, and a Learner that load()s the
    checkpoint resumes with the same statistics and, folded again, the same weights."""
    import os
    import subprocess
    import sys

    from conftest import Golden

    script = os.path.join(os.path.dirname(__file__), "obs_norm_learner_process_check.py")
    out = tmp_path / "weights.npz"
    res = subprocess.run([sys.executable, script, str(tmp_path / "logs"), str(out)], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "OBS_NORM_LEARNER_OK" in res.stdout
    w = np.load(out)
    g = Golden("c1_cartpole_ragged")
    c = g.case
    eng = LearnerEngine(c["T"], c["B"], c["O"], c["A"], c["H_pi"], c["H_v"], g.hp._replace(max_updates=g.updates),
                        obs_norm=True)
    eng.load_state(g.init_params())
    for u in range(g.updates):
        eng.fill_host(g.batch(u), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
    st, stats = eng.state(), eng.obs_norm_stats()
    assert float(w["count"]) == stats["count"]
    np.testing.assert_allclose(w["mean"], stats["mean"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(w["var"], stats["var"], rtol=1e-12, atol=1e-12)
    for grp in st:
        for key, t in st[grp].items():
            np.testing.assert_allclose(w[f"{grp}/{key}"], t.numpy(), rtol=1e-5, atol=1e-6, err_msg=f"{grp}.{key}")
            np.testing.assert_allclose(w[f"resumed/{grp}/{key}"], w[f"{grp}/{key}"], rtol=1e-5, atol=1e-5,
                                       err_msg=f"resumed {grp}.{key}")


# ------------------------------------------------------------------------------------------- two GPUs
@pytest.mark.parametrize("allreduce", ["peer", "peer-standalone", "nccl"])
def test_two_gpus(allreduce):
    """Every all-reduce route: the paired backward's fused push, impala_peer_push, NCCL."""
    import os
    import socket
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    with socket.socket() as s_:
        s_.bind(("127.0.0.1", 0))
        port = s_.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_obs_norm_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240,
                         env=dict(os.environ, IMPALA_ALLREDUCE=allreduce.split("-")[0],
                                  IMPALA_PUSH_FUSED="0" if allreduce == "peer-standalone" else "1"))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_OBS_NORM_OK" in res.stdout
    mode = {"peer": "peer(fused)", "peer-standalone": "peer(standalone)", "nccl": "nccl"}[allreduce]
    assert f"allreduce={mode}" in res.stdout, res.stdout[-2000:]
