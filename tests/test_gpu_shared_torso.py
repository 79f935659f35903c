"""GPU: the shared-torso actor-critic.  The split-head MLP entry points are bitwise equal to the dense ones with
N2 = N + 1 on every route row; their refusals; LearnerEngine(shared_torso=True) against the float64 oracle
(tests/shared_torso_oracle.py) on the first step and over a few updates with diagnostics, PopArt and reward
clipping; frames and uint8 observations equal to the dense engine; replay equal to a plain shared engine fed the
composed batches; a forked Learner behind a RingQueue (publication, checkpoint, the reference's MlpPolicy); two
GPUs."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import shared_torso_oracle as sorc
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.engine import LearnerEngine
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return _cabi.lib()


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------- kernels
# (T, B, O, H, N, byte rows): one or more shapes on every route row (mlp.cu route)
ROUTES = {
    "narrow_cartpole": (5, 13, 4, 128, 2, False),      # N2 = 3; backward H 128
    "narrow_h256": (20, 37, 24, 256, 3, False),         # N2 = 4
    "fp32_bwd_h32": (20, 51, 4, 32, 2, False),          # forward Narrow, backward FP32 (H = 32)
    "wide_np4_ka1": (7, 29, 24, 512, 2, False),
    "wide_np4_ka2": (9, 31, 64, 256, 2, False),
    "wide_np16_ka1_c4": (20, 53, 24, 256, 4, False),   # c4 with A = 4: 5 outputs
    "wide_np16_ka2": (9, 31, 64, 256, 6, False),
    "wide_np32_ka1": (9, 31, 32, 256, 18, False),
    "wide_np32_ka2": (9, 31, 64, 384, 18, False),
    "wide_ka4_np4": (9, 31, 128, 256, 3, False),
    "wide_ka4_ram": (9, 31, 128, 256, 18, False),
    "wide_ka4_np16": (9, 31, 128, 128, 9, False),
    "obs_np4_f32": (5, 23, 512, 256, 2, False),
    "obs_np32_f32": (5, 23, 400, 128, 5, False),
    "obs_np4_u8": (5, 23, 512, 256, 2, True),
    "obs_ram4_u8": (5, 23, 512, 256, 18, True),
    "obs_minatar_u8": (5, 23, 400, 256, 4, True),
}
FP32_ROUTES = {"fp32_o24": (6, 19, 24, 64, 4), "fp32_o128_np32": (6, 19, 128, 128, 18), "fp32_o4": (5, 13, 4, 32, 2)}


def _case(seed, T, B, O, H, N, u8):
    g = torch.Generator(device="cpu").manual_seed(seed)
    M_a, M = T * B, (T + 1) * B
    offs, total = _cabi.param_layout(O, H, N + 1)
    params = torch.zeros(total)
    for off, n in zip(offs, (H * O, H, (N + 1) * H, N + 1)):
        params[off:off + n] = (torch.rand(n, generator=g) - 0.5) * (0.1 if u8 else 1.0)
    if u8:
        x = torch.randint(0, 256, (M, O), generator=g, dtype=torch.uint8)
    else:
        x = torch.randn(M, O, generator=g)
    dl, dv = torch.randn(M_a, N, generator=g), torch.randn(M, generator=g)
    dense_dz = torch.zeros(M, N + 1)
    dense_dz[:M_a, :N], dense_dz[:, N] = dl, dv
    return M_a, M, params.cuda(), x.cuda(), dl.cuda(), dv.cuda(), dense_dz.cuda()


def _compare(lib, T, B, O, H, N, u8):
    M_a, M, params, x, dl, dv, dz = _case(O * 7 + H + N, T, B, O, H, N, u8)
    code = _cabi.OBS_U8 if u8 else _cabi.OBS_F32
    fwd, bwd = ((lib.impala_mlp_forward_u8, lib.impala_mlp_backward_u8) if u8
                else (lib.impala_mlp_forward, lib.impala_mlp_backward))
    out = torch.full((M, N + 1), float("nan"), device="cuda")
    logits = torch.full((M_a, N), float("nan"), device="cuda")
    values = torch.full((M,), float("nan"), device="cuda")
    assert fwd(p(x), p(params), p(out), M, O, H, N + 1, None) == 0
    assert lib.impala_mlp_forward_shared(p(x), code, p(params), p(logits), p(values), M_a, M, O, H, N, None) == 0
    ws_n = lib.impala_mlp_backward_workspace(M, O, H, N + 1)
    assert ws_n > 0
    ws_d, ws_s = (torch.zeros(ws_n, dtype=torch.uint8, device="cuda") for _ in range(2))
    total = params.numel()
    g_d, g_s = (torch.full((total,), float("nan"), dtype=torch.float64, device="cuda") for _ in range(2))
    assert bwd(p(x), p(params), p(dz), p(g_d), p(ws_d), ws_n, M, O, H, N + 1, None) == 0
    assert lib.impala_mlp_backward_shared(p(x), code, p(params), p(dl), p(dv), p(g_s), p(ws_s), ws_n, M_a, M, O, H,
                                          N, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(logits, out[:M_a, :N])
    assert torch.equal(values, out[:, N])
    assert torch.equal(g_s, g_d)
    assert torch.isfinite(g_s).all()


@pytest.mark.parametrize("route", list(ROUTES))
def test_split_equals_dense(lib, route):
    _compare(lib, *ROUTES[route])


@pytest.mark.parametrize("route", list(FP32_ROUTES))
def test_split_equals_dense_fp32(lib, route, monkeypatch):
    monkeypatch.setenv("IMPALA_MLP_TC", "0")
    _compare(lib, *FP32_ROUTES[route], False)


def test_refusals(lib):
    T, B, O, H, N = 4, 8, 24, 128, 3
    M_a, M, params, x, dl, dv, _ = _case(1, T, B, O, H, N, False)
    ws_n = lib.impala_mlp_backward_workspace(M, O, H, N + 1)
    ws = torch.zeros(ws_n, dtype=torch.uint8, device="cuda")
    g = torch.zeros(params.numel(), dtype=torch.float64, device="cuda")
    values = torch.zeros(M, device="cuda")
    F32 = _cabi.OBS_F32

    def fwd(x_=x, code=F32, lg=dl, vals=values, Ma=M_a, n=N):
        return lib.impala_mlp_forward_shared(p(x_), code, p(params), p(lg), p(vals), Ma, M, O, H, n, None)

    def bwd(x_=x, code=F32, d_l=dl, d_v=dv, gr=g, Ma=M_a, n=N):
        return lib.impala_mlp_backward_shared(p(x_), code, p(params), p(d_l), p(d_v), p(gr), p(ws), ws_n, Ma, M, O, H,
                                              n, None)

    for f in (fwd, bwd):
        assert f(n=0) == -1 and f(n=32) == -1 and f(Ma=M + 1) == -1 and f(code=7) == -1 and f(x_=None) == -1
        assert f(code=_cabi.OBS_U8) == -2  # byte rows need O > 128
        assert f() == 0
    assert fwd(lg=None) == -1 and fwd(vals=None) == -1
    assert bwd(d_l=None) == -1 and bwd(d_v=None) == -1 and bwd(gr=None) == -1
    torch.cuda.synchronize()


# -------------------------------------------------------------------------------------------- engine
ENGINE = {  # T, B, O, A, H, obs kind, gaussian
    "c4": (20, 1024, 24, 4, 256, "normal", False),
    "ram_ragged": (20, 512, 128, 18, 256, "normal", False),
    "ram4_u8": (20, 512, 512, 18, 256, "bytes", False),
    "cartpole": (20, 256, 4, 2, 32, "normal", False),
    "gauss_a6": (20, 1024, 28, 6, 256, "normal", True),
}


def _batch(seed, T, B, O, A, kind, gaussian, params):
    if gaussian:
        return synth.make_gaussian_batch(seed, T, B, O, A, ragged=True, params=params)
    return synth.make_batch(seed, T, B, O, A, ragged=True, obs_kind=kind)


def _flat(eng, views):
    flat = np.zeros(eng.n_total)
    for grp, key, off, shp in eng._segments():
        flat[off:off + int(np.prod(shp))] = np.asarray(views[grp][key], np.float64).reshape(-1)
    return flat


def _engine(T, B, O, A, H, kind, gaussian, hp, **kw):
    return LearnerEngine(T, B, O, A, H, H, hp, shared_torso=True, obs_dtype="uint8" if kind != "normal" else "float32",
                         action_dist="gaussian" if gaussian else "categorical", **kw)


@pytest.mark.parametrize("config", list(ENGINE))
def test_engine_first_step_parity(config):
    T, B, O, A, H, kind, gaussian = ENGINE[config]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    N = 2 * A if gaussian else A
    params = synth.init_params(11, O, N, H)
    if kind != "normal":  # byte observations: a smaller first layer keeps the pre-activations O(1)
        for grp in params.values():
            grp["model.0.weight"] = np.asarray(grp["model.0.weight"]) / 64.0
    batch = _batch(21, T, B, O, A, kind, gaussian, params)
    eng = _engine(T, B, O, A, H, kind, gaussian, hp)
    eng.load_state(params)
    eng.fill_host(batch, 0)
    eng.ingest(0)
    eng.step(0)
    sc = eng.read_scalars()
    eng.synchronize()
    lrn = sorc.SharedLearner(params, hp, gaussian=gaussian)
    out = lrn.forward_backward(batch)
    valid_v = np.arange(T + 1)[:, None] <= batch["lens"][None, :]
    assert np.abs(np.where(valid_v, eng.vs.cpu().numpy(), 0.0) - out["vs"]).max() < 1e-5
    assert np.abs(eng.pg_adv.cpu().numpy() - out["pg_adv"]).max() < 1e-5
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
        assert abs(sc[k] - out[k]) < 1e-5 * max(1.0, abs(out[k])), (k, sc[k], out[k])
    ref = _flat(eng, sorc.views(out["grad"]))
    grad = eng.comm[:eng.n_total].cpu().numpy()
    gmax = np.abs(ref).max()
    assert np.abs(grad - ref).max() / gmax < 5e-5
    norms = lrn.apply(out["grad"])
    assert abs(sc["norm_policy"] - norms["norm_policy"]) <= 5e-5 * norms["norm_policy"]
    assert sc["norm_value"] == 0.0  # one clip norm over the whole network
    want = _flat(eng, lrn.views())
    resolved = np.abs(ref) > 1e-3 * gmax
    after = eng.params.cpu().numpy().astype(np.float64)
    assert np.abs(after - want)[resolved].max() < 5e-5
    st = eng.state()
    assert torch.equal(st["policy"]["model.0.weight"], st["value_fn"]["model.0.weight"])
    assert st["policy"]["model.3.weight"].shape == (N, H) and st["value_fn"]["model.3.weight"].shape == (1, H)
    before = eng.params.clone()
    eng.load_state(st)  # round trip: exact
    assert torch.equal(eng.params, before)


def test_engine_flags_over_updates():
    """Diagnostics, PopArt and reward clipping through three updates against the oracle (PopArt statistics and the
    value head's rescale included)."""
    T, B, O, A, H = 20, 512, 24, 4, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    params = synth.init_params(5, O, A, H)
    eng = LearnerEngine(T, B, O, A, H, H, hp, shared_torso=True, diagnostics=True, popart=True, popart_beta=0.1,
                        reward_clip="soft_asymmetric")
    eng.load_state(params)
    lrn = sorc.SharedLearner(params, hp, reward_clip="soft_asymmetric", popart=True, beta=0.1)
    for u in range(3):
        b = synth.make_batch(40 + u, T, B, O, A, ragged=True)
        b["rewards"] *= 4.0
        eng.fill_host(b, 0)
        eng.ingest(0)
        eng.step(0)
        sc = eng.read_scalars()
        out = lrn.update(b)
        for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
            assert abs(sc[k] - out[k]) < 1e-4 * max(1.0, abs(out[k])), (u, k, sc[k], out[k])
        st = eng.popart_stats()
        assert abs(st["mu"] - lrn.mu) < 1e-5 and abs(st["nu"] - lrn.nu) < 1e-5, (u, st, lrn.mu, lrn.nu)
        assert sc["norm_value"] == 0.0 and np.isfinite(sc["value_explained_variance"])
    got = eng.state()
    want = lrn.views()
    for g in ("policy", "value_fn"):
        for k in orc.PKEYS:
            w = np.asarray(want[g][k])
            assert np.abs(got[g][k].numpy() - w).max() < 2e-4 * max(1.0, np.abs(w).max()), (g, k)


@pytest.mark.parametrize("O,kind", [(512, "bytes"), (32, "planes")])
def test_frames_equal_dense(O, kind):
    """frames=4 (unstacked on the device) bit-equal to the same engine fed the dense rows."""
    T, B, A, H = 20, 256, 6, 256
    hp = default_hparams(batch_size=B, max_timesteps=T)
    params = synth.init_params(3, O, A, H)
    for grp in params.values():
        grp["model.0.weight"] = np.asarray(grp["model.0.weight"]) / 64.0
    fb = synth.make_batch(8, T, B, O, A, ragged=True, obs_kind=kind, frames=4)
    db = synth.stack_frames(fb, 4)
    engs = []
    for frames, b in ((4, fb), (1, db)):
        e = LearnerEngine(T, B, O, A, H, H, hp, shared_torso=True, obs_dtype="uint8", frames=frames)
        e.load_state(params)
        for _ in range(2):
            e.fill_host(b, 0)
            e.ingest(0)
            e.step(0)
        e.synchronize()
        engs.append(e)
    assert torch.equal(engs[0].params, engs[1].params)
    assert torch.equal(engs[0].comm, engs[1].comm)


def test_replay_equals_plain_engine_on_composed_batches():
    """A shared replay engine is torch.equal to a plain shared engine fed the batches its compose launch built."""
    from torched_impala_b200 import ops

    T, B, O, A, H, R, Br = 20, 512, 24, 4, 256, 2, 128
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    rep = LearnerEngine(T, B, O, A, H, H, hp, shared_torso=True, replay_slabs=R, replay_columns=Br)
    plain = LearnerEngine(T, B, O, A, H, H, hp, shared_torso=True)
    params = synth.init_params(5, O, A, H)
    rep.load_state(params)
    plain.load_state(params)
    for u in range(4):
        rep.fill_host(synth.make_batch(70 + u, T, B - Br, O, A, ragged=True), u % 2)
        rep.ingest(u % 2)
        rep.step(u % 2)
        rep.synchronize()
        plan = torch.from_numpy(np.ascontiguousarray(rep.replay_plan)).cuda()
        composed = ops.batch_compose(rep.store, plan, T, B, B - Br, O, 1, A)
        assert torch.equal(composed, rep.d_slabs[u % 2])
        for name, _ in plain.fields:
            plain.h_views[u % 2][name][...] = rep.d_views[u % 2][name].cpu().numpy()
        plain.ingest(u % 2)
        plain.step(u % 2)
        plain.synchronize()
        assert rep.read_scalars() == plain.read_scalars()
    for name in ("params", "adam_m", "adam_v", "adam_step"):
        assert torch.equal(getattr(rep, name), getattr(plain, name)), name


def test_forked_learner(tmp_path):
    """A forked shared-torso Learner behind a RingQueue: the published policy and value_fn modules are the views of
    the oracle network, the checkpoint the learner wrote reloads exactly, and the reference's MlpPolicy loads its
    policy view (where oracle/_ref was built)."""
    import shared_torso_learner_process_check as chk
    from torched_impala_b200 import models
    from torched_impala_b200.learner import Learner

    out = tmp_path / "weights.npz"
    res = subprocess.run([sys.executable, chk.__file__, str(tmp_path / "logs"), str(out)], capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "SHARED_LEARNER_OK" in res.stdout
    got = np.load(out)
    assert int(got["published"]) >= 2 and int(got["published"]) % 2 == 0
    want = chk.oracle_run()
    for g in ("policy", "value_fn"):
        for key in orc.PKEYS:
            d = np.abs(got[f"{g}/{key}"] - want[g][key]).max()
            assert d < 1e-4, (g, key, d)
    for key in orc.PKEYS[:2]:  # one torso behind both views
        assert np.array_equal(got[f"policy/{key}"], got[f"value_fn/{key}"]), key
    ckpts = sorted((tmp_path / "logs").glob("**/*.pt"))
    assert ckpts, "the learner wrote no checkpoint"
    ckpt = torch.load(ckpts[-1])
    assert ckpt["shared_torso"] is True
    for g, sd in (("policy", ckpt["policy_state_dict"]), ("value_fn", ckpt["value_fn_state_dict"])):
        for key in orc.PKEYS:
            assert np.array_equal(sd[key].numpy(), got[f"{g}/{key}"]), (g, key)
    hp, _, _ = chk.setup()
    pol, vf = models.MlpPolicy(chk.O, chk.A, chk.H), models.MlpValueFn(chk.O, chk.H)
    lrn = Learner(2, hp, pol, vf, None, None, shared_torso=True)
    lrn.load(str(ckpts[-1]))
    for mod, g in ((pol, "policy"), (vf, "value_fn")):
        for key, t in mod.state_dict().items():
            assert np.array_equal(t.numpy(), got[f"{g}/{key}"]), (g, key)
    from oracle import refload

    if not refload.available():
        pytest.skip("the reference (oracle/_ref) was not built")
    code = ("import sys, torch; sys.path.insert(0, sys.argv[1]); from oracle import refload; "
            "m = refload.load()[1]; p = m.MlpPolicy(int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])); "
            "p.load_state_dict(torch.load(sys.argv[2])['policy_state_dict']); print('REF_LOAD_OK')")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", code, root, str(ckpts[-1]), str(chk.O), str(chk.A), str(chk.H)],
                         capture_output=True, text=True, timeout=120, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert "REF_LOAD_OK" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


@pytest.mark.parametrize("allreduce", ["peer", "nccl"])
def test_two_gpus(allreduce):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs (data-parallel path)")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_shared_torso_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240, env=dict(os.environ, IMPALA_ALLREDUCE=allreduce))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_SHARED_OK" in res.stdout
