"""GPU: multi-discrete policies - impala_vtrace_loss_md against the float64 oracle (tests/multi_discrete_oracle.py)
for every flag combination and the K = 1 identity with the categorical kernel; LearnerEngine(action_dist=
"multi_discrete") at full size against the oracle learner, with the categorical engine's launch count, and replay
equal to the plain engine."""
import numpy as np
import pytest
import torch

import multi_discrete_oracle as morc
from mlp_bounds import MlpBound
from test_gpu_wide_shapes import check_engine_mlp
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.engine import LearnerEngine
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


VARIANTS = ("plain", "diag", "popart")
CLIPS = (None, "abs_one", "soft_asymmetric")
POPART = (0.3, 1.7)  # (mu, sigma) of the PopArt cases
# N = AP (the VEC path) and N off a multiple of 4 (the element path), AP 2 to 32, K 1 to 16
HEADS = {"2": (2,), "3x3": (3, 3), "332": (3, 3, 2), "574": (5, 7, 4), "2x8": (2,) * 8, "ram": (3, 3, 2, 2, 5, 5),
         "16x16": (16, 16), "2x16": (2,) * 16}


def _check(got, want, c, T, B):
    # 1e-5 absolute, or 1e-6 of the largest entry: the reference-mode recurrence of T = 100 steps carries vs and pg_adv
    # to magnitudes of ~20 in float32 (the categorical kernel's recurrence, unchanged)
    valid_v = np.arange(T + 1)[:, None] <= c["lens"][None, :]
    err = np.abs(np.where(valid_v, got["vs"].cpu().numpy(), 0.0) - want["vs"]).max()
    assert err < max(1e-5, 1e-6 * np.abs(want["vs"]).max()), ("vs", err)
    for k in ("pg_adv", "dlogits", "dv"):
        err = np.abs(got[k].cpu().numpy() - want[k]).max()
        assert err < max(1e-5, 1e-6 * np.abs(want[k]).max()), (k, err, np.abs(want[k]).max())
    s = got["scalars"].cpu().tolist()
    for i, k in enumerate(("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward")):
        assert abs(s[i] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, s[i], want[k])
    if "diag" in got:
        d, wd = got["diag"].cpu().numpy(), want["diag"]
        # the clip counts: a float32 ratio within rounding of rho_bar / c_bar may land on the other side
        assert d[0] == wd[0] and abs(d[2] - wd[2]) <= 2 and abs(d[3] - wd[3]) <= 2, (d, wd)
        for j in (1, 4, 5, 6, 7):
            assert abs(d[j] - wd[j]) <= 1e-4 * max(1.0, abs(wd[j])), (j, d[j], wd[j])


@pytest.mark.parametrize("reward_clip", CLIPS)
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("T", [20, 100])
@pytest.mark.parametrize("heads", list(HEADS))
def test_kernel_against_oracle(ops, heads, T, mode, variant, reward_clip):
    heads = HEADS[heads]
    B = 80  # two full lane groups and a partial one
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    c = morc.make_inputs(7 * sum(heads) + len(heads) + T, T, B, heads)
    if reward_clip == "abs_one":
        c["rewards"] = (c["rewards"] * 3.0).astype(np.float32)
    pop = POPART if variant == "popart" else None
    if pop:
        c["v"] = ((c["v"] - pop[0]) / pop[1]).astype(np.float32)
    want = morc.vtrace_loss(c["v"], c["cur"], c["beh"], c["actions"], c["rewards"], c["done"], c["lens"], hp, B,
                            heads, mode, reward_clip, pop)
    args = [dev(c[k]) for k in ("cur", "beh", "actions", "rewards", "done", "lens", "v")]
    popart = ops.popart_stats(mu=pop[0], nu=pop[1] ** 2 + pop[0] ** 2) if pop else None
    got = ops.vtrace_loss_md(*args, hp, 1.0 / B, heads, mode=mode, diagnostics=variant == "diag", popart=popart,
                             reward_clip=reward_clip)
    torch.cuda.synchronize()
    _check(got, want, c, T, B)


@pytest.mark.parametrize("variant", VARIANTS + ("rclip",))
@pytest.mark.parametrize("N", [2, 3, 4, 5, 8, 13, 16, 24, 32])
def test_one_head_equals_the_categorical_kernel(ops, N, variant):
    T, B = 20, 80
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    c = morc.make_inputs(N, T, B, (N,))
    args = [dev(c[k]) for k in ("cur", "beh", "actions", "rewards", "done", "lens", "v")]
    kw = dict(diagnostics=variant == "diag", popart=ops.popart_stats(mu=0.3, nu=3.0) if variant == "popart" else None,
              reward_clip="abs_one" if variant == "rclip" else None)
    got = ops.vtrace_loss_md(*args, hp, 1.0 / B, (N,), **kw)
    cat_args = list(args)
    cat_args[2] = args[2][..., 0].contiguous()
    if variant == "rclip":
        want = ops.vtrace_loss_rclip(*cat_args, hp, 1.0 / B, "abs_one")
    elif variant == "popart":
        want = ops.vtrace_loss_popart(*cat_args, hp, 1.0 / B, kw["popart"])
    elif variant == "diag":
        want = ops.vtrace_loss_diag(*cat_args, hp, 1.0 / B)
    else:
        want = ops.vtrace_loss(*cat_args, hp, 1.0 / B)
    torch.cuda.synchronize()
    # the ratio is formed from other float32 roundings than the categorical kernel's (per-entry differences): each
    # output within 1e-6 of its largest entry (1e-6 absolute below magnitude 1)
    for k in ("vs", "pg_adv", "dlogits", "dv", "scalars"):
        err = (got[k].double() - want[k].double()).abs().max().item()
        assert err <= 1e-6 * max(1.0, want[k].double().abs().max().item()), (k, err)
    if "diag" in want:
        d, wd = got["diag"].cpu().numpy(), want["diag"].cpu().numpy()
        assert d[0] == wd[0] and abs(d[2] - wd[2]) <= 2 and abs(d[3] - wd[3]) <= 2, (d, wd)
        # the log-ratio and KL sums pin the difference form of the ratio and KL to the categorical one: 1e-7 per valid
        # step (the sums are float32 per thread, ~d[0] roundings of their own), 1e-5 of the sum at least
        for j in (1, 4):
            assert abs(d[j] - wd[j]) <= max(1e-7 * d[0], 1e-5 * max(1.0, abs(wd[j]))), (j, d[j], wd[j])
        # the sums of vs, vs^2 and vs - v over the d[0] valid steps: what the per-entry vs bound above allows
        e = 1e-6 * max(1.0, want["vs"].double().abs().max().item())
        vmax = want["vs"].double().abs().max().item()
        for j, tol in ((5, d[0] * e), (6, d[0] * e * (2 * vmax + e)), (7, d[0] * e)):
            assert abs(d[j] - wd[j]) <= tol, (j, d[j], wd[j], tol)


def test_refused_arguments(ops):
    import ctypes as C

    lib = _cabi.lib()
    T, B = 4, 32
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device="cuda")  # noqa: E731
    ws = torch.zeros(int(lib.impala_vtrace_loss_diag_workspace(T, B, 40)), dtype=torch.uint8, device="cuda")
    diag = torch.zeros(8, dtype=torch.float64, device="cuda")
    pop = ops.popart_stats()
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731

    def call(heads, d=None, pp=None, rc=0, A=None, K=None, null_heads=False):
        N, Kh = sum(heads), len(heads)
        A = N if A is None else A
        cur, act = f(T, B, max(A, 1)), torch.zeros(T, B, max(Kh, 1), dtype=torch.int32, device="cuda")
        h = None if null_heads else (C.c_int32 * max(Kh, 1))(*heads)
        return lib.impala_vtrace_loss_md(
            p(cur), p(cur), p(act), p(f(T, B)), p(torch.zeros(T, B, dtype=torch.uint8, device="cuda")),
            p(torch.full((B,), T, dtype=torch.int32, device="cuda")), p(f(T + 1, B)), p(f(T + 1, B)), p(f(T, B)),
            p(f(T, B, max(A, 1))), p(f(T + 1, B)), p(torch.zeros(4, dtype=torch.float64, device="cuda")), p(ws),
            ws.numel(), T, B, A, 0.99, 1.0, 1.0, 0.5, 1.0, 0.01, 1.0 / B, 0, p(d), p(pp), rc, h,
            Kh if K is None else K, None)

    assert call((3, 3), null_heads=True) == -1
    assert call((3, 1, 2)) == -1 and call((3, 3), A=7) == -1 and call((3, 3), A=5) == -1
    assert call((3, 3), K=0) == -1
    assert call((2,) * 17) == -2 and call((20, 20)) == -2
    assert call((3, 3), pp=pop) == -1  # PopArt needs the diagnostic sums
    assert call((3, 3), d=diag, rc=3) == -1 and call((3, 3), rc=-1) == -1
    assert call((16, 16), d=diag, pp=pop, rc=2) == 0 and call((2,)) == 0 and call((2,) * 16, d=diag) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- engine
FULL = {"md_c4": (20, 4096, 24, (3, 3, 2), 256), "md_ram": (20, 4096, 128, (3, 3, 2, 2, 5, 5), 256)}  # T, B, O, heads, H


def md_batch(seed, T, B, O, heads, params, ragged=True):
    """obs N(0, 1), behaviour logits 0.1-0.3 from the policy's own logits, one action per head sampled from them."""
    b = synth.make_md_batch(seed, T, B, O, heads, ragged=ragged, params=params)
    return b


def _tied(eng, params, batch):
    """Gradient entries of the hidden units with a ReLU tie (tests/test_gpu_wide_shapes.py's check_grad_end_to_end)."""
    obs = np.asarray(batch["obs"])
    O = obs.shape[2]
    x = {"policy": obs[:-1].reshape(-1, O), "value_fn": obs.reshape(-1, O)}
    tied = np.zeros(eng.n_total, bool)
    for grp in ("policy", "value_fn"):
        bound = MlpBound(x[grp], params[grp])
        units = torch.nonzero((bound.pre.abs() < bound.e_pre).any(dim=0)).flatten().tolist()
        segs = {key: (off, shp) for g, key, off, shp in eng._segments() if g == grp}
        off_w, shp_w = segs[orc.PKEYS[0]]
        off_b, _ = segs[orc.PKEYS[1]]
        for j in units:
            tied[off_w + j * shp_w[1]:off_w + (j + 1) * shp_w[1]] = tied[off_b + j] = True
    return tied


def _flat(eng, per_group):
    flat = np.zeros(eng.n_total)
    for grp, key, off, shp in eng._segments():
        flat[off:off + int(np.prod(shp))] = np.asarray(per_group[grp][orc.PKEYS.index(key)]).reshape(-1)
    return flat


@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("config", list(FULL))
def test_engine_first_step_parity(config, mode):
    T, B, O, heads, H = FULL[config]
    N = sum(heads)
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    eng = LearnerEngine(T, B, O, N, H, H, hp, mode=mode, action_dist="multi_discrete", action_heads=heads,
                        use_graph=False)  # check_engine_mlp reads the rows of the eager step
    params = synth.init_params(11, O, N, H)
    batch = md_batch(21, T, B, O, heads, params)
    eng.load_state(params)
    eng.fill_host(batch, 0)
    eng.ingest(0)
    eng.step(0)
    sc = eng.read_scalars()
    eng.synchronize()
    orc_l = morc.MdLearner(params, hp, heads)
    out = orc_l.forward_backward(batch, mode)
    valid_v = np.arange(T + 1)[:, None] <= batch["lens"][None, :]
    assert np.abs(np.where(valid_v, eng.vs.cpu().numpy(), 0.0) - out["vs"]).max() < 1e-5
    assert np.abs(eng.pg_adv.cpu().numpy() - out["pg_adv"]).max() < 1e-5
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
        assert abs(sc[k] - out[k]) < 1e-5 * max(1.0, abs(out[k])), (k, sc[k], out[k])
    ref_grad = _flat(eng, {"policy": out["g_policy"], "value_fn": out["g_value"]})
    grad = eng.comm[:eng.n_total].cpu().numpy()
    gmax = np.abs(ref_grad).max()
    # oracle/check.py's 5e-5 of the largest entry, the W1 row and b1 entry of ReLU-tied hidden units (a pre-activation
    # within its float32 error bound of 0: md_ram's 128 features have such units) left to check_engine_mlp, which bounds
    # every MLP output and gradient entry of the engine's step against float64, as tests/test_gpu_wide_shapes.py does
    tied = _tied(eng, params, batch)
    assert np.abs(grad - ref_grad)[~tied].max() / gmax < 5e-5
    check_engine_mlp(eng, params)
    norms = orc_l.apply(out["g_policy"], out["g_value"])
    for k in ("norm_policy", "norm_value"):
        assert abs(sc[k] - norms[k]) <= 5e-5 * norms[k], (k, sc[k], norms[k])
    want_after = _flat(eng, {g: [orc_l.state()[g][k] for k in orc.PKEYS] for g in ("policy", "value_fn")})
    resolved = np.abs(ref_grad) > 1e-3 * gmax
    after = eng.params.cpu().numpy().astype(np.float64)
    assert np.abs(after - want_after)[resolved].max() < 5e-5
    assert eng.state()["policy"]["model.3.weight"].shape == (N, H)


@pytest.mark.parametrize("shared_torso", [False, True])
def test_engine_flags_and_launch_count(shared_torso):
    """Diagnostics + PopArt + reward clip through the multi-discrete slot at md_c4 (and with a shared torso): the
    first update's scalars, off-policy KL and PopArt statistics against the oracle, and the launch count of the
    categorical engine at the same N."""
    T, B, O, heads, H = FULL["md_c4"]
    N = sum(heads)
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    kw = dict(diagnostics=True, popart=True, popart_beta=0.1, reward_clip="soft_asymmetric", shared_torso=shared_torso)
    g = LearnerEngine(T, B, O, N, H, H, hp, action_dist="multi_discrete", action_heads=heads, **kw)
    c = LearnerEngine(T, B, O, N, H, H, hp, **kw)
    params = synth.init_params(4, O, N, H)
    g.load_state(params)
    c.load_state(params)
    st0 = g.state()  # the value view the first update starts from (shared torso: the policy's torso)
    b0 = md_batch(39, T, B, O, heads, params)
    g.fill_host(b0, 0)
    g.ingest(0)
    g.step(0)
    s0 = g.read_scalars()
    f64 = {k: [np.asarray(params[k][n], np.float64) for n in orc.PKEYS] for k in ("policy", "value_fn")}
    obs = b0["obs"].astype(np.float64)
    z = orc.mlp_forward(obs[:-1], *f64["policy"])[0]
    vf = [np.asarray(st0["value_fn"][n], np.float64) for n in orc.PKEYS]
    v = orc.mlp_forward(obs, *vf)[0][..., 0]
    want = morc.vtrace_loss(v, z, b0["beh_logits"], b0["actions"], b0["rewards"], b0["done"], b0["lens"], hp, B,
                            heads, "reference", "soft_asymmetric", (0.0, 1.0))
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
        assert abs(s0[k] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, s0[k], want[k])
    n, s1, s2 = want["diag"][0], want["diag"][5], want["diag"][6]
    mu1, nu1 = 0.1 * s1 / n, 0.9 + 0.1 * s2 / n  # beta = 0.1 from mu = 0, nu = 1
    st = g.popart_stats()
    assert abs(st["mu"] - mu1) < 1e-5 and abs(st["nu"] - nu1) < 1e-5, (st, mu1, nu1)
    kl = want["diag"][4] / n
    assert abs(s0["kl_behaviour_current"] - kl) < 1e-5 * max(1.0, kl), (s0["kl_behaviour_current"], kl)
    for u in range(3):
        gb = md_batch(40 + u, T, B, O, heads, params)
        cb = synth.make_batch(40 + u, T, B, O, N, ragged=True)
        for e, b in ((g, gb), (c, cb)):
            e.fill_host(b, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
        s = g.read_scalars()
        c.read_scalars()
        assert all(np.isfinite(s[k]) for k in ("value_fn_loss", "policy_loss", "policy_entropy",
                                               "kl_behaviour_current", "popart_sigma")), s
    g.synchronize()
    c.synchronize()
    assert g.launches_per_step == c.launches_per_step


def test_replay_equals_plain_engine_on_composed_batches(ops):
    """A multi-discrete replay engine is torch.equal to a plain one fed the batches its compose launch built."""
    T, B, O, heads, H, R, Br = 20, 512, 24, (3, 3, 2), 256, 2, 128
    N = sum(heads)
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    kw = dict(action_dist="multi_discrete", action_heads=heads)
    rep = LearnerEngine(T, B, O, N, H, H, hp, replay_slabs=R, replay_columns=Br, **kw)
    plain = LearnerEngine(T, B, O, N, H, H, hp, **kw)
    params = synth.init_params(5, O, N, H)
    rep.load_state(params)
    plain.load_state(params)
    for u in range(4):
        fresh = md_batch(70 + u, T, B - Br, O, heads, params)
        rep.fill_host(fresh, u % 2)
        rep.ingest(u % 2)
        rep.step(u % 2)
        rep.synchronize()
        composed = ops.batch_compose(rep.store, dev(rep.replay_plan), T, B, B - Br, O, 1, N, **kw)
        assert torch.equal(composed, rep.d_slabs[u % 2])
        for name, _ in plain.fields:
            plain.h_views[u % 2][name][...] = rep.d_views[u % 2][name].cpu().numpy()
        plain.ingest(u % 2)
        plain.step(u % 2)
        plain.synchronize()
        assert rep.read_scalars() == plain.read_scalars()
    for name in ("params", "adam_m", "adam_v", "adam_step"):
        assert torch.equal(getattr(rep, name), getattr(plain, name)), name
