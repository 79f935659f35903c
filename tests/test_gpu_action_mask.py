"""GPU: invalid-action masking - impala_vtrace_loss_mask against the float64 oracle (tests/action_mask_oracle.py) for
categorical and multi-discrete policies, every flag combination and mask density; a full mask bitwise equal to the
unmasked kernels; outputs independent of what the illegal logits hold; padded steps; LearnerEngine(action_mask=True)
against the oracle learner with the unmasked engine's launch count, replay and uint8 frames."""
import numpy as np
import pytest
import torch

import action_mask_oracle as aorc
from test_gpu_multi_discrete import HEADS as MD_HEADS
from test_gpu_multi_discrete import _check, _flat, _tied
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
POPART = (0.3, 1.7)
# categorical: VEC (A = AP), the element path and the streaming rows (A > 16); multi-discrete: the MD test's heads
KINDS = {f"cat{A}": (A,) for A in (2, 3, 4, 5, 8, 9, 16, 18, 32)}
KINDS.update({f"md{k}": h for k, h in MD_HEADS.items()})
DENSITY = {"half": 0.5, "single": 0.0, "full": 1.0}  # single: one legal entry per head at every step


def _inputs(kind, T, B, density, seed=0):
    heads = KINDS[kind]
    d = DENSITY[density]
    c = aorc.make_inputs(seed + 7 * sum(heads) + len(heads) + T, T, B, heads, density=d if d > 0 else 0.5,
                         single=1.0 if d == 0 else 0.1)
    return heads, kind.startswith("md"), c


def _run(ops, c, heads, md, hp, B, mode="reference", variant="plain", reward_clip=None, pop=None):
    args = [dev(c[k]) for k in ("cur", "beh", "actions", "rewards", "done", "lens", "v")]
    popart = ops.popart_stats(mu=pop[0], nu=pop[1] ** 2 + pop[0] ** 2) if pop else None
    return ops.vtrace_loss_mask(*args, hp, 1.0 / B, heads if md else (), mode=mode, diagnostics=variant == "diag",
                                popart=popart, reward_clip=reward_clip)


@pytest.mark.parametrize("reward_clip", CLIPS)
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("T", [20, 100])
@pytest.mark.parametrize("kind", list(KINDS))
def test_kernel_against_oracle(ops, kind, T, mode, variant, reward_clip):
    B = 80
    # rho_bar and c_bar off 1: a step with one legal entry per head has ratio 1 up to rounding, on either side of it
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.05, c_bar=0.95)
    # the densities in turn over the flag combinations (every kind and T sees all three)
    density = list(DENSITY)[(VARIANTS.index(variant) + CLIPS.index(reward_clip)) % 3]
    heads, md, c = _inputs(kind, T, B, density)
    if reward_clip == "abs_one":
        c["rewards"] = (c["rewards"] * 3.0).astype(np.float32)
    pop = POPART if variant == "popart" else None
    if pop:
        c["v"] = ((c["v"] - pop[0]) / pop[1]).astype(np.float32)
    want = aorc.vtrace_loss(c["v"], c["cur"], c["beh"], c["idx"], c["legal"], c["rewards"], c["done"], c["lens"], hp,
                            B, heads, mode, reward_clip, pop)
    got = _run(ops, c, heads, md, hp, B, mode, variant, reward_clip, pop)
    torch.cuda.synchronize()
    _check(got, want, c, T, B)
    ill = ~aorc.normalise(c["legal"], heads)
    assert (got["dlogits"].cpu().numpy()[ill] == 0).all()


@pytest.mark.parametrize("variant", VARIANTS + ("rclip",))
@pytest.mark.parametrize("kind", list(KINDS))
def test_full_mask_is_the_unmasked_kernel(ops, kind, variant):
    T, B = 20, 80
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    heads, md, c = _inputs(kind, T, B, "full")
    # every legal bit set, padded steps included
    c["actions"][..., -1] = np.int32(-1) if sum(heads) == 32 else np.int32((1 << sum(heads)) - 1)
    args = [dev(c[k]) for k in ("cur", "beh", "actions", "rewards", "done", "lens", "v")]
    pop = ops.popart_stats(mu=0.3, nu=3.0) if variant == "popart" else None
    kw = dict(diagnostics=variant == "diag", popart=pop, reward_clip="abs_one" if variant == "rclip" else None)
    got = ops.vtrace_loss_mask(*args, hp, 1.0 / B, heads if md else (), **kw)
    plain = list(args)
    if md:
        plain[2] = args[2][..., :-1].contiguous()
        want = ops.vtrace_loss_md(*plain, hp, 1.0 / B, heads, **kw)
    else:
        plain[2] = args[2][..., 0].contiguous()
        if variant == "rclip":
            want = ops.vtrace_loss_rclip(*plain, hp, 1.0 / B, "abs_one")
        elif variant == "popart":
            want = ops.vtrace_loss_popart(*plain, hp, 1.0 / B, pop)
        elif variant == "diag":
            want = ops.vtrace_loss_diag(*plain, hp, 1.0 / B)
        else:
            want = ops.vtrace_loss(*plain, hp, 1.0 / B)
    torch.cuda.synchronize()
    for k in want:
        assert torch.equal(got[k], want[k]), k


@pytest.mark.parametrize("kind", list(KINDS))
def test_illegal_entries_never_reach_an_output(ops, kind):
    T, B = 20, 80
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    heads, md, c = _inputs(kind, T, B, "half")
    ill = ~aorc.normalise(c["legal"], heads)
    outs = []
    for fill in (-np.inf, np.nan, 1e30, -1e30, None):
        x = dict(c)
        if fill is not None:
            x["cur"] = np.where(ill, np.float32(fill), c["cur"]).astype(np.float32)
            x["beh"] = np.where(ill, np.float32(fill), c["beh"]).astype(np.float32)
        else:  # raw logits
            rng = np.random.default_rng(1)
            x["cur"] = np.where(ill, rng.standard_normal(ill.shape), c["cur"]).astype(np.float32)
            x["beh"] = np.where(ill, rng.standard_normal(ill.shape), c["beh"]).astype(np.float32)
        outs.append(_run(ops, x, heads, md, hp, B, variant="diag"))
    torch.cuda.synchronize()
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(o[k], outs[0][k]), k
    assert (outs[0]["dlogits"].cpu().numpy()[ill] == 0).all()


@pytest.mark.parametrize("kind", ["cat5", "cat8", "cat18", "md332", "mdram"])
def test_padded_steps_and_empty_columns(ops, kind):
    T, B = 20, 64
    hp = default_hparams(batch_size=B, max_timesteps=T)
    heads, md, c = _inputs(kind, T, B, "half")
    c["lens"][:8] = 0  # empty columns: every byte of the step rows 0, legal words 0
    pad = np.arange(T)[:, None] >= c["lens"][None, :]
    c["actions"][pad] = 0
    c["cur"][pad], c["beh"][pad] = 0.0, 0.0
    got = _run(ops, c, heads, md, hp, B, variant="diag")
    torch.cuda.synchronize()
    for k, t in got.items():
        assert torch.isfinite(t).all(), k
    assert (got["dlogits"].cpu().numpy()[pad] == 0).all()


# ---------------------------------------------------------------------------------------------- engine
FULL = {"mask_c4": (20, 4096, 24, 8, (), 256, "float32"), "mask_ram": (20, 4096, 128, 18, (), 256, "uint8"),
        "md_mask_c4": (20, 4096, 24, 8, (3, 3, 2), 256, "float32")}  # T, B, O, A, heads, H, obs


def mask_batch(seed, T, B, O, A, heads, params, obs_dtype="float32", frames=1):
    kind = "planes" if obs_dtype == "uint8" else "normal"  # MinAtar-like 0/1 bytes
    return synth.make_masked_batch(seed, T, B, O, A, heads, density=0.5, ragged=True, params=params, obs_kind=kind,
                                   frames=frames)


def _engine_kw(heads):
    return dict(action_mask=True, **(dict(action_dist="multi_discrete", action_heads=heads) if heads else {}))


@pytest.mark.parametrize("config", list(FULL))
def test_engine_first_step_parity(config):
    from test_gpu_wide_shapes import check_engine_mlp

    T, B, O, A, heads, H, obs_dtype = FULL[config]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    eng = LearnerEngine(T, B, O, A, H, H, hp, obs_dtype=obs_dtype, use_graph=False, **_engine_kw(heads))
    plain = LearnerEngine(T, B, O, A, H, H, hp, obs_dtype=obs_dtype,
                          **(dict(action_dist="multi_discrete", action_heads=heads) if heads else {}))
    params = synth.init_params(11, O, A, H)
    batch = mask_batch(21, T, B, O, A, heads, params, obs_dtype)
    eng.load_state(params)
    eng.fill_host(batch, 0)
    eng.ingest(0)
    eng.step(0)
    sc = eng.read_scalars()
    eng.synchronize()
    orc_l = aorc.MaskLearner(params, hp, heads or (A,))
    out = orc_l.forward_backward(batch)
    valid_v = np.arange(T + 1)[:, None] <= batch["lens"][None, :]
    assert np.abs(np.where(valid_v, eng.vs.cpu().numpy(), 0.0) - out["vs"]).max() < 1e-5
    assert np.abs(eng.pg_adv.cpu().numpy() - out["pg_adv"]).max() < 1e-5
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
        assert abs(sc[k] - out[k]) < 1e-5 * max(1.0, abs(out[k])), (k, sc[k], out[k])
    ref_grad = _flat(eng, {"policy": out["g_policy"], "value_fn": out["g_value"]})
    grad = eng.comm[:eng.n_total].cpu().numpy()
    tied = _tied(eng, params, batch)
    assert np.abs(grad - ref_grad)[~tied].max() / np.abs(ref_grad).max() < 5e-5
    if obs_dtype == "float32":
        check_engine_mlp(eng, params)
    # the launch count of the unmasked engine
    pb = synth.make_batch(21, T, B, O, A, ragged=True, obs_kind="planes" if obs_dtype == "uint8" else "normal")
    if heads:
        pb = synth.make_md_batch(21, T, B, O, heads, ragged=True, obs_kind="planes" if obs_dtype == "uint8" else "normal")
    plain.load_state(params)
    for e, b in ((plain, pb), (eng, batch)):
        e.fill_host(b, 1)
        e.ingest(1)
        e.step(1)
        e.synchronize()
    assert eng.launches_per_step == plain.launches_per_step


@pytest.mark.parametrize("shared_torso", [False, True])
def test_engine_flags(shared_torso):
    """Diagnostics + PopArt + reward clip through the masked slot at mask_c4 (and with a shared torso): the first
    update's scalars, off-policy KL and PopArt statistics against the oracle."""
    T, B, O, A, heads, H, _ = FULL["mask_c4"]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    kw = dict(diagnostics=True, popart=True, popart_beta=0.1, reward_clip="soft_asymmetric", shared_torso=shared_torso)
    g = LearnerEngine(T, B, O, A, H, H, hp, action_mask=True, **kw)
    params = synth.init_params(4, O, A, H)
    g.load_state(params)
    st0 = g.state()
    b0 = mask_batch(39, T, B, O, A, (), params)
    g.fill_host(b0, 0)
    g.ingest(0)
    g.step(0)
    s0 = g.read_scalars()
    f64 = {k: [np.asarray(params[k][n], np.float64) for n in orc.PKEYS] for k in ("policy", "value_fn")}
    obs = b0["obs"].astype(np.float64)
    z = orc.mlp_forward(obs[:-1], *f64["policy"])[0]
    vf = [np.asarray(st0["value_fn"][n], np.float64) for n in orc.PKEYS]
    v = orc.mlp_forward(obs, *vf)[0][..., 0]
    want = aorc.vtrace_loss(v, z, b0["beh_logits"], b0["actions"][..., :-1], b0["legal"], b0["rewards"], b0["done"],
                            b0["lens"], hp, B, (A,), "reference", "soft_asymmetric", (0.0, 1.0))
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
        assert abs(s0[k] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, s0[k], want[k])
    n, s1, s2 = want["diag"][0], want["diag"][5], want["diag"][6]
    st = g.popart_stats()
    assert abs(st["mu"] - 0.1 * s1 / n) < 1e-5 and abs(st["nu"] - (0.9 + 0.1 * s2 / n)) < 1e-5
    kl = want["diag"][4] / n
    assert abs(s0["kl_behaviour_current"] - kl) < 1e-5 * max(1.0, kl), (s0["kl_behaviour_current"], kl)


@pytest.mark.parametrize("heads", [(), (3, 3, 2)])
def test_replay_equals_plain_engine_on_composed_batches(ops, heads):
    """A masked replay engine is torch.equal to a masked engine fed the batches its compose launch built."""
    T, B, O, A, H, R, Br = 20, 512, 24, 8, 256, 2, 128
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    kw = _engine_kw(heads)
    rep = LearnerEngine(T, B, O, A, H, H, hp, replay_slabs=R, replay_columns=Br, **kw)
    plain = LearnerEngine(T, B, O, A, H, H, hp, **kw)
    params = synth.init_params(5, O, A, H)
    rep.load_state(params)
    plain.load_state(params)
    for u in range(4):
        fresh = mask_batch(70 + u, T, B - Br, O, A, heads, params)
        fresh.pop("legal")
        rep.fill_host(fresh, u % 2)
        rep.ingest(u % 2)
        rep.step(u % 2)
        rep.synchronize()
        composed = ops.batch_compose(rep.store, dev(rep.replay_plan), T, B, B - Br, O, 1, A,
                                     action_dist="multi_discrete" if heads else "categorical", action_heads=heads,
                                     action_mask=True)
        assert torch.equal(composed, rep.d_slabs[u % 2])
        for name, _ in plain.fields:
            plain.h_views[u % 2][name][...] = rep.d_views[u % 2][name].cpu().numpy()
        plain.ingest(u % 2)
        plain.step(u % 2)
        plain.synchronize()
        assert rep.read_scalars() == plain.read_scalars()
    for name in ("params", "adam_m", "adam_v", "adam_step"):
        assert torch.equal(getattr(rep, name), getattr(plain, name)), name


def test_uint8_frames_train_as_the_dense_engine():
    """uint8 frames=4 masked slabs train bit for bit as the dense uint8 masked engine on the stacked batch."""
    T, B, O, A, H, k = 20, 512, 128, 18, 256, 4
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    fr = LearnerEngine(T, B, O, A, H, H, hp, obs_dtype="uint8", frames=k, action_mask=True)
    dn = LearnerEngine(T, B, O, A, H, H, hp, obs_dtype="uint8", action_mask=True)
    params = synth.init_params(6, O, A, H)
    fr.load_state(params)
    dn.load_state(params)
    for u in range(3):
        b = mask_batch(80 + u, T, B, O, A, (), params, "uint8", frames=k)
        b.pop("legal")
        dense = dict(synth.stack_frames(b, k))
        for e, x in ((fr, b), (dn, dense)):
            e.fill_host(x, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
            e.synchronize()
        assert fr.read_scalars() == dn.read_scalars()
    assert torch.equal(fr.params, dn.params)
