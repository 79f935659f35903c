"""CPU: invalid-action masking - the float64 oracle (tests/action_mask_oracle.py) against torch autograd and the
unmasked oracles, the slab layouts of the masked kinds, the option checks before any CUDA work, the synthetic batch,
and the SASS of the masked kernels (every launch shape present, no spill where the unmasked twin has none)."""
import ctypes as C
import dataclasses
import json

import numpy as np
import pytest
import torch

import action_mask_oracle as aorc
import multi_discrete_oracle as morc
import reward_clip_oracle as rorc
from test_multi_discrete_cpu import _sass_kernels
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.utils import default_hparams

F64 = torch.float64
HEADS = {"cat5": (5,), "332": (3, 3, 2), "324": (3, 2, 4)}


def _torch_update(x, hp, batch_size, heads, mode, reward_clip):
    """The reference learner's loss one trajectory at a time, with one torch Categorical per head over masked_fill-ed
    logits (-inf at the illegal entries), and autograd for d total / d logits and d total / d v."""
    T, B, N = x["cur"].shape
    legal = torch.tensor(aorc.normalise(x["legal"], heads))
    z = torch.tensor(np.nan_to_num(x["cur"]), dtype=F64, requires_grad=True)
    n = torch.tensor(x["v"], dtype=F64, requires_grad=True)
    beh = torch.tensor(np.nan_to_num(x["beh"]), dtype=F64)
    act = torch.tensor(x["idx"], dtype=torch.int64)
    rw = x["rewards"] if reward_clip is None else rorc.clip_rewards(x["rewards"], reward_clip)
    total = torch.zeros((), dtype=F64)
    vs_all, pg_all, dl = np.zeros((T + 1, B)), np.zeros((T, B)), None
    lp_all, ent_all, kl_all = np.zeros((T, B)), np.zeros((T, B)), np.zeros((T, B))
    for b in range(B):
        L = int(x["lens"][b])
        if L == 0:
            vs_all[0, b] = float(x["v"][0, b])
            continue
        pis, mus, oks = [], [], []
        for s, h in zip(morc.starts(heads), heads):
            ok = legal[:L, b, s:s + h]
            pis.append(torch.distributions.Categorical(logits=z[:L, b, s:s + h].masked_fill(~ok, -torch.inf)))
            mus.append(torch.distributions.Categorical(logits=beh[:L, b, s:s + h].masked_fill(~ok, -torch.inf)))
            oks.append(ok)
        lp = sum(pi.log_prob(act[:L, b, k]) for k, pi in enumerate(pis))
        lpb = sum(mu.log_prob(act[:L, b, k]) for k, mu in enumerate(mus))
        # entropy and KL over the legal entries (0 * -inf at the illegal ones, in the values and in their gradients)
        ent = sum(-(pi.probs * torch.where(ok, pi.logits, 0.0)).sum(-1) for pi, ok in zip(pis, oks))
        kl = sum((mu.probs * torch.where(ok, mu.logits - pi.logits, 0.0)).sum(-1) for mu, pi, ok in zip(mus, pis, oks))
        v = n[:L + 1, b]
        r = torch.tensor(rw[:L, b], dtype=F64)
        disc = (hp.gamma * torch.tensor(1 - x["done"][:L, b].astype(np.int64), dtype=torch.float32)).to(F64)
        with torch.no_grad():
            ratio = torch.exp(lp - lpb)
            rho, c = torch.clamp(ratio, max=hp.rho_bar), torch.clamp(ratio, max=hp.c_bar)
            vt = torch.zeros(L + 1, dtype=F64)
            if mode == "reference":
                delta = rho * (r + hp.gamma * v[1:] - v[:1])
                for i in range(L - 1, -1, -1):
                    vt[i] = delta[i] + disc[i] * c[i] * (vt[i + 1] - v[i + 1])
            else:
                delta = rho * (r + disc * v[1:] - v[:-1])
                for i in range(L - 1, -1, -1):
                    vt[i] = delta[i] + disc[i] * c[i] * vt[i + 1]
            vt = vt + v
            pg = rho * (r + disc * vt[1:] - v[:-1])
        total = total + (hp.v_loss_c * 0.5 * torch.sum((v - vt) ** 2) + hp.policy_loss_c * torch.sum(-lp * pg)
                         - hp.entropy_c * torch.sum(ent)) / batch_size
        vs_all[:L + 1, b], pg_all[:L, b] = vt.numpy(), pg.numpy()
        lp_all[:L, b], ent_all[:L, b], kl_all[:L, b] = lp.detach().numpy(), ent.detach().numpy(), kl.detach().numpy()
    total.backward()
    return dict(vs=vs_all, pg_adv=pg_all, dlogits=z.grad.numpy(), dv=n.grad.numpy(), log_pi=lp_all, entropy=ent_all,
                kl=kl_all, total_loss=total.item())


@pytest.mark.parametrize("reward_clip", [None, "abs_one"])
@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("heads", list(HEADS))
def test_oracle_matches_autograd_on_masked_heads(heads, mode, reward_clip):
    heads = HEADS[heads]
    T, B = 9, 7
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    x = aorc.make_inputs(5, T, B, heads, density=0.5)
    x["rewards"] = (x["rewards"] * 3.0).astype(np.float32)
    got = aorc.vtrace_loss(x["v"], x["cur"], x["beh"], x["idx"], x["legal"], x["rewards"], x["done"], x["lens"], hp,
                           B, heads, mode, reward_clip)
    want = _torch_update(x, hp, B, heads, mode, reward_clip)
    valid = np.arange(T)[:, None] < x["lens"][None, :]
    for k in ("log_pi", "entropy", "kl"):
        np.testing.assert_allclose(np.where(valid, got[k], 0.0), want[k], rtol=0, atol=1e-12, err_msg=k)
    for k in ("vs", "pg_adv", "dlogits", "dv"):
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-12, err_msg=k)
    assert abs(got["total_loss"] - want["total_loss"]) <= 1e-12 * max(1.0, abs(want["total_loss"]))
    # illegal entries: exactly zero gradient
    assert (got["dlogits"][~aorc.normalise(x["legal"], heads)] == 0).all()


@pytest.mark.parametrize("heads", list(HEADS))
def test_full_mask_and_minus_1e30_are_the_unmasked_oracle(heads):
    heads = HEADS[heads]
    T, B = 8, 6
    hp = default_hparams(batch_size=B, max_timesteps=T)
    x = aorc.make_inputs(3, T, B, heads, density=1.0)
    got = aorc.vtrace_loss(x["v"], x["cur"], x["beh"], x["idx"], x["legal"], x["rewards"], x["done"], x["lens"], hp,
                           B, heads)
    want = morc.vtrace_loss(x["v"], x["cur"], x["beh"], x["idx"], x["rewards"], x["done"], x["lens"], hp, B, heads)
    for k in ("vs", "pg_adv", "dlogits", "dv", "scalars", "diag"):
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-12, err_msg=k)
    # a mask = the unmasked oracle with -1e30 at the illegal current and behaviour entries
    x = aorc.make_inputs(4, T, B, heads, density=0.5)
    ill = ~aorc.normalise(x["legal"], heads)
    cur, beh = np.where(ill, -1e30, x["cur"]), np.where(ill, -1e30, x["beh"])
    got = aorc.vtrace_loss(x["v"], x["cur"], x["beh"], x["idx"], x["legal"], x["rewards"], x["done"], x["lens"], hp,
                           B, heads)
    want = morc.vtrace_loss(x["v"], cur, beh, x["idx"], x["rewards"], x["done"], x["lens"], hp, B, heads)
    for k in ("vs", "pg_adv", "dlogits", "dv", "scalars"):
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-12, err_msg=k)


@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_layout_masked_kinds(obs_dtype):
    lib = _cabi.lib()
    T, B, F, frames, code = 7, 33, 6, 2, _cabi.obs_dtype_code(obs_dtype)
    for heads, kind in (((), 0x200), ((3, 3, 2), 0x303), ((2,) * 16, 0x310)):
        N = sum(heads) or 18
        K = len(heads)
        off = (C.c_int64 * 6)()
        tot = C.c_int64()
        assert lib.impala_batch_layout_act(T, B, F, frames, N, code, kind, off, C.byref(tot)) == 0
        assert 0 <= off[3] - off[2] - T * B * (K + 1 if K else 2) * 4 < 256  # one more int32 column
        dist = "multi_discrete" if K else "categorical"
        assert (list(off), tot.value) == tuple(
            (list(o), t) for o, t in [_cabi.batch_layout(T, B, F * frames, N, obs_dtype, frames, dist, heads, True)])[0]
        from torched_impala_b200.ring import _layout

        assert _layout(T, B, F * frames, N, obs_dtype, frames, dist, heads, True) == (list(off), tot.value)
    bad = (C.c_int64 * 6)()
    for kind, N in ((0x201, 4), (0x200, 33), (0x200 | 0x100, 4), (0x205, 4), (0x400, 4)):
        assert lib.impala_batch_layout_act(T, B, F, frames, N, code, kind, bad, C.byref(C.c_int64())) == -1
    assert _cabi.act_kind_code("categorical", (), True) == 0x200
    assert _cabi.act_kind_code("multi_discrete", (3, 3, 2), True) == 0x303


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


@pytest.mark.parametrize("bad", [dict(action_mask=True, action_dist="gaussian", A=4), dict(action_mask=1),
                                 dict(action_mask="yes"), dict(action_mask=True, A=40)])
def test_options_refuse_bad_masks_before_cuda(monkeypatch, bad):
    from torched_impala_b200.engine import LearnerEngine, LearnerOptions
    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpPolicy, MlpValueFn

    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    A = bad.get("A", 8)
    kw = {k: v for k, v in bad.items() if k != "A"}
    msgs = []
    with pytest.raises(ValueError) as e:
        LearnerOptions(**kw).check(8, 4, A, 8, 8)
    msgs.append(str(e.value))
    with pytest.raises(ValueError) as e:
        LearnerEngine(5, 8, 4, A, 8, 8, hp, **kw)
    msgs.append(str(e.value))
    if A <= 32 and kw.get("action_dist") != "gaussian":
        with pytest.raises(ValueError) as e:
            Learner(0, hp, MlpPolicy(4, A, 8), MlpValueFn(4, 8), None, None, **kw)
        msgs.append(str(e.value))
    assert len(set(msgs)) == 1, msgs
    # good values go on to the device checks
    for kw in (dict(action_mask=True), dict(action_mask=True, action_dist="multi_discrete", action_heads=(3, 3, 2))):
        with pytest.raises(AssertionError):
            LearnerEngine(5, 8, 4, 8, 8, 8, hp, **kw)


def test_options_carry_the_mask():
    from torched_impala_b200.engine import LearnerOptions, engine_from_cfg
    import torched_impala_b200.engine as engine

    o = LearnerOptions(action_mask=True)
    assert o.action_mask is True and o.check(8, 4, 8, 8, 8).act_kind == 0x200
    assert o == LearnerOptions(action_mask=True) and o != LearnerOptions()
    assert "action_mask" not in {f.name for f in dataclasses.fields(o)} and LearnerOptions().action_mask is False
    md = LearnerOptions(action_dist="multi_discrete", action_heads=(3, 3, 2), action_mask=True)
    assert md.check(8, 4, 8, 8, 8).act_kind == 0x303

    calls = []

    class Rec:
        def __init__(self, *a, **k):
            calls.append(k)

    hp = default_hparams(batch_size=8, max_timesteps=5)
    cfg = dict(T=5, B=8, O=4, A=8, H_pi=8, H_v=8, mode="reference", hp=dict(hp._asdict()),
               **dataclasses.asdict(LearnerOptions()))
    orig = engine.LearnerEngine
    try:
        engine.LearnerEngine = Rec
        engine_from_cfg(json.loads(json.dumps(dict(cfg, action_mask=True))), 1, "cpu")
        engine_from_cfg(json.loads(json.dumps(dict(cfg, action_mask=False))), 1, "cpu")
        engine_from_cfg(json.loads(json.dumps(cfg)), 1, "cpu")
    finally:
        engine.LearnerEngine = orig
    assert calls[0]["action_mask"] is True and "action_mask" not in calls[1] and "action_mask" not in calls[2]


def test_make_masked_batch():
    T, B, O = 6, 40, 5
    for heads, A in (((), 8), ((3, 3, 2), 8)):
        b = synth.make_masked_batch(3, T, B, O, A, heads, density=0.4, ragged=True)
        K = len(heads) or 1
        assert b["actions"].shape == (T, B, K + 1) and b["actions"].dtype == np.int32
        legal = b["legal"]
        pad = np.arange(T)[:, None] >= b["lens"][None, :]
        assert (b["actions"][pad] == 0).all() and not legal[pad].any()
        words = b["actions"][..., -1].view(np.uint32)
        assert np.array_equal(words, synth.legal_words(legal).view(np.uint32))
        hs = heads or (A,)
        for k, (s, n) in enumerate(zip(morc.starts(hs), hs)):
            h = legal[~pad][:, s:s + n]
            assert h.any(-1).all()  # at least one legal entry per head
            a = b["actions"][~pad][:, k]
            assert h[np.arange(len(a)), a].all()  # the taken actions are legal
        assert (legal[~pad].sum(-1) == len(hs)).any()  # some single-legal steps
        ill = ~legal & ~pad[..., None]
        assert not np.isfinite(b["beh_logits"][ill]).all() or (np.abs(b["beh_logits"][ill]) >= 1e30).all()
        again = synth.make_masked_batch(3, T, B, O, A, heads, density=0.4, ragged=True)
        assert all(np.array_equal(b[k], again[k], equal_nan=b[k].dtype.kind == "f") for k in b)


@pytest.fixture(scope="module")
def sass():
    return (_sass_kernels("vtrace_mask_kernel"), _sass_kernels("vtrace_md_mask_kernel"),
            _sass_kernels("vtrace_lane_kernel"), _sass_kernels("vtrace_md_kernel"))


def test_mask_instantiations(sass):
    cat, md, _, _ = sass
    # template arguments: AP, S, MAXT, MINB, VEC, DIAG, POPART, RCLIP - every shape the launcher picks
    assert len(cat) == 60 and {k[:3] for k in cat} == {(2, 2, 512), (4, 2, 512), (8, 2, 512), (16, 1, 512),
                                                       (32, 1, 320)}
    assert len(md) == 60 and {k[:3] for k in md} == {(2, 2, 512), (4, 2, 512), (8, 2, 512), (16, 1, 512),
                                                     (32, 1, 256)}


def test_mask_kernels_spill_only_where_their_twin_does(sass):
    cat, md, lane, mdk = sass
    for kernels, twins, lane_twin in ((cat, lane, True), (md, mdk, False)):
        for k, ops in kernels.items():
            ap, s, _, _, vec, diag, popart, rclip = k
            if lane_twin:  # vtrace_lane_kernel<AP, S, MAXT, MINB, WITH_LOSS, VEC, DIAG, POPART[, RCLIP]>
                twin = next(o for t, o in twins.items() if t[0] == ap and t[1] == s and t[4] == 1 and t[5] == vec
                            and t[6] == diag and t[7] == popart and (t[8] if len(t) > 8 else 0) == rclip)
            else:
                twin = next(o for t, o in twins.items() if t[0] == ap and t[1] == s and t[4:] == k[4:])
            if not (twin["LDL"] or twin["STL"]):
                assert not (ops["LDL"] or ops["STL"]), (k, ops["LDL"], ops["STL"])


def _traj(T=6, A=8, heads=(), seed=0):
    b = synth.make_masked_batch(seed, T, 2, 3, A, heads, density=0.5)
    b["lens"][:] = T
    return synth.to_trajectories(b)[0], b


@pytest.mark.parametrize("heads", [(), (3, 3, 2)])
@pytest.mark.parametrize("case", ["missing", "width", "values", "empty", "illegal"])
def test_put_and_put_block_refuse_bad_masks(heads, case):
    from torched_impala_b200.ring import RingQueue

    T, A, B = 6, 8, 4
    kw = dict(action_dist="multi_discrete", action_heads=heads) if heads else {}
    q = RingQueue(T, B, 3, A, slabs=2, action_mask=True, **kw)
    try:
        tr, b = _traj(T, A, heads)
        good = [m.clone() for m in tr.action_mask]
        a0 = [int(x) for x in np.asarray(tr.a[2]).reshape(-1)]
        m = good[2].clone()
        if case == "missing":
            tr.action_mask, match = None, "action_mask"
        elif case == "width":
            tr.action_mask[2], match = torch.ones(A + 1, dtype=torch.bool), "step 2 action_mask has shape"
        elif case == "values":
            m = m.to(torch.int64)
            m[0] = 2
            tr.action_mask[2], match = m, "step 2 .*not 0 / 1"
        elif case == "empty":
            m[:] = False
            tr.action_mask[2], match = m, "step 2 head 0 has no legal action"
        else:
            m[a0[0]] = False
            if not m[:(heads or (A,))[0]].any():
                m[(a0[0] + 1) % (heads or (A,))[0]] = True
            tr.action_mask[2], match = m, "step 2 head 0 action .* is illegal"
        with pytest.raises(ValueError, match=match):
            q.put(tr, timeout=1)
        assert int(q._control()["ticket"][0]) == 0  # no column taken
        # put_block: the same masks as a (T, n, N) block
        n = 2
        blk = synth.make_masked_batch(1, T, n, 3, A, heads, density=0.5)
        blk["lens"][:] = T
        mask = blk.pop("legal").copy()
        blk["actions"] = blk["actions"][..., :-1] if heads else blk["actions"][..., 0]
        blk["action_mask"] = mask
        bad = dict(blk)
        if case == "missing":
            del bad["action_mask"]
        elif case == "width":
            bad["action_mask"] = np.ones((T, n, A + 1), bool)
        elif case == "values":
            mm = mask.astype(np.int8)
            mm[2, 1, 0] = 3
            bad["action_mask"] = mm
        elif case == "empty":
            mm = mask.copy()
            mm[2, 1, :(heads or (A,))[0]] = False
            bad["action_mask"] = mm
        else:
            mm = mask.copy()
            a = int(np.asarray(blk["actions"]).reshape(T, n, -1)[2, 1, 0])
            mm[2, 1, a] = False
            mm[2, 1, (a + 1) % (heads or (A,))[0]] = True
            bad["action_mask"] = mm
        with pytest.raises(ValueError, match="action_mask" if case in ("missing", "width") else "column 1 step 2"):
            q.put_block(bad, timeout=1)
        assert int(q._control()["ticket"][0]) == 0
        # the good trajectory and block go in, legal words last
        tr.action_mask = good
        q.put(tr, timeout=1)
        v = q.views(0)
        assert np.array_equal(v["actions"][:T, 0, -1], synth.legal_words(torch.stack(good).numpy()))
        q.put(_traj(T, A, heads, 1)[0], timeout=1)
        q.put_block(blk, timeout=1)
        assert np.array_equal(v["actions"][:, 2:4, -1], synth.legal_words(mask))
    finally:
        q.close()


def test_select_action_masks():
    from torched_impala_b200.models import MlpPolicy, MultiDiscreteMlpPolicy

    torch.manual_seed(0)
    pol = MlpPolicy(6, 5, 16).eval()
    obs = torch.randn(6, dtype=torch.float64)
    mask = torch.tensor([0, 1, 0, 1, 0], dtype=torch.bool)
    seen = {int(pol.select_action(obs, action_mask=mask)[0]) for _ in range(300)}
    assert seen <= {1, 3} and seen
    a, z = pol.select_action(obs, deterministic=True, action_mask=mask)
    assert int(a) == [1, 3][int(z[[1, 3]].argmax())] and torch.isfinite(z).all()
    md = MultiDiscreteMlpPolicy(6, (3, 3, 2), 16).eval()
    m = torch.tensor([1, 0, 0, 0, 1, 1, 0, 1], dtype=torch.bool)
    for _ in range(100):
        a, z = md.select_action(obs, action_mask=m)
        assert int(a[0]) == 0 and int(a[1]) in (1, 2) and int(a[2]) == 1
    assert torch.equal(md.select_action(obs, deterministic=True)[1], z)
