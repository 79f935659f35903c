"""CPU: multi-discrete policies - the float64 oracle against torch autograd on per-head
torch.distributions.Categorical, the K = 1 identity with the categorical oracle, the slab layouts, argument checks
before any CUDA work, the C ABI and the local-memory traffic of the multi-discrete kernels' SASS."""
import ctypes as C
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

import multi_discrete_oracle as morc
import reward_clip_oracle as rorc
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi
from torched_impala_b200.utils import default_hparams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _torch_update(x, hp, batch_size, heads, mode, reward_clip, popart):
    """The reference learner's loss (learner.py:104-162), one trajectory at a time, with one Categorical per head and
    autograd for d total / d logits and d total / d v (PopArt: v normalized, targets in reward units)."""
    T, B, N = x["cur"].shape
    mu_p, sig = (0.0, 1.0) if popart is None else popart
    z = torch.tensor(x["cur"], dtype=F64, requires_grad=True)
    n = torch.tensor(x["v"], dtype=F64, requires_grad=True)
    beh = torch.tensor(x["beh"], dtype=F64)
    act = torch.tensor(x["actions"], dtype=torch.int64)
    rw = x["rewards"] if reward_clip is None else rorc.clip_rewards(x["rewards"], reward_clip)
    total = torch.zeros((), dtype=F64)
    sums = dict(value_fn_loss=0.0, policy_loss=0.0, policy_entropy=0.0)
    vs_all, pg_all = np.zeros((T + 1, B)), np.zeros((T, B))
    lp_all, ent_all, kl_all = np.zeros((T, B)), np.zeros((T, B)), np.zeros((T, B))
    st = morc.starts(heads)
    for b in range(B):
        L = int(x["lens"][b])
        if L == 0:  # an empty trajectory: vs = v at step 0, nothing enters the loss (Categorical takes no empty batch)
            vs_all[0, b] = sig * float(x["v"][0, b]) + mu_p
            continue
        pis = [torch.distributions.Categorical(logits=z[:L, b, s:s + h]) for s, h in zip(st, heads)]
        mus = [torch.distributions.Categorical(logits=beh[:L, b, s:s + h]) for s, h in zip(st, heads)]
        lp = sum(pi.log_prob(act[:L, b, k]) for k, pi in enumerate(pis))
        lpb = sum(mu.log_prob(act[:L, b, k]) for k, mu in enumerate(mus))
        ent = sum(pi.entropy() for pi in pis)
        kl = sum(torch.distributions.kl_divergence(mu, pi) for mu, pi in zip(mus, pis))
        v = sig * n[:L + 1, b] + mu_p
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
            pg = rho * (r + disc * vt[1:] - v[:-1]) / sig
        vl = 0.5 * torch.sum(((v - vt) / sig) ** 2)
        pl = torch.sum(-lp * pg)
        pe = torch.sum(ent)
        total = total + (hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * pe) / batch_size
        for k, t in (("value_fn_loss", vl), ("policy_loss", pl), ("policy_entropy", pe)):
            sums[k] += t.item() / batch_size
        vs_all[:L + 1, b], pg_all[:L, b] = vt.numpy(), pg.numpy()
        lp_all[:L, b], ent_all[:L, b], kl_all[:L, b] = lp.detach().numpy(), ent.detach().numpy(), kl.detach().numpy()
    total.backward()
    return dict(sums, vs=vs_all, pg_adv=pg_all, dlogits=z.grad.numpy(), dv=n.grad.numpy(), log_pi=lp_all,
                entropy=ent_all, kl=kl_all, total_loss=total.item())


@pytest.mark.parametrize("popart", [None, (0.4, 2.5)])
@pytest.mark.parametrize("reward_clip", [None, "abs_one", "soft_asymmetric"])
@pytest.mark.parametrize("mode", ["reference", "paper"])
def test_oracle_matches_autograd_on_categorical_heads(mode, reward_clip, popart):
    T, B, heads = 9, 7, (3, 2, 4)
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    x = morc.make_inputs(5, T, B, heads)
    x["rewards"] = (x["rewards"] * 3.0).astype(np.float32)  # past the clip ranges
    got = morc.vtrace_loss(x["v"], x["cur"], x["beh"], x["actions"], x["rewards"], x["done"], x["lens"], hp, B,
                           heads, mode, reward_clip, popart)
    want = _torch_update(x, hp, B, heads, mode, reward_clip, popart)
    valid = np.arange(T)[:, None] < x["lens"][None, :]
    for k in ("log_pi", "entropy", "kl"):
        np.testing.assert_allclose(np.where(valid, got[k], 0.0), want[k], rtol=0, atol=1e-12, err_msg=k)
    for k in ("vs", "pg_adv", "dlogits", "dv"):
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-12, err_msg=k)
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "total_loss"):
        assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), (k, got[k], want[k])
    assert got["diag"][0] == valid.sum() and abs(got["diag"][4] - want["kl"].sum()) <= 1e-12 * max(1, got["diag"][4])


@pytest.mark.parametrize("mode", ["reference", "paper"])
def test_one_head_is_the_categorical_oracle(mode):
    T, B, A = 8, 6, 5
    hp = default_hparams(batch_size=B, max_timesteps=T)
    x = morc.make_inputs(3, T, B, (A,))
    got = morc.vtrace_loss(x["v"], x["cur"], x["beh"], x["actions"], x["rewards"], x["done"], x["lens"], hp, B, (A,),
                           mode)
    a1 = x["actions"][..., 0]
    vs, pg, rho = orc.vtrace(x["v"], x["cur"], x["beh"], a1, x["rewards"], x["done"], x["lens"], hp.gamma, hp.rho_bar,
                             hp.c_bar, mode)
    lo = orc.losses(np.asarray(x["v"], np.float64), vs, x["cur"], a1, pg, x["lens"], hp.v_loss_c, hp.policy_loss_c,
                    hp.entropy_c, B)
    np.testing.assert_allclose(got["vs"], vs, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got["pg_adv"], pg, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got["dlogits"], lo["dlogits"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(got["dv"], lo["dv"], rtol=0, atol=1e-12)
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "total_loss"):
        assert abs(got[k] - lo[k]) <= 1e-12 * max(1.0, abs(lo[k])), k


@pytest.mark.parametrize("frames", [1, 4])
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_layout_act(obs_dtype, frames):
    lib = _cabi.lib()
    T, B, F, code = 7, 33, 6, _cabi.obs_dtype_code(obs_dtype)
    for heads in ((2,), (3, 3, 2), (5, 7, 4), (2,) * 16, (16, 16)):
        N, K = sum(heads), len(heads)
        md = (C.c_int64 * 6)()
        tot = C.c_int64()
        assert lib.impala_batch_layout_act(T, B, F, frames, N, code, 0x100 | K, md, C.byref(tot)) == 0
        cat = (C.c_int64 * 6)()
        tc = C.c_int64()
        assert lib.impala_batch_layout_frames(T, B, F, frames, N, code, cat, C.byref(tc)) == 0
        if K == 1:  # K = 1 is the categorical layout
            assert list(md) == list(cat) and tot.value == tc.value
        sizes = [md[i + 1] - md[i] for i in range(5)] + [tot.value - md[5]]
        assert sizes[1] >= T * B * N * 4 and sizes[2] >= T * B * K * 4 and sizes[2] < T * B * K * 4 + 256
        assert (list(md), tot.value) == (list(_cabi.batch_layout(T, B, F * frames, N, obs_dtype, frames,
                                                                 "multi_discrete", heads)[0]),
                                         _cabi.batch_layout(T, B, F * frames, N, obs_dtype, frames,
                                                            "multi_discrete", heads)[1])
    bad = (C.c_int64 * 6)()
    for kind, N in ((0x100, 4), (0x100 | 17, 40), (0x100 | 3, 5), (0x200 | 1, 4)):  # K = 0, K > 16, N < 2K, unknown
        assert lib.impala_batch_layout_act(T, B, F, frames, N, code, kind, bad, C.byref(C.c_int64())) == -1


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


@pytest.mark.parametrize("bad", [dict(action_heads=(3, 3)), dict(action_heads=(3, 1, 2)), dict(action_heads=()),
                                 dict(action_heads=(2,) * 17, A=34), dict(action_heads=(20, 20), A=40),
                                 dict(action_heads=(3, 2.5)), dict(action_heads=5),
                                 dict(action_dist="categorical", action_heads=(3, 3, 2)),
                                 dict(action_dist="gaussian", action_heads=(4,), A=4)])
def test_engine_refuses_bad_heads_before_cuda(monkeypatch, bad):
    from torched_impala_b200.engine import LearnerEngine, LearnerOptions

    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    A = bad.get("A", 8)
    kw = dict(action_dist=bad.get("action_dist", "multi_discrete"), action_heads=bad["action_heads"])
    with pytest.raises(ValueError):
        LearnerOptions(**kw).check(8, 4, A, 8, 8)
    with pytest.raises(ValueError):
        LearnerEngine(5, 8, 4, A, 8, 8, hp, **kw)
    # good values go on to the device checks
    for heads in ((3, 3, 2), [3, 3, 2], (8,)):
        with pytest.raises(AssertionError):
            LearnerEngine(5, 8, 4, 8, 8, 8, hp, action_dist="multi_discrete", action_heads=heads)
    # shared torso: N + 1 <= 32 outputs
    with pytest.raises(ValueError):
        LearnerEngine(5, 8, 4, 32, 8, 8, hp, action_dist="multi_discrete", action_heads=(16, 16), shared_torso=True)


def test_options_carry_heads():
    import dataclasses

    from torched_impala_b200.engine import LearnerOptions

    o = LearnerOptions(action_dist="multi_discrete", action_heads=[3, 3, 2])
    assert o.action_heads == (3, 3, 2) and o.check(8, 4, 8, 8, 8).act_kind == 0x100 | 3
    assert o == LearnerOptions(action_dist="multi_discrete", action_heads=(3, 3, 2))
    assert o != LearnerOptions(action_dist="multi_discrete", action_heads=(3, 2, 3))
    assert LearnerOptions().action_heads == () and "action_heads" not in {f.name for f in dataclasses.fields(o)}


def test_learner_and_ring_refuse_multi_discrete(monkeypatch):
    """Bad multi-discrete arguments: the Learner refuses heads that do not sum to the policy's outputs and the ring
    heads of a single action or an action count they do not sum to, before any CUDA work."""
    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpValueFn, MultiDiscreteMlpPolicy
    from torched_impala_b200.ring import RingQueue

    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    with pytest.raises(ValueError, match="outputs"):
        Learner(0, hp, MultiDiscreteMlpPolicy(4, (3, 3, 2), 8), MlpValueFn(4, 8), None, None,
                action_dist="multi_discrete", action_heads=(3, 3))
    with pytest.raises(ValueError):
        RingQueue(5, 8, 4, 8, action_dist="multi_discrete")
    with pytest.raises(ValueError, match="outputs"):
        RingQueue(5, 8, 4, 9, action_dist="multi_discrete", action_heads=(3, 3, 2))


def test_policy_module():
    from torched_impala_b200.models import MlpPolicy, MultiDiscreteMlpPolicy

    torch.manual_seed(0)
    heads = (3, 3, 2)
    pol = MultiDiscreteMlpPolicy(6, heads, 16).eval()  # no dropout: one logit vector for every call below
    assert set(pol.state_dict()) == set(MlpPolicy(6, 8, 16).state_dict())
    obs = torch.randn(6, dtype=next(pol.parameters()).dtype)
    a, z = pol.select_action(obs)
    assert a.shape == (3,) and a.dtype == torch.int64 and z.shape == (8,)
    assert all(0 <= int(a[k]) < n for k, n in enumerate(heads))
    a, z = pol.select_action(obs, deterministic=True)
    assert [int(x) for x in a] == [int(z[s:s + n].argmax()) for s, n in zip(morc.starts(heads), heads)]
    counts = np.zeros(3)
    for _ in range(3000):
        counts[int(pol.select_action(obs)[0][0])] += 1
    p = torch.softmax(z[:3].detach(), -1).numpy()
    assert np.abs(counts / 3000 - p).max() < 0.05


def test_make_md_batch():
    from torched_impala_b200 import synth

    heads = (3, 3, 2, 2, 5, 5)
    b = synth.make_md_batch(3, 6, 40, 5, heads, ragged=True)
    assert b["beh_logits"].shape == (6, 40, 20) and b["actions"].shape == (6, 40, 6) and b["actions"].dtype == np.int32
    assert (b["actions"] >= 0).all() and (b["actions"] < np.array(heads)).all()
    pad = np.arange(6)[:, None] >= b["lens"][None, :]
    assert (b["beh_logits"][pad] == 0).all() and (b["actions"][pad] == 0).all()
    again = synth.make_md_batch(3, 6, 40, 5, heads, ragged=True)
    assert all(np.array_equal(b[k], again[k]) for k in b)
    params = synth.init_params(1, 5, 20, 8)
    bp = synth.make_md_batch(3, 6, 40, 5, heads, ragged=True, params=params)
    assert np.array_equal(bp["obs"], b["obs"]) and not np.array_equal(bp["beh_logits"], b["beh_logits"])
    tr = synth.to_trajectories(b)
    L = int(b["lens"][2])
    assert len(tr) == 40 and len(tr[2].a) == L
    if L:
        assert tr[2].a[0].shape == (6,) and tr[2].a[0].dtype == torch.int64 and tr[2].logits[0].shape == (20,)


def test_header_and_signature():
    hdr = open(os.path.join(ROOT, "include", "impala_b200.h")).read()
    assert re.search(r"\bint impala_vtrace_loss_md\(", hdr)
    assert "#define IMPALA_ACT_MULTI_DISCRETE(K) (0x100 | (K))" in hdr
    assert _cabi.ACT_MULTI_DISCRETE == 0x100
    assert _cabi.act_kind_code("multi_discrete", (3, 3, 2)) == 0x103
    sig = _cabi.SIGNATURES["impala_vtrace_loss_md"]
    assert sig[1][:-1] == _cabi.SIGNATURES["impala_vtrace_loss_gauss"][1][:-1] + [C.c_void_p, C.c_int]


def test_library_exports_entry_point():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([nm, "-D", "--defined-only", _cabi.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    assert re.search(r"\bT impala_vtrace_loss_md$", out, re.M)


def _sass_kernels(name):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([exe, "-sass", _cabi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, cur = {}, None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            t = re.search(name + r"I((?:L[ib]\d+E)+)E", m.group(1))
            cur = tuple(int(v) for v in re.findall(r"L[ib](\d+)E", t.group(1))) if t else None
            if cur is not None:
                kernels[cur] = Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and cur is not None:
            kernels[cur][m.group(1)] += 1
    return kernels


@pytest.fixture(scope="module")
def sass():
    return _sass_kernels("vtrace_md_kernel"), _sass_kernels("vtrace_lane_kernel")


def test_md_instantiations(sass):
    md, _ = sass
    # template arguments: AP, S, MAXT, MINB, VEC, DIAG, POPART, RCLIP
    assert len(md) == 60  # AP 2, 4, 8, 16, 32 x VEC x {plain, diag, popart} x reward clip
    assert {k[:3] for k in md} == {(2, 2, 512), (4, 2, 512), (8, 2, 512), (16, 1, 512), (32, 1, 256)}


def test_md_kernels_spill_only_where_their_categorical_twin_does(sass):
    md, cat = sass
    for k, ops in md.items():
        ap, s, _, _, vec, diag, popart, rclip = k
        twin = next(o for t, o in cat.items() if t[0] == ap and t[1] == s and t[4] == 1 and t[5] == vec
                    and t[6] == diag and t[7] == popart and (t[8] if len(t) > 8 else 0) == rclip)
        if not (twin["LDL"] or twin["STL"]):
            assert not (ops["LDL"] or ops["STL"]), (k, ops["LDL"], ops["STL"])
