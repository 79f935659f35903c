"""GPU: PopArt value normalization - impala_vtrace_loss_popart and impala_clip_optim_popart against the float64
statement in tests/popart_oracle.py, bit-identity with the entry points they extend, and the engine (launch
count, exact scale invariance, the oracle over several updates)."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import popart_oracle as porc
from conftest import PKEYS
from oracle import impala_oracle as orc
from test_gpu_diagnostics import _launch_shapes
from test_gpu_optim_exchange import TIMEOUT_S, Ranks
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


def _close(got, want, what, scale_tol=2e-5):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    tol = scale_tol * max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= tol, (what, err, tol)


def _vt_inputs(T, B, A, S, cluster, ragged, seed):
    b = synth.make_batch(T + A + S + seed, T, B, 3, A, ragged=ragged)
    rng = np.random.default_rng(T * A + S + cluster + seed)
    logits = (b["beh_logits"] + 0.5 * rng.standard_normal((T, B, A))).astype(np.float32)
    n = rng.standard_normal((T + 1, B), dtype=np.float32)
    return b, logits, n


STATS = [(0.0, 1.0), (0.3, 1e-2), (-7.5, 1e3), (2.0, 0.5)]


@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("A,S,cluster", _launch_shapes())
def test_vtrace_popart_matches_oracle(ops, monkeypatch, A, S, cluster, mode):
    if S:
        monkeypatch.setenv("IMPALA_VTRACE_S", str(S))
    monkeypatch.setenv("IMPALA_VTRACE_CLUSTER", str(cluster))
    T, B = 20, 77
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9, gamma=0.97)
    b, logits, n = _vt_inputs(T, B, A, S, cluster, True, 0)
    args = (dev(logits), dev(b["beh_logits"]), dev(b["actions"]), dev(b["rewards"]), dev(b["done"]),
            dev(b["lens"]), dev(n), hp, 1.0 / B)
    for mu, sigma in STATS:
        st = ops.popart_stats(mu, sigma * sigma + mu * mu)
        st[2] = sigma  # exactly the sigma under test
        res = ops.vtrace_loss_popart(*args, st, mode=mode)
        want = porc.vtrace_popart(n, mu, sigma, logits, b, hp, B, mode)
        # reward-unit outputs carry float32 rounding of sigma n + mu; normalized ones are divided by sigma
        vscale = max(1.0, abs(mu) + 4 * sigma)
        _close(res["vs"].cpu(), want["vs"], ("vs", mu, sigma), 2e-5 * vscale)
        nscale = vscale / sigma
        _close(res["pg_adv"].cpu(), want["pg_adv"], ("pg_adv", mu, sigma), 2e-5 * nscale)
        _close(res["dv"].cpu(), want["dv"], ("dv", mu, sigma), 2e-5 * nscale / B)
        _close(res["dlogits"].cpu(), want["dlogits"], ("dlogits", mu, sigma), 2e-5 * nscale / B)
        sc = res["scalars"].cpu().tolist()
        for i, k in enumerate(("value_fn_loss", "policy_loss", "policy_entropy")):
            assert abs(sc[i] - want[k]) <= 1e-4 * max(1.0, abs(want[k])) * (nscale if i < 2 else 1.0), (k, sc[i], want[k])
        d = res["diag"].cpu().tolist()
        assert d[0] == want["n"]
        assert abs(d[5] - want["s1"]) <= 1e-5 * vscale * want["n"], (d[5], want["s1"])
        assert abs(d[6] - want["s2"]) <= 1e-5 * vscale * vscale * want["n"], (d[6], want["s2"])


@pytest.mark.parametrize("A,S,cluster", _launch_shapes())
def test_vtrace_popart_identity_is_diag(ops, monkeypatch, A, S, cluster):
    """mu = 0, sigma = 1: every output bit-identical to impala_vtrace_loss_diag."""
    if S:
        monkeypatch.setenv("IMPALA_VTRACE_S", str(S))
    monkeypatch.setenv("IMPALA_VTRACE_CLUSTER", str(cluster))
    for T, mode in ((20, "reference"), (100, "paper")):
        B = 77
        hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9, gamma=0.97)
        b, logits, n = _vt_inputs(T, B, A, S, cluster, True, 1)
        args = (dev(logits), dev(b["beh_logits"]), dev(b["actions"]), dev(b["rewards"]), dev(b["done"]),
                dev(b["lens"]), dev(n), hp, 1.0 / B)
        pop = ops.vtrace_loss_popart(*args, ops.popart_stats(0.0, 1.0), mode=mode)
        diag = ops.vtrace_loss_diag(*args, mode=mode)
        for k in ("vs", "pg_adv", "dlogits", "dv", "scalars", "diag"):
            assert torch.equal(pop[k], diag[k]), (k, T, mode)


def _optim_case(A, H_v, O, seed):
    """A parameter vector [policy | value net] in the engine's layout (_cabi.param_layout) with a gradient, room for
    the 12 extras, and the offsets of the value head's W2 and b2."""
    rng = np.random.default_rng(seed)
    n_pi = _cabi.param_layout(O, H_v, A)[1]
    offs, n_vf = _cabi.param_layout(O, H_v, 1)
    n_total = n_pi + n_vf
    p = (rng.standard_normal(n_total) * 0.1).astype(np.float32)
    g = np.concatenate([rng.standard_normal(n_total) * 0.05, np.zeros(12)])
    return p, g, n_pi, n_total, n_pi + offs[2], n_pi + offs[3]


def _value(ops, flat, n_pi, x, O, H):
    return ops.mlp_forward(x, flat[n_pi:], O, H, 1).reshape(-1).double()


# the largest parameter vector the route table takes (O = 1024, H = 256, A = 18) and the c4 / c5 nets
OPT_SHAPES = [(4, 256, 24), (4, 512, 64), (18, 256, 1024)]


@pytest.mark.parametrize("rule,h", [("adam", (0.9, 0.999, 1e-8)), ("rmsprop", (0.99, 0.9, 0.01))])
@pytest.mark.parametrize("A,H_v,O", OPT_SHAPES)
def test_clip_optim_popart(ops, rule, h, A, H_v, O):
    p0, g, n_pi, n_total, w2, b2 = _optim_case(A, H_v, O, H_v + O)
    x = torch.randn(333, O, device="cuda")
    table = torch.tensor([3e-4, 2e-4, 1e-4], dtype=torch.float32, device="cuda")
    beta = np.float32(0.05)
    mu, nu = 0.7, 2.5
    bufs = {k: [torch.from_numpy(p0.copy()).cuda(), torch.zeros(n_total, device="cuda"),
                torch.zeros(n_total, device="cuda"), torch.zeros(3, dtype=torch.int64, device="cuda")]
            for k in ("plain", "pop")}
    st = ops.popart_stats(mu, nu)
    rng = np.random.default_rng(7)
    for step in range(4):
        gg = g.copy()
        gg[:n_total] *= rng.uniform(0.5, 40.0)  # below and far above max_norm
        n = 0.0 if step == 2 else float(rng.integers(100, 5000))
        gg[n_total + 4:n_total + 12] = [n, 0.0, 0.0, 0.0, 0.0, n * rng.normal(3.0, 1.0), n * rng.uniform(10, 30), 0.0]
        grad = dev(gg)
        P, M, V, S_ = bufs["plain"]
        ops.clip_optim(P, grad, M, V, S_, n_pi, 0.5, table, rule, *h)
        before = st.cpu().tolist()
        Q, M2, V2, S2 = bufs["pop"]
        ops.clip_optim_popart(Q, grad, M2, V2, S2, n_pi, 0.5, table, st, n_total + 4, w2, H_v, b2, beta, rule, *h)
        torch.cuda.synchronize()
        head = np.zeros(n_total, bool)
        head[w2:w2 + H_v] = True
        head[b2] = True
        q, pl = Q.cpu().numpy(), P.cpu().numpy()
        assert np.array_equal(q[~head], pl[~head]), step
        for a_, b_ in ((M2, bufs["plain"][1]), (V2, bufs["plain"][2]), (S2, bufs["plain"][3])):
            assert torch.equal(a_, b_), step
        mu1, nu1, sg1 = porc.stats_update(before[0], before[1], gg[n_total + 4], gg[n_total + 9], gg[n_total + 10],
                                          float(beta))
        got = st.cpu().tolist()
        assert np.allclose(got[:3], [mu1, nu1, sg1], rtol=1e-13, atol=0), (got, mu1, nu1, sg1)
        assert got[3] == before[0] and got[4] == before[2]
        if n == 0.0:
            assert got[:3] == before[:3]
        # the head: the plain update's value, rescaled; output preservation sigma' head' + mu' = sigma head + mu
        sg0 = before[2]
        want_w2 = pl[w2:w2 + H_v].astype(np.float64) * sg0 / sg1
        want_b2 = (sg0 * float(pl[b2]) + before[0] - mu1) / sg1
        assert np.all(np.abs(q[w2:w2 + H_v] - want_w2) <= 2 ** -23 * np.abs(want_w2) + 1e-30)
        assert abs(q[b2] - want_b2) <= 2 ** -23 * abs(want_b2) + 1e-30
        # output preservation through the value forward: the rescaled head under the new statistics against the
        # head before the rescale (the plain update) under the old ones, to float32 rounding of the outputs
        v_new = got[2] * _value(ops, Q, n_pi, x, O, H_v) + got[0]
        v_old = before[2] * _value(ops, P, n_pi, x, O, H_v) + before[0]
        tol = 2e-5 * max(float(v_old.abs().max()), abs(before[0]), 1e-3 * before[2])
        assert float((v_new - v_old).abs().max()) <= tol, (step, float((v_new - v_old).abs().max()), tol)
        # keep the two runs on the same parameters for the next step
        P.copy_(Q)


ENGINE = {"small": (20, 64, 8, 4, 64), "c4": (20, 1024, 24, 4, 256), "ram4": (20, 256, 512, 18, 256)}


def _engines(shape, **kw):
    T, B, O, A, H = ENGINE[shape]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    return (T, B, O, A, H, hp), [LearnerEngine(T, B, O, A, H, H, hp, popart=on, **kw) for on in (True, False)]


ENGINE_CASES = {  # shape, engine arguments
    "small": ("small", {}),
    "c4": ("c4", {}),
    "small-rmsprop": ("small", dict(optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01), lr_lambda=lambda e: 1 - e / 8)),
    "small-replay": ("small", dict(replay_slabs=2, replay_columns=24)),
    "ram4-u8-frames4": ("ram4", dict(obs_dtype="uint8", frames=4)),
}


def _training_batch(eng, slot):
    """The B-column batch the engine trained on in `slot` (composed from the store with replay), dense obs."""
    eng.synchronize()
    d = {k: v.cpu().numpy() for k, v in eng.d_views[slot].items()}
    if eng.frames > 1:
        d = synth.stack_frames(d, eng.frames)
    return d


@pytest.mark.parametrize("case", list(ENGINE_CASES))
def test_engine_launches_and_oracle(case):
    """Several updates against the float64 PopArt oracle fed the very batches the engine trained on: statistics,
    losses, the policy and the folded value function; the launch count equals the engine without PopArt."""
    shape, kw = ENGINE_CASES[case]
    T, B, O, A, H = ENGINE[shape]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9, max_updates=8)
    on, off = (LearnerEngine(T, B, O, A, H, H, hp, popart=p_, popart_beta=0.1, **kw) for p_ in (True, False))
    params = synth.init_params(3, O, A, H)
    for e in (on, off):
        e.load_state(params)
    okw = {k: kw[k] for k in ("optimizer_kwargs", "lr_lambda") if k in kw}
    ref = porc.BatchedLearner(params, hp, kw.get("optimizer", "adam"), beta=float(np.float32(0.1)), **okw)
    Bf = B - kw.get("replay_columns", 0)
    kind = "bytes" if kw.get("obs_dtype") == "uint8" else "normal"
    n_up = 4
    for u in range(n_up):
        bt = synth.make_batch(40 + u, T, Bf, O, A, ragged=(u % 2 == 1), obs_kind=kind, frames=kw.get("frames", 1))
        for e in (on, off):
            e.fill_host(bt, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
        sc = on.read_scalars()
        off.read_scalars()
        want = ref.update(_training_batch(on, u % 2))
        assert on.launches_per_step == off.launches_per_step
        st = on.popart_stats()
        assert abs(st["mu"] - ref.mu) <= 1e-5 * max(1.0, abs(ref.mu)), (u, st, ref.mu)
        assert abs(st["nu"] - ref.nu) <= 1e-5 * max(1.0, abs(ref.nu)), (u, st, ref.nu)
        assert sc["popart_mu"] == st["mu"] and sc["popart_sigma"] == st["sigma"]
        assert abs(sc["value_fn_loss"] - want["value_fn_loss"]) <= 1e-4 * max(1.0, abs(want["value_fn_loss"]))
        assert abs(sc["policy_loss"] - want["policy_loss"]) <= 1e-4 * max(1.0, abs(want["policy_loss"]))
    # the update moves every entry by at most ~lr per step whatever the gradient, so a handful of entries whose
    # gradient is at float32 noise level may differ by that much; everything else agrees to a tiny fraction of it
    # (RMSprop's first steps are up to lr / sqrt(1 - alpha) = 10 lr)
    step = hp.lr * (10.0 if kw.get("optimizer") == "rmsprop" else 1.0)
    got = on.normalized_state()
    for grp, mine in (("policy", ref.pi), ("value_fn", ref.vf)):
        for k, w in zip(PKEYS, mine):
            err = np.abs(got[grp][k].numpy() - w)
            assert err.max() <= 3 * step * n_up, (grp, k, err.max())
            assert np.median(err) <= 1e-3 * step, (grp, k, np.median(err))
    folded = porc.fold(ref.vf, ref.mu, ref.sigma)
    for k, w in zip(PKEYS, folded):
        _close(on.state()["value_fn"][k].numpy(), w, k, 5e-3)


@pytest.mark.parametrize("kw", [dict(), dict(optimizer="rmsprop", optimizer_kwargs=dict(alpha=0.99, eps=0.01)),
                                dict(replay_slabs=2, replay_columns=16)])
def test_engine_scale_invariance_exact(kw):
    """Rewards x 2^10 from (mu, nu) = (0, 2^20) with the folded value function x 2^10: after 10 updates the policy
    and the normalized value function equal the run at rewards x 1 from (0, 1), bit for bit."""
    T, B, O, A, H = ENGINE["small"]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    params = synth.init_params(4, O, A, H)
    big = {"policy": dict(params["policy"]), "value_fn": dict(params["value_fn"])}
    big["value_fn"][PKEYS[2]] = np.asarray(params["value_fn"][PKEYS[2]], np.float64) * 1024.0
    big["value_fn"][PKEYS[3]] = np.asarray(params["value_fn"][PKEYS[3]], np.float64) * 1024.0
    Bf = B - kw.get("replay_columns", 0)
    e1 = LearnerEngine(T, B, O, A, H, H, hp, popart=True, popart_beta=0.25, **kw)
    e2 = LearnerEngine(T, B, O, A, H, H, hp, popart=True, popart_beta=0.25, **kw)
    e1.load_state(params)
    e2.load_state(big, {"mu": 0.0, "nu": 2.0 ** 20})
    assert torch.equal(e1.params, e2.params)
    for u in range(10):
        bt = synth.make_batch(60 + u, T, Bf, O, A, ragged=True)
        bt2 = dict(bt, rewards=(bt["rewards"] * np.float32(1024.0)).astype(np.float32))
        for e, b_ in ((e1, bt), (e2, bt2)):
            e.fill_host(b_, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
    e1.synchronize(), e2.synchronize()
    s1, s2 = e1.popart_stats(), e2.popart_stats()
    assert s2["mu"] == 1024.0 * s1["mu"] and s2["sigma"] == 1024.0 * s1["sigma"], (s1, s2)
    assert s1["sigma"] != 1.0  # the statistics moved
    assert torch.equal(e1.params, e2.params)


def test_engine_state_round_trip():
    (T, B, O, A, H, hp), (on, _) = _engines("small", popart_beta=0.2)
    params = synth.init_params(5, O, A, H)
    on.load_state(params)
    for u in range(3):
        on.fill_host(synth.make_batch(80 + u, T, B, O, A, ragged=True), u % 2)
        on.ingest(u % 2)
        on.step(u % 2)
    on.synchronize()
    raw = on.params.clone()
    st, stats = on.state(), on.popart_stats()
    on.load_state(st, {"mu": stats["mu"], "nu": stats["nu"]})
    assert torch.equal(on.params, raw)


# ------------------------------------------------------------------------------------- simulated ranks
def _gather_popart(lib, R, r, max_norm, table, rule, h, stats, w2, H, b2, beta):
    _cabi.check(lib.impala_gather_clip_optim_popart(
        _p(R.params[r]), _p(R.reduced[r]), _p(R.gather[r]), _p(R.seq[r]), R.slot, R.buf, R.W, R.n_extra, _p(R.m[r]),
        _p(R.v[r]), _p(R.state[r]), R.n_policy, R.n, float(max_norm), _p(table), table.numel(), _cabi.OPT_RULES[rule],
        *h, _p(R.norms[r]), _p(R.err[r]), TIMEOUT_S, _p(stats), R.n + 4, w2, H, b2, float(beta), _st()),
        "impala_gather_clip_optim_popart")


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("rule,h", [("adam", (0.9, 0.999, 1e-8)), ("rmsprop", (0.99, 0.9, 0.01))])
@pytest.mark.parametrize("W", [2, 4, 8])
def test_gather_popart_simulated_ranks(ops, W, rule, h):
    """W ranks' gather buffers on one device: W stand-alone producers, then W consumers (every producer enqueued
    before any consumer).  Statistics, parameters and optimizer state are bit-identical on every rank and equal to
    one impala_clip_optim_popart call on the rank-ordered float64 sum of the payloads."""
    lib = _cabi.lib()
    A, H, O = 4, 256, 24
    p0, _, n_pi, n_total, w2, b2 = _optim_case(A, H, O, W)
    R = Ranks(W, n_total, 12, n_pi, torch.from_numpy(p0).cuda())
    stats = [ops.popart_stats(0.4, 3.0) for _ in range(W)]
    one = dict(p=torch.from_numpy(p0).cuda(), m=torch.zeros(n_total, device="cuda"),
               v=torch.zeros(n_total, device="cuda"), state=torch.zeros(3, dtype=torch.int64, device="cuda"),
               stats=ops.popart_stats(0.4, 3.0))
    table = torch.tensor([5e-4, 3e-4], dtype=torch.float32, device="cuda")
    beta = 0.125
    rng = np.random.default_rng(W)
    for step in range(3):
        kept = one["stats"].cpu().tolist()
        payloads = []
        for r in range(W):
            g = np.zeros(n_total + 12)
            g[:n_total] = rng.standard_normal(n_total) * rng.uniform(0.01, 0.5)
            n = 0.0 if step == 1 else float(rng.integers(50, 500))
            g[n_total:n_total + 4] = rng.standard_normal(4)
            g[n_total + 4:] = [n, 0.1, 3.0, 2.0, 0.5, n * rng.normal(2.0, 1.0), n * rng.uniform(5, 9), 0.3]
            payloads.append(torch.from_numpy(g).cuda())
        for r in range(W):  # every producer first
            R.push(lib, r, payloads[r])
        torch.cuda.synchronize()
        for r in range(W):
            _gather_popart(lib, R, r, 0.5, table, rule, h, stats[r], w2, H, b2, beta)
        total = torch.zeros(n_total + 12, dtype=torch.float64, device="cuda")
        for g in payloads:  # ((0 + g_0) + g_1) + ...: the consumers' order
            total = total + g
        ops.clip_optim_popart(one["p"], total, one["m"], one["v"], one["state"], n_pi, 0.5, table, one["stats"],
                              n_total + 4, w2, H, b2, beta, rule, *h)
        torch.cuda.synchronize()
        R.assert_no_error()
        for r in range(W):
            assert torch.equal(R.reduced[r], total), (step, r)
            assert torch.equal(stats[r], one["stats"]), (step, r, stats[r].tolist(), one["stats"].tolist())
            for a_, b_ in ((R.params[r], one["p"]), (R.m[r], one["m"]), (R.v[r], one["v"]),
                           (R.state[r], one["state"])):
                assert torch.equal(a_, b_), (step, r)
        if step == 1:  # no valid step on any rank: the statistics stay, the head's rescale is the identity
            assert stats[0][:3].tolist() == kept[:3]
        assert stats[0][3:5].tolist() == [kept[0], kept[2]]  # the (mu, sigma) this update's loss used


def test_entry_points_refuse_bad_arguments(ops):
    """IMPALA_ERR_BAD_ARG before any launch: NULL statistics, beta outside (0, 1], a head outside the value net,
    b2 inside the W2 block, sums outside the gradient / the gathered extras."""
    lib = _cabi.lib()
    _, _, n_pi, n_total, w2, b2 = _optim_case(4, 64, 8, 0)
    H = 64
    f = torch.zeros(n_total, device="cuda")
    g = torch.zeros(n_total + 12, dtype=torch.float64, device="cuda")
    st3 = torch.zeros(3, dtype=torch.int64, device="cuda")
    table = torch.ones(1, device="cuda")
    stats = ops.popart_stats()
    norms = torch.zeros(2, dtype=torch.float64, device="cuda")
    good = dict(popart=_p(stats), sums_at=n_total + 4, w2=w2, w2_len=H, b2=b2, beta=3e-4)
    bad = [dict(popart=None), dict(beta=0.0), dict(beta=-1.0), dict(beta=1.5), dict(beta=float("nan")),
           dict(w2=n_pi - 1), dict(w2_len=0), dict(w2=n_total - H + 1), dict(b2=n_pi - 1), dict(b2=n_total),
           dict(b2=w2 + 3), dict(sums_at=n_total - 1)]

    def clip(**kw):
        a = dict(good, **kw)
        return lib.impala_clip_optim_popart(_p(f), _p(g), _p(f), _p(f), _p(st3), n_pi, n_total, 1.0, _p(table), 1,
                                            _cabi.OPT_ADAM, 0.9, 0.999, 1e-8, _p(norms), a["popart"], a["sums_at"],
                                            a["w2"], a["w2_len"], a["b2"], a["beta"], _st())

    W = 2
    R = Ranks(W, n_total, 12, n_pi, f.clone())

    def gather(**kw):
        a = dict(good, **kw)
        return lib.impala_gather_clip_optim_popart(
            _p(R.params[0]), _p(R.reduced[0]), _p(R.gather[0]), _p(R.seq[0]), R.slot, R.buf, W, R.n_extra, _p(R.m[0]),
            _p(R.v[0]), _p(R.state[0]), n_pi, n_total, 1.0, _p(table), 1, _cabi.OPT_ADAM, 0.9, 0.999, 1e-8,
            _p(norms), _p(R.err[0]), TIMEOUT_S, a["popart"], a["sums_at"], a["w2"], a["w2_len"], a["b2"], a["beta"],
            _st())

    before = lib.impala_launch_count()
    for kw in bad:
        assert clip(**kw) == -1, kw
        assert gather(**kw) == -1, kw
    assert gather(sums_at=n_total + 5) == -1  # the eight sums must be among the gathered extras
    T, B, A = 5, 32, 4
    z = torch.zeros(T, B, A, device="cuda")
    i = torch.zeros(T, B, dtype=torch.int32, device="cuda")
    ws = torch.zeros(int(lib.impala_vtrace_loss_diag_workspace(T, B, A)), dtype=torch.uint8, device="cuda")
    vt = [_p(z), _p(z), _p(i), _p(z), _p(i), _p(i), _p(z), _p(z), _p(z), _p(z), _p(z), _p(norms), _p(g), _p(ws),
          ws.numel(), T, B, A, 0.99, 1.0, 1.0, 0.5, 1.0, 0.01, 1.0 / B, 0]
    assert lib.impala_vtrace_loss_popart(*vt, None, _st()) == -1
    assert lib.impala_vtrace_loss_popart(*vt[:12], None, *vt[13:], _p(stats), _st()) == -1  # NULL diag
    assert lib.impala_launch_count() == before  # nothing was launched


# --------------------------------------------------------------------------------------- forked Learner
def test_forked_learner_popart(tmp_path):
    """Forked Learner(popart=True) behind a RingQueue (tests/popart_learner_process_check.py): its weights equal an
    engine run of the same configuration on the same batches and the oracle; the checkpoint holds the folded value
    function and the "popart" key; popart/mu and popart/sigma are logged; load() of that checkpoint into a new
    Learner resumes with the same normalized weights and statistics."""
    from conftest import Golden

    script = os.path.join(os.path.dirname(__file__), "popart_learner_process_check.py")
    out = tmp_path / "weights.npz"
    res = subprocess.run([sys.executable, script, str(tmp_path / "logs"), str(out)], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "POPART_LEARNER_OK" in res.stdout
    w = np.load(out)
    g = Golden("c1_cartpole_ragged")
    c = g.case
    hp = g.hp._replace(max_updates=g.updates)
    eng = LearnerEngine(c["T"], c["B"], c["O"], c["A"], c["H_pi"], c["H_v"], hp, popart=True, popart_beta=0.2)
    eng.load_state(g.init_params())
    ref = porc.BatchedLearner(g.init_params(), hp, beta=float(np.float32(0.2)))
    for u in range(g.updates):
        eng.fill_host(g.batch(u), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        ref.update(g.batch(u))
    st, norm, stats = eng.state(), eng.normalized_state(), eng.popart_stats()
    assert abs(float(w["mu"]) - stats["mu"]) <= 1e-12 * max(1.0, abs(stats["mu"]))
    assert abs(float(w["nu"]) - stats["nu"]) <= 1e-12 * max(1.0, abs(stats["nu"]))
    assert abs(stats["mu"] - ref.mu) <= 1e-5 * max(1.0, abs(ref.mu))
    want = {"policy": ref.pi, "value_fn": porc.fold(ref.vf, ref.mu, ref.sigma)}
    for grp in ("policy", "value_fn"):
        for k, wk in zip(PKEYS, want[grp]):
            # same kernels on the same values (a few float32 ulps allow for the ring's column packing)
            assert np.abs(w[f"{grp}/{k}"] - st[grp][k].numpy()).max() <= 2e-6 * max(1.0, np.abs(wk).max()), (grp, k)
            # oracle: an entry moves by at most ~lr per update, so that bounds a float32-noise gradient's effect
            bound = 3 * hp.lr * g.updates * (ref.sigma if (grp, k) in (("value_fn", PKEYS[2]), ("value_fn", PKEYS[3]))
                                              else 1.0)
            assert np.abs(w[f"{grp}/{k}"] - wk).max() <= bound + 1e-5 * np.abs(wk).max(), (grp, k)
            # the resumed engine holds the normalized weights the run ended with
            assert np.abs(w[f"resumed/{grp}/{k}"] - norm[grp][k].numpy()).max() <= 2e-6 * max(
                1.0, np.abs(norm[grp][k].numpy()).max()), (grp, k)


# ------------------------------------------------------------------------------------------- two GPUs
@pytest.mark.parametrize("allreduce", ["peer", "peer-standalone", "nccl"])
def test_two_ranks_popart(allreduce):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs (data-parallel path)")
    with socket.socket() as s_:
        s_.bind(("127.0.0.1", 0))
        port = s_.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_popart_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240,
                         env=dict(os.environ, IMPALA_ALLREDUCE=allreduce.split("-")[0],
                                  IMPALA_PUSH_FUSED="0" if allreduce == "peer-standalone" else "1"))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_POPART_OK" in res.stdout
