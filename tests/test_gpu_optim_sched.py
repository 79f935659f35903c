"""GPU: impala_clip_optim / impala_gather_clip_optim - RMSprop and learning-rate tables - from the kernel up to the
engine and the forked Learner.

  * Adam under a constant table equals impala_clip_adam bit for bit (the same template body);
  * RMSprop against a float64 step from the kernel's own float32 state (`rms_ref`, per-entry bounds in the
    manner of `adam_ref`), and over 200 steps against a float64 run;
  * schedules against torch + LambdaLR, past the table's end, and at a rate of 0;
  * the gather variant on W simulated ranks (tests/test_gpu_optim_exchange.py's harness), every producer
    enqueued before any consumer;
  * one captured graph replayed across the table's end;
  * the engine against the float64 oracle (tests/optim_oracle.py) on the golden batches, with bounds derived from
    the gradient's error bound (tests/mlp_bounds.py);
  * a forked Learner behind a RingQueue, and two GPUs (peer push and NCCL) where there are two."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import optim_oracle as oorc
from conftest import PKEYS, Golden
from mlp_bounds import MlpBound
from oracle import impala_oracle as orc
from oracle.check import _flat_oracle_grad
from test_gpu_optim_exchange import (B1, B2, EPS, FUSED, SIZES, STANDALONE, TIMEOUT_S, Net, Ranks, _largest_route_size,
                                     _same_bits, adam_ref, assert_step, contribution, random_inputs)
from torched_impala_b200 import _cabi, ops
from torched_impala_b200.engine import LearnerEngine

pytestmark = pytest.mark.gpu

ADAM, RMSPROP = _cabi.OPT_ADAM, _cabi.OPT_RMSPROP
F32 = np.float32


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    torch.cuda.set_device(0)
    return _cabi.lib()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _table(values):
    return torch.tensor(np.asarray(values, F32), device="cuda")


def _f32(x):
    return float(F32(x))


# ------------------------------------------------------------------------------------------- float64 step
def rms_ref(p, m, v, g, n_policy, max_norm, lr, alpha, momentum, eps):
    """One float64 clip + RMSprop step from the kernel's float32 state (p, m = momentum buffer, v = square_avg),
    gradient g (float64), with the float32 hyperparameters the kernel receives.  Per-entry bounds: v as Adam's
    (8e-7 of its terms); the direction d = g / (sqrt(v) + eps) within 1.2e-6 of itself (float32 g, coefficient,
    product, half of v's bound, root, sum, quotient); m 4e-7 of its terms plus d's bound, and m exactly unchanged
    at momentum 0; p four float32 ulps plus lr times the step's bound and 4e-7 of the step."""
    alpha, momentum, eps, lr = (_f32(x) for x in (alpha, momentum, eps, lr))
    p, m, v = (np.asarray(a, np.float64) for a in (p, m, v))
    norms, coefs = [], []
    for lo, hi in ((0, n_policy), (n_policy, len(g))):
        c, nrm = orc.clip_coef([g[lo:hi]], max_norm)
        norms.append(nrm)
        coefs.append(c)
    gc = g * np.where(np.arange(len(g)) < n_policy, coefs[0], coefs[1])
    va, vb = alpha * v, (1.0 - alpha) * gc * gc
    v2 = va + vb
    d = gc / (np.sqrt(v2) + eps)
    tol_d = 1.2e-6 * np.abs(d)
    if momentum > 0:
        ma = momentum * m
        m2 = ma + d
        tol_m = 4e-7 * (np.abs(ma) + np.abs(d)) + tol_d + 1e-38
        step, tol_step = m2, tol_m
    else:
        m2, tol_m = m.copy(), np.zeros_like(m)
        step, tol_step = d, tol_d
    p2 = p - lr * step
    tol_p = 4 * np.spacing(np.abs(p2).astype(F32)).astype(np.float64) + lr * (tol_step + 4e-7 * np.abs(step))
    return dict(p=p2, m=m2, v=v2, norms=norms, tol_p=tol_p, tol_m=tol_m, tol_v=8e-7 * v2 + 1e-38, d=d)


class Opt:
    """impala_clip_optim on one state (params, m, v, state) with a device learning-rate table."""

    def __init__(self, p0, n_policy, table, rule=RMSPROP, h0=0.99, h1=0.0, eps=0.01):
        self.p, self.m, self.v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
        self.state = torch.zeros(3, dtype=torch.int64, device="cuda")
        self.n_policy, self.table, self.rule, self.h = n_policy, _table(table), rule, (h0, h1, eps)

    def host(self):
        return dict(p=self.p.cpu().numpy(), m=self.m.cpu().numpy(), v=self.v.cpu().numpy(),
                    t=int(self.state[0].item()))

    def lr(self, t):
        return float(self.table[min(t, self.table.numel() - 1)].item())

    def step(self, g, max_norm):
        norms = ops.clip_optim(self.p, g, self.m, self.v, self.state, self.n_policy, max_norm, self.table,
                               "rmsprop" if self.rule == RMSPROP else "adam", *self.h)
        torch.cuda.synchronize()
        return dict(p=self.p.cpu().numpy(), m=self.m.cpu().numpy(), v=self.v.cpu().numpy(),
                    norms=norms.cpu().numpy().tolist())

    def checked_step(self, g, max_norm, what):
        b = self.host()
        lr = self.lr(b["t"])
        if self.rule == RMSPROP:
            ref = rms_ref(b["p"], b["m"], b["v"], g, self.n_policy, max_norm, lr, *self.h)
        else:
            ref = adam_ref(b["p"], b["m"], b["v"], g, b["t"], self.n_policy, max_norm, lr)
        got = self.step(torch.from_numpy(g).cuda(), max_norm)
        assert_step(got, ref, what)
        return got, ref, b


# ------------------------------------------------------------------ 1. Adam under a table == impala_clip_adam
@pytest.mark.parametrize("n_total", SIZES)
def test_adam_table_equals_scalar_bit_for_bit(lib, n_total):
    n = _largest_route_size() if n_total == "largest" else n_total
    rng = np.random.default_rng(n + 1)
    lr = _f32(0.95 * 1e-3)
    table = _table([lr] * 3)
    for n_policy in sorted({0, 1, min(n, 17), n - 1, n}):
        p0 = torch.from_numpy(rng.standard_normal(n).astype(F32)).cuda()
        a = [p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0), torch.zeros(3, dtype=torch.int64, device="cuda")]
        b = [t.clone() for t in a]
        for it in range(5):
            g = torch.from_numpy(rng.standard_normal(n) * (1.0, 1e-3, 30.0, 0.1, 1.0)[it]).cuda()
            max_norm = (0.3, 10.0, 1.0, 1e30, 2.0)[it]
            na = ops.clip_adam(a[0], g, *a[1:], n_policy, max_norm, lr, B1, B2, EPS)
            nb = ops.clip_optim(b[0], g, *b[1:], n_policy, max_norm, table, "adam", B1, B2, EPS)
            torch.cuda.synchronize()
            for name, x, y in zip(("params", "m", "v", "state", "norms"), a + [na], b + [nb]):
                assert _same_bits(x, y), (n, n_policy, it, name)
        assert int(b[3][0].item()) == 5


# ------------------------------------------------------------------------- 2. RMSprop against float64 torch
@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("n_total", SIZES)
def test_rmsprop_sizes_and_groups(lib, n_total, momentum):
    n = _largest_route_size() if n_total == "largest" else n_total
    rng = np.random.default_rng(n + 7)
    for n_policy in sorted({0, 1, min(n, 17), n - 1, n}):
        opt = Opt(torch.from_numpy(rng.standard_normal(n).astype(F32)).cuda(), n_policy, [0.05, 0.02], h1=momentum)
        for it, (scale, max_norm) in enumerate(((1.0, 0.3), (1e-3, 10.0), (2.0, 1e30))):
            opt.checked_step(rng.standard_normal(n) * scale, max_norm, (n, n_policy, it))
        assert opt.state.cpu().tolist() == [3, 0, 0]  # RMSprop counts steps in state[0] only
        if momentum == 0:
            assert not opt.m.any()  # the momentum buffer is never written


@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("regime", ["below", "far_above", "zero_gradient", "one_zero_group"])
def test_rmsprop_clip_regimes(lib, regime, momentum):
    n, n_policy, max_norm = 20000, 9000, 1.0
    rng = np.random.default_rng(2)
    opt = Opt(torch.from_numpy(rng.standard_normal(n).astype(F32)).cuda(), n_policy, [0.01], h1=momentum)
    opt.checked_step(rng.standard_normal(n) * 0.01, max_norm, "warm-up")  # nonzero square_avg and buffer
    g = rng.standard_normal(n) * {"below": 1e-3, "far_above": 1e3}.get(regime, 1.0)
    if regime == "zero_gradient":
        g[:] = 0.0
    if regime == "one_zero_group":
        g[:n_policy] = 0.0
    got, ref, before = opt.checked_step(g, max_norm, regime)
    if regime == "below":
        assert max(ref["norms"]) + 1e-6 < max_norm
    if regime == "far_above":
        assert min(ref["norms"]) > 100 * max_norm
    if regime in ("zero_gradient", "one_zero_group"):
        z = slice(0, n if regime == "zero_gradient" else n_policy)
        # square_avg decays, params move by the momentum buffer only (not at all without momentum)
        np.testing.assert_array_equal(got["v"][z], (F32(0.99) * before["v"][z]).astype(F32))
        if momentum == 0:
            np.testing.assert_array_equal(got["p"][z].view(np.int32), before["p"][z].view(np.int32))
        assert got["norms"][0] == 0.0


@pytest.mark.parametrize("momentum", [0.0, 0.9])
def test_rmsprop_long_run_bounded_drift(lib, momentum):
    """200 steps against an independent float64 run of the same gradients (torch.optim.RMSprop, clip per group):
    the drift stays within the sum of the per-step bounds plus one float32 rounding of p per step."""
    n, n_policy, steps, max_norm, lr, eps = 5000, 1234, 200, 1.0, 0.01, 0.01
    gen = torch.Generator().manual_seed(3)
    grads = torch.randn(steps, n, dtype=torch.float64, generator=gen) * torch.tensor(
        [(3.0, 0.01, 0.3)[s % 3] for s in range(steps)], dtype=torch.float64)[:, None]
    p0 = torch.randn(n, generator=gen).to(torch.float32)
    opt = Opt(p0.cuda(), n_policy, [lr], h1=momentum, eps=eps)
    tp = [p0[:n_policy].double().requires_grad_(), p0[n_policy:].double().requires_grad_()]
    ref = torch.optim.RMSprop(tp, lr=_f32(lr), alpha=_f32(0.99), eps=_f32(eps), momentum=_f32(momentum),
                              foreach=False)
    budget = np.zeros(n)
    for s in range(steps):
        g = grads[s].numpy()
        _, r, _ = opt.checked_step(g, max_norm, s)
        budget += r["tol_p"] + np.spacing(np.abs(r["p"]).astype(F32)).astype(np.float64)
        tp[0].grad, tp[1].grad = grads[s][:n_policy].clone(), grads[s][n_policy:].clone()
        for t in tp:
            torch.nn.utils.clip_grad_norm_([t], max_norm)
        ref.step()
    want = torch.cat([t.detach() for t in tp]).numpy()
    drift = np.abs(opt.p.cpu().numpy() - want)
    # the float64 run starts from the same float32 values; its alpha / eps / momentum are the kernel's float32
    # values, so what remains is float32 rounding, fed back through the state: allow 4x the summed bounds
    assert (drift <= 4 * budget).all(), float((drift / budget).max())
    assert float(drift.max()) < 1e-3 * lr * steps


# ------------------------------------------------------------------------------------------ 3. schedules
def _linear(e, n=10):
    return 1.0 - e / n


@pytest.mark.parametrize("rule,momentum", [(RMSPROP, 0.0), (RMSPROP, 0.9), (ADAM, None)])
def test_linear_schedule_against_lambda_lr(lib, rule, momentum):
    """lr * (1 - e / 10) over 10 updates, then 4 more past the table's end (the last entry repeats): every step
    against the float64 step at that rate, and the end against torch.optim + LambdaLR run on the same gradients
    with the schedule extended the same way."""
    n, n_policy, max_norm, lr, steps = 3000, 1000, 1.0, 0.02, 14
    rng = np.random.default_rng(10)
    table = [lr * _linear(e) for e in range(10)]
    p0 = rng.standard_normal(n).astype(F32)
    if rule == RMSPROP:
        opt = Opt(torch.from_numpy(p0).cuda(), n_policy, table, RMSPROP, 0.99, momentum, 0.01)
    else:
        opt = Opt(torch.from_numpy(p0).cuda(), n_policy, table, ADAM, B1, B2, EPS)
    tp = [torch.tensor(p0[:n_policy], dtype=torch.float64, requires_grad=True),
          torch.tensor(p0[n_policy:], dtype=torch.float64, requires_grad=True)]
    to = (torch.optim.RMSprop(tp, lr=lr, alpha=_f32(0.99), eps=_f32(0.01), momentum=_f32(momentum), foreach=False)
          if rule == RMSPROP else torch.optim.Adam(tp, lr=lr, betas=(B1, B2), eps=_f32(EPS), foreach=False))
    sched = torch.optim.lr_scheduler.LambdaLR(to, lambda e: _f32(lr * _linear(min(e, 9))) / lr)
    for s in range(steps):
        g = rng.standard_normal(n) * 0.5
        assert opt.lr(s) == _f32(table[min(s, 9)])
        opt.checked_step(g, max_norm, s)
        tp[0].grad, tp[1].grad = torch.from_numpy(g[:n_policy].copy()), torch.from_numpy(g[n_policy:].copy())
        for t in tp:
            torch.nn.utils.clip_grad_norm_([t], max_norm)
        to.step()
        sched.step()
    want = torch.cat([t.detach() for t in tp]).numpy()
    assert np.abs(opt.p.cpu().numpy() - want).max() < 2e-5 * lr * steps + 1e-6


@pytest.mark.parametrize("rule", [RMSPROP, ADAM])
def test_zero_rate_leaves_params_and_moves_moments(lib, rule):
    """A rate of 0 from update 2 on (and past the table's end): params keep their bits, the moments advance as in
    torch (m, v for Adam; square_avg and the momentum buffer for RMSprop)."""
    n, n_policy = 5000, 2000
    rng = np.random.default_rng(11)
    h = (0.99, 0.9, 0.01) if rule == RMSPROP else (B1, B2, EPS)
    opt = Opt(torch.from_numpy(rng.standard_normal(n).astype(F32)).cuda(), n_policy, [0.01, 0.0], rule, *h)
    opt.checked_step(rng.standard_normal(n), 1.0, "first")
    for s in range(3):
        before = opt.host()
        got, _, _ = opt.checked_step(rng.standard_normal(n), 1.0, ("zero rate", s))
        assert np.array_equal(got["p"].view(np.int32), before["p"].view(np.int32)), s
        assert not np.array_equal(got["v"], before["v"]) and not np.array_equal(got["m"], before["m"]), s
    assert int(opt.state[0].item()) == 4


# --------------------------------------------------------------------------------- 4. the gather variant
def consume_optim(lib, R, r, max_norm, table, rule, h):
    _cabi.check(lib.impala_gather_clip_optim(
        _p(R.params[r]), _p(R.reduced[r]), _p(R.gather[r]), _p(R.seq[r]), R.slot, R.buf, R.W, R.n_extra, _p(R.m[r]),
        _p(R.v[r]), _p(R.state[r]), R.n_policy, R.n, float(max_norm), _p(table), table.numel(), rule, *h,
        _p(R.norms[r]), _p(R.err[r]), TIMEOUT_S, _st()), "impala_gather_clip_optim")


def gather_step(lib, R, net, inputs, fused, max_norm, table, rule, h):
    """Every producer, a check that the stores are complete, then every consumer: the rank-ordered sum on every
    rank, replicas bit-identical, and rank 0 bit-equal to impala_clip_optim on the sum with a copy of its state."""
    W = R.W
    comms = []
    for r in range(W):
        comms.append(contribution(lib, net, R.params[r], inputs[r], R.n_extra))
        if fused:
            R.push_fused(lib, r, net, inputs[r])
        else:
            R.push(lib, r, comms[r])
    torch.cuda.synchronize()
    step = int(R.seq[0].item()) + 1
    tags = R.words(0)[step & 1, :, : R.n + R.n_extra, 1]
    assert (tags == step).all(), "a producer store is missing: the consumer would wait"
    shadow = [t.clone() for t in (R.params[0], R.m[0], R.v[0], R.state[0])]
    for r in range(W):
        consume_optim(lib, R, r, max_norm, table, rule, h)
    torch.cuda.synchronize()
    R.assert_no_error()
    s = np.zeros(R.n + R.n_extra)
    for c in comms:
        s = s + c.cpu().numpy()
    for r in range(W):
        assert np.array_equal(R.reduced[r].cpu().numpy().view(np.uint64), s.view(np.uint64)), r
        assert int(R.seq[r].item()) == step
    for name in ("params", "m", "v", "state", "norms"):
        for r in range(1, W):
            assert _same_bits(getattr(R, name)[r], getattr(R, name)[0]), (name, r)
    norms = torch.empty(2, dtype=torch.float64, device="cuda")
    _cabi.check(lib.impala_clip_optim(_p(shadow[0]), _p(R.reduced[0][: R.n].clone()), _p(shadow[1]), _p(shadow[2]),
                                      _p(shadow[3]), R.n_policy, R.n, float(max_norm), _p(table), table.numel(), rule,
                                      *h, _p(norms), _st()), "impala_clip_optim")
    torch.cuda.synchronize()
    for name, got, want in zip(("params", "m", "v", "state"), (R.params[0], R.m[0], R.v[0], R.state[0]), shadow):
        assert _same_bits(got, want), name
    assert _same_bits(R.norms[0], norms)


@pytest.mark.parametrize("rule", [RMSPROP, ADAM])
@pytest.mark.parametrize("producer", ["fused", "standalone"])
@pytest.mark.parametrize("W", [1, 3, 8])
def test_gather_clip_optim_ranks(lib, W, producer, rule):
    net = Net(*(FUSED[0] if producer == "fused" else STANDALONE[0]))
    n_extra = 4
    R = Ranks(W, net.n_total, n_extra, net.n_pi, net.init_params(W + 20))
    h = (0.99, 0.9, 0.01) if rule == RMSPROP else (B1, B2, EPS)
    table = _table([1e-3 * (1 - e / 4) for e in range(4)])
    rng = np.random.default_rng(W)
    for it in range(5):  # both parities, across the table's end
        inputs = [random_inputs(lib, net, rng, n_extra) for _ in range(W)]
        gather_step(lib, R, net, inputs, producer == "fused", (0.05, 1e3, 1.0, 1.0, 1.0)[it], table, rule, h)
    assert R.state[0].cpu().tolist()[0] == 5


# ------------------------------------------------------------------------ 5. one graph for every update
@pytest.mark.parametrize("rule", [RMSPROP, ADAM])
def test_one_graph_serves_every_step(lib, rule):
    """The launch captured once and replayed 12 times across the end of an 8-entry table of distinct rates: each
    replay is bit-equal to an eager call with a one-entry table holding the entry that replay must have read."""
    n, n_policy = 14144, 6144
    rng = np.random.default_rng(5)
    h = (0.99, 0.9, 0.01) if rule == RMSPROP else (B1, B2, EPS)
    table = _table([1e-3 * (1.0 + e) for e in range(8)])
    p0 = torch.from_numpy(rng.standard_normal(n).astype(F32)).cuda()
    G = [p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0), torch.zeros(3, dtype=torch.int64, device="cuda")]
    E = [t.clone() for t in G]
    grad, norms = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(2, dtype=torch.float64, device="cuda")
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream, capture_error_mode="thread_local"):
            _cabi.check(lib.impala_clip_optim(*(_p(t) for t in G[:1]), _p(grad), *(_p(t) for t in G[1:]), n_policy, n,
                                              1.0, _p(table), 8, rule, *h, _p(norms), _st()), "impala_clip_optim")
    for k in range(12):
        g = torch.from_numpy(rng.standard_normal(n)).cuda()
        grad.copy_(g)
        graph.replay()
        torch.cuda.synchronize()
        one = table[min(k, 7): min(k, 7) + 1].clone()
        ne = torch.empty(2, dtype=torch.float64, device="cuda")
        _cabi.check(lib.impala_clip_optim(_p(E[0]), _p(g), _p(E[1]), _p(E[2]), _p(E[3]), n_policy, n, 1.0, _p(one), 1,
                                          rule, *h, _p(ne), _st()), "impala_clip_optim")
        torch.cuda.synchronize()
        for name, a, b in zip(("params", "m", "v", "state"), G, E):
            assert _same_bits(a, b), (k, name)
        assert _same_bits(norms, ne), k
    assert int(G[3][0].item()) == 12


# --------------------------------------------------------------------------- 6. the engine and the oracle
def _flat_bounds(eng, batch, params):
    """Per-entry error bound of the engine's raw gradient in the flat layout: the MLP backward's bound from the
    rows, dlogits and dv the engine used (ReLU-tie allowance included), plus 5e-5 of the largest entry for the
    float32 V-trace / loss gradients feeding it (test_gpu_wide_shapes.check_grad_end_to_end)."""
    obs = np.asarray(batch["obs"], np.float64)
    O = obs.shape[2]
    e = np.zeros(eng.n_total)
    dz = {"policy": eng.dlogits.reshape(eng.M_pi, eng.A), "value_fn": eng.dv.reshape(eng.M_vf, 1)}
    x = {"policy": obs[:-1].reshape(-1, O), "value_fn": obs.reshape(-1, O)}
    bounds = {g: MlpBound(x[g], params[g], dz[g]) for g in ("policy", "value_fn")}
    for grp, key, off, shp in eng._segments():
        t = bounds[grp].e_grad[PKEYS.index(key)].cpu().numpy().reshape(-1)
        e[off:off + t.size] = t
    return e


def _rms_tol_from_grad(ref, g, e_g, before, n_policy, max_norm, lr, alpha, eps):
    """How far the float64 RMSprop step may move for a gradient error of at most e_g per entry: |d/dg g / (sqrt(
    alpha v + (1 - alpha) g^2) + eps)| <= 1 / (sqrt(alpha v) + eps), and the clip coefficient's own change."""
    lr, alpha, eps = _f32(lr), _f32(alpha), _f32(eps)
    avg_lo = np.sqrt(alpha * np.asarray(before["v"], np.float64)) + eps
    tol = np.zeros(len(g))
    for lo, hi in ((0, n_policy), (n_policy, len(g))):
        c, nrm = orc.clip_coef([g[lo:hi]], max_norm)
        dn = float(np.sqrt((e_g[lo:hi] ** 2).sum()))
        dc = 0.0 if nrm + 1e-6 - dn > max_norm else max_norm * dn / max(nrm + 1e-6 - dn, 1e-300) ** 2
        tol[lo:hi] = lr * (c * e_g[lo:hi] + dc * (np.abs(g[lo:hi]) + e_g[lo:hi])) / avg_lo[lo:hi]
    return tol


def _engine(g, hp, **kw):
    c = g.case
    eng = LearnerEngine(c["T"], c["B"], c["O"], c["A"], c["H_pi"], c["H_v"], hp, **kw)
    eng.load_state(g.init_params())
    return eng


@pytest.mark.parametrize("name", ["c3_small_fixed", "c3_small_ragged"])
def test_engine_rmsprop_schedule_against_oracle(lib, name):
    """LearnerEngine(optimizer="rmsprop", eps=0.01, linear schedule): three updates (golden batches 0, 1, 0).
    Every update against (a) the float64 step on the engine's own gradient from its own state, (b) the step on
    the ORACLE's gradient with bounds from the gradient's error bound, and the three updates against the oracle
    run from the same initial parameters within the sum of (b)'s bounds."""
    g = Golden(name)
    hp = g.hp._replace(max_updates=4)
    lam = lambda e: 1.0 - e / 4  # noqa: E731
    eng = _engine(g, hp, optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01), lr_lambda=lam)
    ref = oorc.BatchedLearner(g.init_params(), hp, "rmsprop", dict(eps=0.01), lam)
    budget = np.zeros(eng.n_total)
    for u, bu in enumerate((0, 1, 0)):
        batch = g.batch(bu)
        params = eng.state()
        before = dict(p=eng.params.cpu().numpy(), m=eng.adam_m.cpu().numpy(), v=eng.adam_v.cpu().numpy())
        eng.fill_host(batch, u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        eng.synchronize()
        assert eng.lr_of(u + 1) == _f32(hp.lr * lam(min(u, 3)))
        got = dict(p=eng.params.cpu().numpy(), m=eng.adam_m.cpu().numpy(), v=eng.adam_v.cpu().numpy(),
                   norms=eng.norms.cpu().numpy().tolist())
        g_eng = eng.comm[: eng.n_total].cpu().numpy()
        own = rms_ref(before["p"], before["m"], before["v"], g_eng, eng.n_pi, hp.max_norm, eng.lr_of(u + 1), 0.99, 0.0,
                      0.01)
        assert_step(got, own, (name, u, "own gradient"))
        out = orc.BatchedLearner(params, hp).forward_backward(batch, batch_size=eng.global_batch)
        g_or = _flat_oracle_grad(eng, out)
        e_g = _flat_bounds(eng, batch, params) + 5e-5 * np.abs(g_or).max()
        assert (np.abs(g_eng - g_or) <= e_g).all(), (name, u, "gradient outside its bound")
        oracle_step = rms_ref(before["p"], before["m"], before["v"], g_or, eng.n_pi, hp.max_norm, eng.lr_of(u + 1),
                              0.99, 0.0, 0.01)
        tol = _rms_tol_from_grad(oracle_step, g_or, e_g, before, eng.n_pi, hp.max_norm, eng.lr_of(u + 1), 0.99, 0.01)
        err = np.abs(got["p"] - oracle_step["p"])
        assert (err <= tol + oracle_step["tol_p"]).all(), (name, u, float((err / (tol + oracle_step["tol_p"])).max()))
        budget += tol + oracle_step["tol_p"]
        ref.update(batch)
    want = ref.state()
    got_state = eng.state()
    for grp, key, off, shp in eng._segments():
        w = np.asarray(want[grp][key]).reshape(-1)
        d = np.abs(got_state[grp][key].numpy().reshape(-1) - w)
        # three steps' bounds, the first two also fed through the next gradients: 4x
        assert (d <= 4 * budget[off:off + w.size] + 1e-7).all(), (name, grp, key, float(d.max()))


@pytest.mark.parametrize("name", ["c3_small_fixed", "c3_small_ragged"])
def test_engine_adam_schedule(lib, name):
    """Adam under a table: a constant 0.95 schedule gives the default engine's bits (impala_clip_adam), and a
    decaying one matches the float64 Adam step on the engine's own gradient at every update's rate."""
    g = Golden(name)
    hp = g.hp._replace(max_updates=4)
    plain = _engine(g, hp)
    const = _engine(g, hp, lr_lambda=lambda e: 0.95)
    decay = _engine(g, hp, lr_lambda=lambda e: 0.95 * (1.0 - e / 4))
    assert plain.lr_table is None and const.lr_table.numel() == 4
    for u, bu in enumerate((0, 1, 0)):
        before = dict(p=decay.params.cpu().numpy(), m=decay.adam_m.cpu().numpy(), v=decay.adam_v.cpu().numpy())
        for eng in (plain, const, decay):
            eng.fill_host(g.batch(bu), u % 2)
            eng.ingest(u % 2)
            eng.step(u % 2)
            eng.synchronize()
        for name_, t in (("params", "params"), ("m", "adam_m"), ("v", "adam_v"), ("state", "adam_step")):
            assert _same_bits(getattr(plain, t), getattr(const, t)), (u, name_)
        got = dict(p=decay.params.cpu().numpy(), m=decay.adam_m.cpu().numpy(), v=decay.adam_v.cpu().numpy(),
                   norms=decay.norms.cpu().numpy().tolist())
        ref = adam_ref(before["p"], before["m"], before["v"], decay.comm[: decay.n_total].cpu().numpy(), u,
                       decay.n_pi, hp.max_norm, decay.lr_of(u + 1))
        assert_step(got, ref, (name, u))
        assert decay.launches_per_step == plain.launches_per_step


# ------------------------------------------------------------------------------- 7. the forked Learner
def test_forked_learner_rmsprop_schedule(lib, tmp_path):
    """Forked Learner(optimizer="rmsprop", lr_lambda=...) behind a RingQueue (tests/optim_learner_process_check.py):
    its weights after the golden updates equal an engine run of the same configuration on the same batches, and the
    oracle within the bounds of test_engine_rmsprop_schedule_against_oracle's kind; the logged
    optim/lr values are hp.lr * lambda(n - 1)."""
    script = os.path.join(os.path.dirname(__file__), "optim_learner_process_check.py")
    out = tmp_path / "weights.npz"
    res = subprocess.run([sys.executable, script, str(tmp_path / "logs"), str(out)], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "OPTIM_LEARNER_OK" in res.stdout
    w = np.load(out)
    g = Golden("c1_cartpole_ragged")
    hp = g.hp._replace(max_updates=g.updates)
    lam = lambda e: 1.0 - e / g.updates  # noqa: E731 - the script's schedule
    eng = _engine(g, hp, optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01, momentum=0.5), lr_lambda=lam)
    ref = oorc.BatchedLearner(g.init_params(), hp, "rmsprop", dict(eps=0.01, momentum=0.5), lam)
    for u in range(g.updates):
        eng.fill_host(g.batch(u), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        ref.update(g.batch(u))
    st, want = eng.state(), ref.state()
    for grp in ("policy", "value_fn"):
        for k in PKEYS:
            # the engine run fed the same batches: the same kernels on the same values (a few float32 ulps allow for
            # a different column packing of the ring's slabs)
            assert np.abs(w[f"{grp}/{k}"] - st[grp][k].numpy()).max() <= 2e-7, (grp, k)
            # oracle: three steps of at most lr * 10 each (first RMSprop steps are ~lr / sqrt(1 - alpha)); float32
            # rounding is 1e-6 of a step
            assert np.abs(w[f"{grp}/{k}"] - want[grp][k]).max() < 1e-4 * hp.lr * 10 * g.updates + 1e-6, (grp, k)


# ------------------------------------------------------------------------------------------- 8. two GPUs
@pytest.mark.parametrize("allreduce", ["peer", "peer-standalone", "nccl"])
def test_two_ranks_rmsprop_schedule(lib, allreduce):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs (data-parallel path)")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_optim_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240,
                         env=dict(os.environ, IMPALA_ALLREDUCE=allreduce.split("-")[0],
                                  IMPALA_PUSH_FUSED="0" if allreduce == "peer-standalone" else "1"))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_OPTIM_OK" in res.stdout
