"""CPU: RMSprop and learning-rate schedules without a device - the argument refusals of impala_clip_optim and
impala_gather_clip_optim (all before any launch), the ptxas report of their four kernels, the float64 oracle
against torch.optim + LambdaLR + clip_grad_norm_, and the host-side checks and tabulation (optim.py) up to the
table a data-parallel worker rank reads."""
import json
import math
import os
import queue
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import optim_oracle as oorc
from oracle import impala_oracle as orc
from test_optim_cpu import BAD_ARG, _buf
from torched_impala_b200 import _cabi, dp
from torched_impala_b200.learner import Learner
from torched_impala_b200.models import MlpPolicy, MlpValueFn
from torched_impala_b200.optim import optim_config, tabulate_lr
from torched_impala_b200.utils import Counter, default_hparams

ADAM, RMSPROP = 0, 1


def _no_device():
    return not torch.cuda.is_available()


# ------------------------------------------------------------------------------------------ C entry points
def _clip_optim(lib, p):
    def rc(params=p, grad=p, m=p, v=p, state=p, n_policy=3, n_total=7, table=p, n_lr=4, rule=RMSPROP, h0=0.99,
           h1=0.0, eps=0.01):
        return lib.impala_clip_optim(params, grad, m, v, state, n_policy, n_total, 1.0, table, n_lr, rule, h0, h1,
                                     eps, None, None)
    return rc


BAD_RULE_ARGS = [dict(table=None), dict(n_lr=0), dict(n_lr=-1), dict(rule=2), dict(rule=-1), dict(eps=-1e-3),
                 dict(eps=float("nan")), dict(rule=ADAM, eps=-1e-8), dict(h0=1.0), dict(h0=-0.1), dict(h0=float("nan")),
                 dict(h1=-0.5), dict(h1=float("nan"))]


def test_clip_optim_refuses_bad_arguments():
    rc = _clip_optim(_cabi.lib(), _buf())
    for name in ("params", "grad", "m", "v", "state"):
        assert rc(**{name: None}) == BAD_ARG, name
    for n_policy, n_total in ((-1, 7), (8, 7), (0, 0), (0, -3)):
        assert rc(n_policy=n_policy, n_total=n_total) == BAD_ARG, (n_policy, n_total)
    for kw in BAD_RULE_ARGS:
        assert rc(**kw) == BAD_ARG, kw


@pytest.mark.skipif(not _no_device(), reason="a device would run the launch")
def test_clip_optim_accepts_edges():
    """Arguments at the edges pass every check and reach the launch (which fails without a GPU)."""
    rc = _clip_optim(_cabi.lib(), _buf())
    for kw in (dict(), dict(h0=0.0), dict(h1=0.9), dict(eps=0.0), dict(n_lr=1), dict(rule=ADAM, h0=0.9, h1=0.999),
               dict(rule=ADAM, h0=2.0, h1=-1.0)):  # Adam's betas are the caller's, as for impala_clip_adam
        assert rc(**kw) not in (BAD_ARG, 0), kw


def test_gather_clip_optim_refuses_bad_arguments():
    lib = _cabi.lib()
    p = _buf()
    n_total, n_extra = 100, 4
    slot = n_total + n_extra

    def rc(params=p, reduced=p, gather=p, seq=p, slot=slot, buf=2 * slot, world=2, n_extra=n_extra, m=p, v=p,
           state=p, n_policy=40, n_total=n_total, table=p, n_lr=4, rule=RMSPROP, h0=0.99, h1=0.0, eps=0.01):
        return lib.impala_gather_clip_optim(params, reduced, gather, seq, slot, buf, world, n_extra, m, v, state,
                                            n_policy, n_total, 10.0, table, n_lr, rule, h0, h1, eps, None, None, 1.0,
                                            None)

    for name in ("params", "reduced", "gather", "seq", "m", "v", "state"):
        assert rc(**{name: None}) == BAD_ARG, name
    for kw in (dict(n_policy=-1), dict(n_policy=n_total + 1), dict(n_total=0, n_policy=0), dict(world=0),
               dict(world=9, buf=9 * slot), dict(n_extra=-1), dict(n_extra=1025, slot=n_total + 1025),
               dict(slot=slot - 1), dict(buf=2 * slot - 1), dict(world=8, buf=8 * slot - 1),
               dict(gather=_buf(offset=8)), dict(gather=_buf(offset=4)), *BAD_RULE_ARGS):
        assert rc(**kw) == BAD_ARG, kw
    if _no_device():
        assert rc() not in (BAD_ARG, 0)


def test_optim_kernels_ptxas_report(tmp_path):
    """Every instantiation of the two templated kernels: at most 64 registers (1024-thread CTAs), no spills, no
    local memory."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.fail("nvcc not found")
    src = os.path.join(os.path.dirname(_cabi.__file__), "csrc", "optim.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", src, "-o", str(tmp_path / "optim.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    blocks = re.split(r"Compiling entry function", res.stderr)[1:]
    seen = []
    for name in ("17clip_optim_kernelINS_8AdamRule", "17clip_optim_kernelINS_11RmspropRule",
                 "24gather_clip_optim_kernelINS_8AdamRule", "24gather_clip_optim_kernelINS_11RmspropRule"):
        mine = [b for b in blocks if name in b.split("'")[1]]
        assert len(mine) == 1, (name, len(mine))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in mine[0], mine[0]
        assert not re.search(r"\d+ bytes lmem", mine[0]) or re.search(r"\b0 bytes lmem", mine[0]), mine[0]
        regs = int(re.search(r"Used (\d+) registers", mine[0]).group(1))
        assert regs <= 64, (name, regs)
        seen.append(regs)
    assert len(seen) == 4


# ------------------------------------------------------------------------------------------------ the oracle
def _torch_run(kind, params0, grads, lr, max_norm, lr_lambda, **kw):
    ts = [torch.tensor(p, dtype=torch.float64, requires_grad=True) for p in params0]
    opt = (torch.optim.RMSprop(ts, lr=lr, foreach=False, **kw) if kind == "rmsprop"
           else torch.optim.Adam(ts, lr=lr, foreach=False))
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda)
    for gs in grads:
        for t, g in zip(ts, gs):
            t.grad = torch.tensor(g, dtype=torch.float64)
        torch.nn.utils.clip_grad_norm_(ts[:2], max_norm)  # learner.py:176-181: one call per network
        torch.nn.utils.clip_grad_norm_(ts[2:], max_norm)
        opt.step()
        sched.step()
    return [t.detach().numpy() for t in ts], opt


@pytest.mark.parametrize("kind,kw", [("rmsprop", dict(momentum=0.0)), ("rmsprop", dict(momentum=0.9)),
                                     ("rmsprop", dict(alpha=0.9, eps=0.01, momentum=0.5)), ("adam", {})])
def test_oracle_matches_torch(kind, kw):
    rng = np.random.default_rng(20)
    shapes = [(5, 3), (5,), (2, 5), (2,)]
    params0 = [rng.standard_normal(s) for s in shapes]
    grads = [[rng.standard_normal(s) * (0.1, 3.0)[step % 2] for s in shapes] for step in range(20)]
    lr, max_norm = 0.01, 1.0
    lam = lambda e: 1.0 - e / 25  # noqa: E731 - the paper's linear decay
    want, _ = _torch_run(kind, params0, grads, lr, max_norm, lam, **kw)
    ps = [p.copy() for p in params0]
    opt = oorc.RMSprop(ps, lr, lr_lambda=lam, **kw) if kind == "rmsprop" else oorc.Adam(ps, lr, lam)
    for gs in grads:
        c0, _ = orc.clip_coef(gs[:2], max_norm)
        c1, _ = orc.clip_coef(gs[2:], max_norm)
        opt.step(ps, [g * c0 for g in gs[:2]] + [g * c1 for g in gs[2:]])
    for got, w in zip(ps, want):
        np.testing.assert_allclose(got, w, rtol=0, atol=1e-14)


def test_oracle_default_is_the_reference_adam():
    rng = np.random.default_rng(1)
    params = {g: {k: rng.standard_normal((3, 2)) for k in orc.PKEYS} for g in ("policy", "value_fn")}
    hp = default_hparams(lr=0.002)
    assert type(oorc.BatchedLearner(params, hp).opt) is orc.Adam
    assert oorc.BatchedLearner(params, hp).opt.lr == orc.BatchedLearner(params, hp).opt.lr
    sched = oorc.BatchedLearner(params, hp, lr_lambda=lambda e: 0.95)
    grads = [rng.standard_normal((3, 2)) for _ in range(8)]
    a, b = orc.BatchedLearner(params, hp), sched
    for _ in range(3):
        a.opt.step(a.pi + a.vf, grads)
        b.opt.step(b.pi + b.vf, grads)
    for x, y in zip(a.pi + a.vf, b.pi + b.vf):
        np.testing.assert_array_equal(x, y)


# ------------------------------------------------------------------------------- host checks, tabulation
def test_default_config_keeps_the_scalar_path():
    hp = default_hparams(lr=0.001, max_updates=50)
    cfg = optim_config(hp)
    assert cfg.is_default and cfg.lr_table is None and cfg.rule == "adam"
    assert cfg.lr_of(1) == cfg.lr_of(10 ** 9) == float(np.float32(0.95 * 0.001))
    r = optim_config(hp, "rmsprop")  # lr_lambda None: the reference's constant 0.95 for either rule
    assert not r.is_default and r.lr_table.tolist() == [np.float32(0.95 * 0.001)]
    assert (r.h0, r.h1, r.eps) == (0.99, 0.0, 1e-8)  # torch's RMSprop defaults
    a = optim_config(hp, lr_lambda=lambda e: 0.5)
    assert a.rule == "adam" and (a.h0, a.h1, a.eps) == (0.9, 0.999, 1e-8) and a.lr_table.size == 50


def test_tabulation_is_lambda_lr():
    hp = default_hparams(lr=0.003, max_updates=7)
    lam = lambda e: 1.0 - e / 7  # noqa: E731
    cfg = optim_config(hp, "rmsprop", dict(eps=0.01), lam)
    want = (0.003 * np.array([1.0 - e / 7 for e in range(7)])).astype(np.float32)
    assert cfg.lr_table.dtype == np.float32 and np.array_equal(cfg.lr_table, want)
    assert [cfg.lr_of(n) for n in range(1, 10)] == [float(x) for x in want] + [float(want[-1])] * 2
    assert cfg.lr_of(7) == float(np.float32(0.003 * (1.0 / 7)))  # update n uses lambda(n - 1)
    with pytest.raises(ValueError):
        cfg.lr_of(0)
    # LambdaLR's own rates, update by update
    p = torch.zeros(1, requires_grad=True)
    opt = torch.optim.RMSprop([p], lr=0.003)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lam)
    for n in range(1, 8):
        assert cfg.lr_of(n) == float(np.float32(opt.param_groups[0]["lr"])), n
        opt.step()
        sched.step()
    assert optim_config(default_hparams(max_updates=0), lr_lambda=lam).lr_table.size == 1


@pytest.mark.parametrize("bad,where", [(float("nan"), 3), (-1e-9, 5), (float("inf"), 0), (1e60, 2)])
def test_bad_schedule_names_the_epoch(bad, where):
    hp = default_hparams(lr=1e-3, max_updates=10)
    with pytest.raises(ValueError, match=f"e={where}"):
        optim_config(hp, "rmsprop", lr_lambda=lambda e: bad if e == where else 1.0)
    with pytest.raises(ValueError, match=f"e={where}"):
        optim_config(hp, lr_table=[1e-3 if e != where else bad for e in range(10)])


@pytest.mark.parametrize("optimizer,kw,match", [
    ("sgd", {}, "optimizer"), ("adam", dict(betas=(0.9, 0.99)), "betas"), ("adam", dict(eps=0.1), "eps"),
    ("rmsprop", dict(centered=True), "centered"), ("rmsprop", dict(weight_decay=1e-4), "weight_decay"),
    ("rmsprop", dict(lr=0.1), "lr"), ("rmsprop", dict(foreach=True), "foreach"), ("rmsprop", dict(alpha=1.0), "alpha"),
    ("rmsprop", dict(alpha=-0.1), "alpha"), ("rmsprop", dict(alpha=1 - 1e-10), "alpha"),
    ("rmsprop", dict(eps=-1e-3), "eps"), ("rmsprop", dict(momentum=-0.5), "momentum"),
    ("rmsprop", dict(momentum=float("nan")), "momentum"), ("rmsprop", dict(eps="x"), "eps")])
def test_bad_optimizer_arguments_are_named(optimizer, kw, match):
    with pytest.raises(ValueError, match=match):
        optim_config(default_hparams(), optimizer, kw)


def test_bad_lambda_calls():
    hp = default_hparams(max_updates=3)
    with pytest.raises(ValueError, match="callable"):
        optim_config(hp, lr_lambda=0.5)
    with pytest.raises(ValueError, match="lr_lambda"):
        optim_config(hp, lr_lambda=lambda e: "fast")
    with pytest.raises(ValueError, match="not both"):
        optim_config(hp, lr_lambda=lambda e: 1.0, lr_table=[1.0])
    with pytest.raises(ValueError, match="empty"):
        optim_config(hp, lr_table=[])
    assert optim_config(hp, "rmsprop", dict(centered=False, weight_decay=0)).rule == "rmsprop"  # torch's defaults


def test_tabulate_many_updates():
    t = tabulate_lr(1e-3, lambda e: 1.0 - e / 200000, 200000)
    assert t.size == 200000 and t[0] == np.float32(1e-3) and t[-1] == np.float32(1e-3 / 200000)


def test_worker_sees_the_same_schedule(tmp_path):
    """A data-parallel worker rank rebuilds its engine from the JSON config and the init-state file: the same
    rule, hyperparameters and table as rank 0, whatever the lambda was."""
    hp = default_hparams(batch_size=4, max_timesteps=5, max_updates=40000, log_path=None)
    lam = lambda e: 0.5 ** (e / 1000)  # noqa: E731 - a lambda does not pickle; the table crosses instead
    lrn = Learner(1, hp, MlpPolicy(4, 2, 8), MlpValueFn(4, 8), queue.Queue(), Counter(0), optimizer="rmsprop",
                  optimizer_kwargs=dict(eps=0.01, momentum=0.9), lr_lambda=lam)
    cfg = json.loads(json.dumps(lrn._cfg()))  # what the worker's command line carries
    assert len(json.dumps(lrn._cfg())) < 8192  # the table is not in it
    assert cfg["optimizer"] == "rmsprop" and cfg["optimizer_kwargs"] == dict(eps=0.01, momentum=0.9)
    path = str(tmp_path / "init_state.npz")
    dp.write_init_state(path, lrn._init_state(), lrn.optim.lr_table)
    state, table = dp.read_init_state(path)
    assert set(state) == {"policy", "value_fn"} and set(state["policy"]) == set(orc.PKEYS)
    worker = optim_config(hp, cfg["optimizer"], cfg["optimizer_kwargs"], lr_table=table)
    assert (worker.rule, worker.h0, worker.h1, worker.eps) == (lrn.optim.rule, 0.99, 0.9, 0.01)
    assert np.array_equal(worker.lr_table, lrn.optim.lr_table) and worker.lr_table.size == 40000
    assert all(worker.lr_of(n) == lrn.optim.lr_of(n) for n in (1, 2, 1000, 40000, 40001))
    # the default writes no table, and the worker keeps impala_clip_adam
    plain = Learner(2, hp, MlpPolicy(4, 2, 8), MlpValueFn(4, 8), queue.Queue(), Counter(0))
    dp.write_init_state(path, plain._init_state(), plain.optim.lr_table)
    assert dp.read_init_state(path)[1] is None
    c = json.loads(json.dumps(plain._cfg()))
    assert optim_config(hp, c["optimizer"], c["optimizer_kwargs"], lr_table=None).is_default


def test_learner_refuses_bad_arguments_before_starting():
    hp = default_hparams(batch_size=4, max_timesteps=5, max_updates=10, log_path=None)
    with pytest.raises(ValueError, match="e=2"):
        Learner(1, hp, MlpPolicy(4, 2, 8), MlpValueFn(4, 8), queue.Queue(), Counter(0), optimizer="rmsprop",
                lr_lambda=lambda e: -1.0 if e == 2 else 1.0)
    with pytest.raises(ValueError, match="centered"):
        Learner(1, hp, MlpPolicy(4, 2, 8), MlpValueFn(4, 8), queue.Queue(), Counter(0), optimizer="rmsprop",
                optimizer_kwargs=dict(centered=True))


def test_header_and_bindings_agree():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(_cabi.__file__)), "include", "impala_b200.h")).read()
    assert re.search(r"#define IMPALA_OPT_ADAM 0\b", hdr) and re.search(r"#define IMPALA_OPT_RMSPROP 1\b", hdr)
    assert (_cabi.OPT_ADAM, _cabi.OPT_RMSPROP) == (0, 1)
    for name in ("impala_clip_optim", "impala_gather_clip_optim"):
        assert f"int {name}(" in hdr and name in _cabi.SIGNATURES
    assert len(_cabi.SIGNATURES["impala_clip_optim"][1]) == 16
    assert len(_cabi.SIGNATURES["impala_gather_clip_optim"][1]) == 24
    assert math.isclose(float(np.float32(0.95 * 1e-3)), optim_config(default_hparams(lr=1e-3)).lr_of(1))
