"""CPU: the off-policy diagnostics' oracle against an independent torch restatement, the derived values,
and the host surface of the switch (Learner config, C header / ctypes signatures)."""
import math
import queue

import numpy as np
import pytest
import torch
from torch.distributions import Categorical, kl_divergence

import diagnostics_oracle as dorc
from conftest import ROOT
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.engine import DIAG_NAMES, diagnostic_values
from torched_impala_b200.learner import Learner
from torched_impala_b200.models import MlpPolicy, MlpValueFn
from torched_impala_b200.utils import Counter, default_hparams


def restated(v, vs, cur_logits, beh_logits, actions, lens, rho_bar, c_bar):
    """One trajectory at a time with torch.distributions (float64), as a user would write it."""
    T, B, _ = cur_logits.shape
    s = torch.zeros(8, dtype=torch.float64)
    for b in range(B):
        L = int(min(max(int(lens[b]), 0), T))
        if L == 0:
            continue
        pi = Categorical(logits=torch.as_tensor(cur_logits[:L, b], dtype=torch.float64))
        mu = Categorical(logits=torch.as_tensor(beh_logits[:L, b], dtype=torch.float64))
        a = torch.as_tensor(actions[:L, b], dtype=torch.int64)
        lr = pi.log_prob(a) - mu.log_prob(a)
        ratio = lr.exp()
        vs_b = torch.as_tensor(vs[:L, b], dtype=torch.float64)
        err = vs_b - torch.as_tensor(v[:L, b], dtype=torch.float64)
        s += torch.stack([torch.tensor(float(L), dtype=torch.float64), lr.sum(), (ratio > rho_bar).sum().double(),
                          (ratio > c_bar).sum().double(), kl_divergence(mu, pi).sum(), vs_b.sum(),
                          (vs_b * vs_b).sum(), err.sum()])
    return s.numpy()


def close(got, want, tol=1e-12):
    return np.all(np.abs(np.asarray(got) - np.asarray(want)) <= tol * np.maximum(1.0, np.abs(want)))


def test_oracle_matches_restatement_on_golden(golden):
    hp = golden.hp
    for u in range(golden.updates):
        b = golden.batch(u)
        out = orc.BatchedLearner(golden.init_params() if u == 0 else golden.params_after(u - 1),
                                 hp).forward_backward(b)
        args = (out["v"], out["vs"], out["logits"], b["beh_logits"], b["actions"], b["lens"], hp.rho_bar, hp.c_bar)
        got, want = dorc.diagnostics(*args), restated(*args)
        assert close(got, want), (u, got, want)
        assert got[0] == int(np.clip(b["lens"], 0, out["logits"].shape[0]).sum())


@pytest.mark.parametrize("T,B,A,mode,rho_bar,c_bar", [
    (20, 37, 4, "reference", 1.0, 1.0), (33, 19, 3, "reference", 0.9, 0.8), (7, 64, 18, "paper", 1.0, 0.5),
    (50, 8, 6, "reference", 2.0, 1.0), (5, 5, 2, "paper", 1.0, 1.0), (64, 12, 32, "reference", 1.0, 1.0)])
def test_oracle_matches_restatement_ragged(T, B, A, mode, rho_bar, c_bar):
    b = synth.make_batch(T + B + A, T, B, 3, A, ragged=True)
    rng = np.random.default_rng(T * B + A)
    logits = (2.0 * rng.standard_normal((T, B, A))).astype(np.float32)
    v = rng.standard_normal((T + 1, B)).astype(np.float32)
    vs, _, _ = orc.vtrace(v, logits, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], 0.99,
                          rho_bar, c_bar, mode)
    args = (v, vs, logits, b["beh_logits"], b["actions"], b["lens"], rho_bar, c_bar)
    got = dorc.diagnostics(*args)
    assert close(got, restated(*args))
    assert 0 < got[2] < got[0]  # some ratios are clipped, not all
    # on-policy: the same logits as behaviour -> no log ratio, no KL, nothing clipped at rho_bar = c_bar = 1
    on = dorc.diagnostics(v, vs, logits, logits, b["actions"], b["lens"], 1.0, 1.0)
    assert abs(on[1]) < 1e-12 and abs(on[4]) < 1e-12 and on[2] == 0 and on[3] == 0


def test_sum_err_sq_is_twice_batch_times_value_loss(golden):
    """The derived explained variance uses sum (vs - v)^2 = 2 B value_fn_loss instead of a ninth sum."""
    hp = golden.hp
    for u in range(golden.updates):
        b = golden.batch(u)
        out = orc.BatchedLearner(golden.init_params() if u == 0 else golden.params_after(u - 1),
                                 hp).forward_backward(b)
        T = out["logits"].shape[0]
        valid = np.arange(T)[:, None] < b["lens"][None, :]
        err2 = np.where(valid, (out["vs"][:T] - out["v"][:T]) ** 2, 0.0).sum()
        assert abs(err2 - 2.0 * hp.batch_size * out["value_fn_loss"]) <= 1e-12 * max(1.0, err2)
        s = dorc.diagnostics(out["v"], out["vs"], out["logits"], b["beh_logits"], b["actions"], b["lens"],
                             hp.rho_bar, hp.c_bar)
        d = dorc.derived(s, out["value_fn_loss"], hp.batch_size)
        vs_v, err_v = out["vs"][:T][valid], (out["vs"][:T] - out["v"][:T])[valid]
        if len(vs_v) >= 2 and vs_v.var() > 0:
            assert abs(d["value_explained_variance"] - (1.0 - err_v.var() / vs_v.var())) < 1e-9
        assert d["valid_steps"] == valid.sum()


def test_derived_values_and_nan_cases():
    #       n  log_ratio  n_rho  n_c   kl    vs   vs^2   err
    s = [4.0, -0.4, 1.0, 2.0, 0.2, 2.0, 6.0, 1.0]
    d = dorc.derived(s, value_fn_loss=0.25, batch_size=2)  # sum err^2 = 1
    var_vs, var_err = 6.0 / 4 - 0.25, 1.0 / 4 - 1.0 / 16
    assert d == pytest.approx(dict(valid_steps=4.0, log_ratio_mean=-0.1, rho_clip_fraction=0.25, c_clip_fraction=0.5,
                                   kl_behaviour_current=0.05, value_explained_variance=1.0 - var_err / var_vs))
    one = dorc.derived([1.0, 0.1, 0, 0, 0.0, 1.0, 1.0, 0.0], 0.0, 1)  # n < 2
    assert math.isnan(one["value_explained_variance"]) and one["log_ratio_mean"] == pytest.approx(0.1)
    flat = dorc.derived([3.0, 0.0, 0, 0, 0.0, 6.0, 12.0, 0.0], 0.0, 1)  # Var(vs) = 0
    assert math.isnan(flat["value_explained_variance"])
    empty = dorc.derived([0.0] * 8, 0.0, 1)
    assert all(math.isnan(empty[k]) for k in DIAG_NAMES[:5]) and empty["valid_steps"] == 0
    # the engine's derivation (what the learner logs) is the oracle's
    for sums, vfl, B in ((s, 0.25, 2), ([1.0, 0.1, 0, 0, 0.0, 1.0, 1.0, 0.0], 0.0, 1),
                         ([3.0, 0.0, 0, 0, 0.0, 6.0, 12.0, 0.0], 0.0, 1), ([0.0] * 8, 0.0, 1)):
        got, want = diagnostic_values(sums, vfl, B), dorc.derived(sums, vfl, B)
        assert set(got) == set(DIAG_NAMES) == set(want)
        for k in DIAG_NAMES:
            assert (math.isnan(got[k]) and math.isnan(want[k])) or got[k] == want[k], k


def test_learner_config_carries_the_switch():
    """Every data-parallel rank builds its engine from _cfg(): a rank without the switch would push 4 logged
    values where the others push 12."""
    hp = default_hparams(batch_size=4, max_timesteps=5, log_path=None)
    off = Learner(1, hp, MlpPolicy(4, 2, 8), MlpValueFn(4, 8), queue.Queue(), Counter(0))
    on = Learner(2, hp, MlpPolicy(4, 2, 8), MlpValueFn(4, 8), queue.Queue(), Counter(0), diagnostics=True,
                 devices=["cuda:0", "cuda:1"])
    assert off._cfg()["diagnostics"] is False and on._cfg()["diagnostics"] is True


def test_header_and_signatures_declare_the_diag_entry_points():
    import os
    import re

    hdr = open(os.path.join(ROOT, "include", "impala_b200.h")).read()
    declared = set(re.findall(r"^\s*(?:int64_t|long long|int)\s+(impala_\w+)\s*\(", hdr, flags=re.M))
    for name in ("impala_vtrace_loss_diag_workspace", "impala_vtrace_loss_diag"):
        assert name in declared and name in _cabi.SIGNATURES
    # same arguments as impala_vtrace_loss plus the diag pointer after the scalars
    plain, diag = _cabi.SIGNATURES["impala_vtrace_loss"][1], _cabi.SIGNATURES["impala_vtrace_loss_diag"][1]
    assert diag[:12] == plain[:12] and diag[12] is _cabi._p and diag[13:] == plain[12:]
