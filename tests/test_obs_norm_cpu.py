"""CPU: observation normalization (obs_norm) - option checks, the JSON config round trip, and the float64 oracle:
fold and unfold are inverses, the folded network on raw observations is the trained one on normalized rows, Chan's
merge over successive batches gives the statistics of their concatenation, and only valid rows count."""
import dataclasses
import json
import math

import numpy as np
import pytest

import obs_norm_oracle as onorc
from torched_impala_b200.engine import LearnerOptions, check_obs_norm_args, obs_norm_f32

SHAPES = dict(B=16, O=24, A=4, H_pi=32, H_v=32)


@pytest.mark.parametrize("eps", [0.0, -1e-8, math.nan, math.inf, "1e-8", True, None])
def test_eps_must_be_finite_and_positive(eps):
    with pytest.raises(ValueError, match="obs_norm_eps"):
        check_obs_norm_args(True, eps, 24)
    with pytest.raises(ValueError, match="obs_norm_eps"):
        LearnerOptions(obs_norm=True, obs_norm_eps=eps).check(**SHAPES)


@pytest.mark.parametrize("flag", [1, "yes", None])
def test_obs_norm_must_be_bool(flag):
    with pytest.raises(ValueError, match="obs_norm must be a bool"):
        LearnerOptions(obs_norm=flag).check(**SHAPES)


def test_feature_limit():
    LearnerOptions(obs_norm=True).check(16, 1024, 4, 32, 32)
    with pytest.raises(ValueError, match="at most 1024"):
        LearnerOptions(obs_norm=True).check(16, 1025, 4, 32, 32)
    LearnerOptions().check(16, 1025, 4, 32, 32)  # off: no limit of its own


def test_defaults_and_config_round_trip(monkeypatch):
    """Init-only options like action_mask: the JSON config carries them next to the fields (Learner._cfg)."""
    import torched_impala_b200.engine as engine_mod
    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpPolicy, MlpValueFn
    from torched_impala_b200.utils import default_hparams

    o = LearnerOptions()
    assert o.obs_norm is False and o.obs_norm_eps == 1e-8
    assert {"obs_norm", "obs_norm_eps"}.isdisjoint(dataclasses.asdict(o))
    on = LearnerOptions(obs_norm=True, obs_norm_eps=1e-5, popart=True, frames=2)
    assert on != o and on != LearnerOptions(obs_norm=True, popart=True, frames=2)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    lrn = Learner(0, hp, MlpPolicy(24, 4, 32), MlpValueFn(24, 32), None, None, obs_norm=True, obs_norm_eps=1e-5,
                  popart=True, frames=2)
    assert lrn.options == on
    cfg = json.loads(json.dumps(lrn._cfg()))
    seen = {}
    monkeypatch.setattr(engine_mod, "LearnerEngine", lambda *a, **kw: seen.update(kw))
    engine_mod.engine_from_cfg(cfg, 1, "cpu")
    opts = {k: seen[k] for k in ("obs_norm", "obs_norm_eps") + tuple(f.name for f in dataclasses.fields(o))}
    assert LearnerOptions(**opts) == on


def test_fresh_statistics_are_the_identity():
    mu_f, r_f = obs_norm_f32(np.zeros(5), np.ones(5), 1e-8)
    assert (mu_f == 0).all() and (r_f == np.float32(1.0)).all()


def _net(rng, O, H, N):
    return (rng.standard_normal((H, O)) * 0.3, rng.standard_normal(H) * 0.1, rng.standard_normal((N, H)) * 0.3,
            rng.standard_normal(N) * 0.1)


def test_fold_and_unfold_are_inverses():
    rng = np.random.default_rng(0)
    W1, b1, _, _ = _net(rng, 17, 64, 6)
    mu_f, r_f = onorc.norm_f32(rng.uniform(-100, 100, 17), 10.0 ** rng.uniform(-4, 4, 17), 1e-8)
    W, b = onorc.unfold(*onorc.fold(W1, b1, mu_f, r_f), mu_f, r_f)
    np.testing.assert_allclose(W, W1, rtol=1e-15, atol=0)
    np.testing.assert_allclose(b, b1, rtol=1e-12, atol=1e-12)
    Wf, bf = onorc.fold(*onorc.unfold(W1, b1, mu_f, r_f), mu_f, r_f)
    np.testing.assert_allclose(Wf, W1, rtol=1e-15, atol=0)
    np.testing.assert_allclose(bf, b1, rtol=1e-12, atol=1e-12)


def test_folded_net_on_raw_rows_is_the_trained_net_on_normalized_rows():
    rng = np.random.default_rng(1)
    W1, b1, W2, b2 = _net(rng, 17, 64, 12)
    x = onorc.scaled_obs(2, 5, 9, 17, np.full(9, 5)).reshape(-1, 17).astype(np.float64)
    mu_f, r_f = onorc.norm_f32(x.mean(0), x.var(0), 1e-8)
    xn = (x - mu_f.astype(np.float64)) * r_f.astype(np.float64)

    def f(x, W1, b1):
        return np.maximum(x @ W1.T + b1, 0.0) @ W2.T + b2

    Wf, bf = onorc.fold(W1, b1, mu_f, r_f)
    np.testing.assert_allclose(f(x, Wf, bf), f(xn, W1, b1), rtol=1e-9, atol=1e-9)


def test_chan_merge_equals_the_concatenation():
    rng = np.random.default_rng(3)
    T, B, O = 7, 11, 9
    run = onorc.Running(O)
    rows = []
    for k in range(5):
        lens = rng.integers(0, T + 1, B)
        x = onorc.scaled_obs(10 + k, T, B, O, lens).astype(np.float64)
        run.update(x, lens, T)
        rows.append(x[onorc.valid_rows(lens, T)])
    n, mean, var = onorc.stats_of(np.concatenate(rows))
    assert run.count == n
    np.testing.assert_allclose(run.mean, mean, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(run.var, var, rtol=1e-9, atol=1e-12)
    assert run.var[0] == pytest.approx(0.0, abs=1e-20 + 1e-12 * abs(mean[0]) ** 2)  # the constant feature


def test_valid_rows_rule_on_ragged_lens():
    T, B, O = 6, 8, 3
    lens = np.array([0, 1, 6, 3, 0, 5, 2, 6])
    x = np.arange((T + 1) * B * O, dtype=np.float64).reshape(T + 1, B, O)
    s1, s2, n = onorc.batch_sums(x, lens, T)
    keep = np.zeros((T + 1, B), bool)
    for b, L in enumerate(lens):
        keep[:L, b] = True  # never the bootstrap row t = lens[b], never padding
    assert n == keep.sum() == lens.sum()
    np.testing.assert_array_equal(s1, x[keep].sum(0))
    np.testing.assert_array_equal(s2, (x[keep] ** 2).sum(0))
    # a batch with no valid row leaves the statistics as they are
    s1, s2, n = onorc.batch_sums(x, np.zeros(B, int), T)
    assert n == 0 and (s1 == 0).all() and (s2 == 0).all()
    c, m, v = onorc.merge(4.0, np.ones(O), np.full(O, 2.0), s1, s2, n)
    assert c == 4.0 and (m == 1).all() and (v == 2).all()


def test_frames_statistics_are_per_dense_feature():
    T, B, k, F = 4, 3, 3, 2
    frames = np.random.default_rng(5).standard_normal((T + k, B, F))
    dense = onorc.dense_rows(frames, T, k)
    assert dense.shape == (T + 1, B, k * F)
    np.testing.assert_array_equal(dense[2, 1, F:2 * F], frames[3, 1])


def test_obs_norm_push_refusals():
    """impala_mlp_backward_pair_push_obs_norm: at most 32 logged extras (as impala_mlp_backward_pair_push), a slot that
    holds them and the 2 O + 1 observation sums, O <= 1024; refused before any launch."""
    import ctypes as C

    from torched_impala_b200 import _cabi

    lib = _cabi.lib()
    p = C.c_void_p(1 << 20)
    T, B, O, H, A = 5, 8, 24, 256, 4
    M_pi, M_vf = T * B, (T + 1) * B
    n = _cabi.param_layout(O, H, A)[1] + _cabi.param_layout(O, H, 1)[1]
    big = 1 << 40

    def rc(n_extra=4, slot=n + 4 + 2 * O + 1, O=O):
        return lib.impala_mlp_backward_pair_push_obs_norm(p, p, p, p, p, p, big, p, big, M_pi, M_vf, O, H, H, A, p,
                                                          n_extra, p, p, slot, 2 * slot, 0, 2, None)

    assert rc(n_extra=33, slot=n + 33 + 2 * O + 1) == -1  # IMPALA_ERR_BAD_ARG
    assert rc(slot=n + 4 + 2 * O) == -1  # the slot must hold the observation sums too
    assert rc(O=1025, slot=n + 4 + 2 * 1025 + 1) == -1
