"""CPU: Gaussian policies on the host side - the ring and packer round trip, their refusals, the Learner's
argument checks and configuration, the policy module and the synthetic batches."""
import multiprocessing as mp

import numpy as np
import pytest
import torch

from torched_impala_b200 import _cabi, synth
from torched_impala_b200.learner import Learner, pack_trajectory
from torched_impala_b200.models import GaussianMlpPolicy, MlpPolicy, MlpValueFn
from torched_impala_b200.ring import RingQueue, _layout
from torched_impala_b200.utils import default_hparams

T, B, O, A = 6, 8, 5, 3


@pytest.fixture
def ring():
    q = RingQueue(T, B, O, A, slabs=2, action_dist="gaussian")
    yield q
    q.close()


@pytest.mark.parametrize("frames", [1, 5])
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_python_layout_equals_library(obs_dtype, frames):
    assert _layout(20, 96, 40, 6, obs_dtype, frames, "gaussian") == _cabi.batch_layout(20, 96, 40, 6, obs_dtype,
                                                                                      frames, "gaussian")
    assert _layout(20, 96, 40, 6, obs_dtype, frames) == _cabi.batch_layout(20, 96, 40, 6, obs_dtype, frames)


def test_ring_round_trip_put_and_put_block(ring):
    b = synth.make_gaussian_batch(1, T, B, O, A, ragged=True)
    for tr in synth.to_trajectories(b, torch.float32):  # any float dtype
        ring.put(tr)
    k, reward = ring.collect_batch(1)
    v = ring.views(k)
    for name in ("obs", "beh_logits", "actions", "rewards", "done", "lens"):
        assert np.array_equal(v[name], b[name]), name
    ring.release(k)
    b2 = synth.make_gaussian_batch(2, T, B, O, A, ragged=True)
    for lo in range(0, B, 4):
        ring.put_block({n: (x[lo:lo + 4] if n == "lens" else x[:, lo:lo + 4]) for n, x in b2.items()})
    k, _ = ring.collect_batch(1)
    for name in ("beh_logits", "actions", "lens"):
        assert np.array_equal(ring.views(k)[name], b2[name]), name


def _traj(**change):
    tr = synth.to_trajectories(synth.make_gaussian_batch(3, T, 1, O, A))[0]
    for name, (t, val) in change.items():
        getattr(tr, name)[t] = val
    return tr


@pytest.mark.parametrize("change", [dict(a=(1, torch.zeros(A + 1, dtype=torch.float64))),
                                    dict(a=(0, torch.zeros(1, dtype=torch.int64))),
                                    dict(logits=(2, torch.zeros(A, dtype=torch.float64))),
                                    dict(a=(3, torch.tensor([0.0, float("nan"), 0.0], dtype=torch.float64))),
                                    dict(logits=(0, torch.tensor([0.0] * 5 + [float("inf")], dtype=torch.float64)))])
def test_packer_refuses_bad_steps(ring, change):
    tr = _traj(**change)
    tr.id = 77
    with pytest.raises(ValueError, match="trajectory 77"):
        ring.put(tr)
    for tr in synth.to_trajectories(synth.make_gaussian_batch(4, T, B - 1, O, A)):  # the ring stays usable
        ring.put(tr)
    k, _ = ring.collect_batch(1)
    assert ring.views(k)["lens"][0] == 0  # the refused column went out empty


def test_put_block_refuses_bad_blocks(ring):
    b = synth.make_gaussian_batch(5, T, 4, O, A)
    with pytest.raises(ValueError, match="actions"):
        ring.put_block(dict(b, actions=b["actions"][..., :2]))
    bad = b["beh_logits"].copy()
    bad[1, 2, 0] = np.nan
    with pytest.raises(ValueError, match="non-finite beh_logits"):
        ring.put_block(dict(b, beh_logits=bad))


def test_ring_refuses_bad_arguments():
    with pytest.raises(ValueError):
        RingQueue(T, B, O, 17, action_dist="gaussian")
    with pytest.raises(ValueError):
        RingQueue(T, B, O, A, action_dist="beta")


def test_pack_trajectory_into_engine_layout():
    views = {"obs": np.zeros((T + 1, B, O), np.float32), "beh_logits": np.zeros((T, B, 2 * A), np.float32),
             "actions": np.zeros((T, B, A), np.float32), "rewards": np.zeros((T, B), np.float32),
             "done": np.zeros((T, B), np.uint8), "lens": np.zeros(B, np.int32)}
    b = synth.make_gaussian_batch(6, T, B, O, A, ragged=True)
    for j, tr in enumerate(synth.to_trajectories(b)):
        pack_trajectory(views, j, tr, T)
    for name in views:
        assert np.array_equal(views[name], b[name]), name


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


def test_learner_refusals_and_config(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=B, max_timesteps=T)
    v = MlpValueFn(O, 16)
    for n_out in (5, 34):  # odd, more than 2 x 16
        with pytest.raises(ValueError, match="2A outputs"):
            Learner(0, hp, MlpPolicy(O, n_out, 16), v, mp.Queue(), None, action_dist="gaussian")
    with pytest.raises(ValueError, match="action_dist"):
        Learner(0, hp, GaussianMlpPolicy(O, A, 16), v, mp.Queue(), None, action_dist="normal")
    cat_ring, g_ring = RingQueue(T, B, O, 2 * A, slabs=2), RingQueue(T, B, O, A, slabs=2, action_dist="gaussian")
    try:
        with pytest.raises(ValueError, match="categorical actions"):
            Learner(0, hp, GaussianMlpPolicy(O, A, 16), v, cat_ring, None, action_dist="gaussian")
        with pytest.raises(ValueError, match="gaussian actions"):
            Learner(0, hp, MlpPolicy(O, 2 * A, 16), v, g_ring, None)
        lrn = Learner(0, hp, GaussianMlpPolicy(O, A, 16), v, g_ring, None, action_dist="gaussian")
        c = lrn._cfg()
        assert c["action_dist"] == "gaussian" and c["A"] == A
        assert lrn._evaluate(lrn.policy) is None  # no evaluator: skipped
        assert Learner(0, hp, MlpPolicy(O, 2 * A, 16), v, cat_ring, None)._cfg()["A"] == 2 * A
    finally:
        cat_ring.close()
        g_ring.close()


def test_gaussian_policy_module():
    p = GaussianMlpPolicy(O, A, 16)
    assert set(p.state_dict()) == set(MlpPolicy(O, A, 16).state_dict())
    assert p.state_dict()["model.3.weight"].shape == (2 * A, 16)
    obs = torch.randn(O, dtype=torch.float64)
    a, params = p.select_action(obs)
    assert a.shape == (A,) and a.dtype == torch.float64 and params.shape == (2 * A,)
    p.eval()
    m, params = p.select_action(obs, deterministic=True)
    assert torch.equal(m, p(obs)[:A])


def test_make_gaussian_batch():
    params = synth.init_params(1, O, 2 * A, 16)
    b = synth.make_gaussian_batch(8, T, B, O, A, ragged=True, params=params)
    assert b["beh_logits"].shape == (T, B, 2 * A) and b["actions"].shape == (T, B, A)
    assert b["actions"].dtype == np.float32 and np.isfinite(b["actions"]).all()
    pad = np.arange(T)[:, None] >= b["lens"][None, :]
    assert not b["actions"][pad].any() and not b["beh_logits"][pad].any()
