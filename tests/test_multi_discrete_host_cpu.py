"""CPU: multi-discrete policies on the host side - the ring and packer round trips, their refusals, the Learner's
ring check, configuration and evaluation."""
import json

import numpy as np
import pytest
import torch

from torched_impala_b200 import _cabi, engine, synth
from torched_impala_b200.learner import Learner, pack_trajectory
from torched_impala_b200.models import MlpValueFn, MultiDiscreteMlpPolicy
from torched_impala_b200.ring import RingQueue, _layout
from torched_impala_b200.utils import default_hparams

T, B, O, HEADS = 6, 8, 5, (3, 3, 2)
N, K = sum(HEADS), len(HEADS)


@pytest.fixture
def ring():
    q = RingQueue(T, B, O, N, slabs=2, action_dist="multi_discrete", action_heads=HEADS)
    yield q
    q.close()


@pytest.mark.parametrize("heads", [(2,), (3, 3, 2), (3, 3, 2, 2, 5, 5), (2,) * 16])
@pytest.mark.parametrize("frames", [1, 5])
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_python_layout_equals_library(obs_dtype, frames, heads):
    n = sum(heads)
    assert _layout(20, 96, 40, n, obs_dtype, frames, "multi_discrete", heads) == _cabi.batch_layout(
        20, 96, 40, n, obs_dtype, frames, "multi_discrete", heads)
    if len(heads) == 1:  # one head: the categorical layout
        assert _layout(20, 96, 40, n, obs_dtype, frames, "multi_discrete", heads) == _layout(20, 96, 40, n, obs_dtype,
                                                                                           frames)


def test_ring_round_trip_put_and_put_block(ring):
    b = synth.make_md_batch(1, T, B, O, HEADS, ragged=True)
    for tr in synth.to_trajectories(b, torch.float32):
        ring.put(tr)
    k, _ = ring.collect_batch(1)
    v = ring.views(k)
    for name in ("obs", "beh_logits", "actions", "rewards", "done", "lens"):
        assert np.array_equal(v[name], b[name]), name
    ring.release(k)
    b2 = synth.make_md_batch(2, T, B, O, HEADS, ragged=True)
    for lo in range(0, B, 4):
        ring.put_block({n: (x[lo:lo + 4] if n == "lens" else x[:, lo:lo + 4]) for n, x in b2.items()})
    k, _ = ring.collect_batch(1)
    for name in ("beh_logits", "actions", "lens"):
        assert np.array_equal(ring.views(k)[name], b2[name]), name


def _traj(**change):
    b = synth.make_md_batch(3, T, 1, O, HEADS)
    b["lens"][:] = T
    tr = synth.to_trajectories(b)[0]
    for name, (t, val) in change.items():
        getattr(tr, name)[t] = val
    return tr


@pytest.mark.parametrize("change, match", [
    (dict(a=(1, torch.zeros(K + 1, dtype=torch.int64))), "step 1 action has shape"),
    (dict(a=(0, torch.zeros(1, dtype=torch.int64))), "step 0 action has shape"),
    (dict(a=(2, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64))), "step 2 action has dtype"),
    (dict(a=(3, torch.tensor([0, 3, 0]))), "step 3 head 1 action 3 is outside"),
    (dict(a=(4, torch.tensor([0, 0, -1]))), "step 4 head 2 action -1 is outside"),
    (dict(logits=(2, torch.zeros(N - 1, dtype=torch.float64))), "step 2 behaviour logits have shape")])
def test_packer_and_put_refuse_bad_steps(ring, change, match):
    tr = _traj(**change)
    views = {name: np.zeros_like(x) for name, x in ring.views(0).items()}
    with pytest.raises(ValueError, match=match):
        pack_trajectory(views, 0, tr, T, heads=HEADS)
    with pytest.raises(ValueError, match=match):
        ring.put(tr)
    assert int(ring._control()["ticket"][0]) == 0  # refused before a column was taken


def test_put_block_refuses_bad_blocks(ring):
    b = synth.make_md_batch(4, T, 4, O, HEADS)
    ok = {n: x for n, x in b.items()}
    for name, val, match in (("actions", b["actions"][..., :2], "actions of shape"),
                             ("actions", b["actions"].astype(np.float32), "dtype"),
                             ("beh_logits", b["beh_logits"][..., 1:], "beh_logits of shape")):
        with pytest.raises(ValueError, match=match):
            ring.put_block(dict(ok, **{name: val}))
    bad = b["actions"].copy()
    bad[2, 3, 2] = 2  # head 2 has 2 actions
    with pytest.raises(ValueError, match="column 3 step 2 head 2 action 2 is outside"):
        ring.put_block(dict(ok, actions=bad))
    ring.put_block(ok)  # the good block goes through


def test_ring_refuses_bad_arguments():
    for kw in (dict(action_heads=(3, 3)), dict(action_heads=(3, 1, 4)), dict(action_heads=()),
               dict(action_dist="categorical", action_heads=HEADS)):
        with pytest.raises(ValueError):
            RingQueue(T, B, O, N, slabs=2, **dict(dict(action_dist="multi_discrete"), **kw))


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


def test_learner_ring_check_config_and_evaluation(monkeypatch, capsys):
    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=B, max_timesteps=T)
    pol, vf = MultiDiscreteMlpPolicy(O, HEADS, 16), MlpValueFn(O, 16)
    kw = dict(action_dist="multi_discrete", action_heads=HEADS)
    for q_kw, match in ((dict(action_dist="multi_discrete", action_heads=(3, 2, 3)), "action heads"),
                        (dict(), "actions")):
        q = RingQueue(T, B, O, N, slabs=2, **q_kw)
        try:
            with pytest.raises(ValueError, match=match):
                Learner(0, hp, pol, vf, q, None, **kw)
        finally:
            q.close()
    with pytest.raises(ValueError):  # the heads must sum to the policy's outputs
        Learner(0, hp, pol, vf, None, None, action_dist="multi_discrete", action_heads=(3, 3))
    q = RingQueue(T, B, O, N, slabs=2, **kw)
    try:
        lrn = Learner(0, hp, pol, vf, q, None, **kw)
    finally:
        q.close()
    cfg = json.loads(json.dumps(lrn._cfg()))
    assert cfg["A"] == N and cfg["action_heads"] == list(HEADS)
    calls = []
    monkeypatch.setattr(engine, "LearnerEngine", lambda *a, **k: calls.append(k))
    engine.engine_from_cfg(cfg, 1, "cuda:0")
    assert calls[0]["action_heads"] == HEADS and calls[0]["action_dist"] == "multi_discrete"
    assert lrn._evaluate(pol) is None
    assert "evaluation skipped: a multi-discrete policy" in capsys.readouterr().out
