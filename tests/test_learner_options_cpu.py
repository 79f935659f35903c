"""CPU: the learner's feature options (engine.LearnerOptions) - one refusal, with one message, for a bad value wherever
the options are given (their own checks, LearnerEngine, Learner), the JSON round trip, and a data-parallel worker
rank building the engine of rank 0 from the JSON config."""
import dataclasses
import json
import queue

import numpy as np
import pytest
import torch

from torched_impala_b200 import _cabi, dp, engine
from torched_impala_b200.engine import LearnerEngine, LearnerOptions, engine_from_cfg
from torched_impala_b200.learner import Learner
from torched_impala_b200.models import MlpPolicy, MlpValueFn
from torched_impala_b200.optim import optim_config
from torched_impala_b200.utils import default_hparams

T, B, O, A, H = 5, 8, 12, 2, 16
DIMS = dict(A=A, H_pi=H, H_v=H, world=1)
DEVICES = ["cuda:0", "cuda:1"]


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


@pytest.fixture
def no_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda group=None: 2)  # the process group below


def _hp():
    return default_hparams(batch_size=B, max_timesteps=T)


def _checks(opts, d):
    """The options' own checks: LearnerOptions.check, and optim_config for the optimizer and its keywords."""
    o = LearnerOptions(**opts)
    o.check(B, O, d["A"], d["H_pi"], d["H_v"], d["world"])
    optim_config(_hp(), o.optimizer, o.optimizer_kwargs)


def _engine(opts, d):
    w = d["world"]
    return LearnerEngine(T, B // w, O, d["A"], d["H_pi"], d["H_v"], _hp(), process_group=object() if w > 1 else None,
                         **opts)


def _learner(opts, d):
    n_out = 2 * d["A"] if opts.get("action_dist") == "gaussian" else d["A"]
    return Learner(0, _hp(), MlpPolicy(O, n_out, d["H_pi"]), MlpValueFn(O, d["H_v"]), queue.Queue(), None,
                   devices=DEVICES[:d["world"]], **opts)


def _refusal(build, opts, d):
    with pytest.raises(Exception) as e:
        build(opts, d)
    return type(e.value), str(e.value)


# name: (bad options, their shapes, good options, their shapes); shapes default to DIMS, O = 12
CASES = {
    "obs_dtype": (dict(obs_dtype="float16"), {}, dict(obs_dtype="uint8"), {}),
    "reward_clip": (dict(reward_clip="clip"), {}, dict(reward_clip="soft_asymmetric"), {}),
    "action_dist": (dict(action_dist="normal"), {}, dict(action_dist="gaussian"), {}),
    "popart": (dict(popart="yes"), {}, dict(popart=True), {}),
    "popart_beta": (dict(popart=True, popart_beta=2.0), {}, dict(popart=True, popart_beta=1.0), {}),
    "optimizer": (dict(optimizer="sgd"), {}, dict(optimizer="rmsprop"), {}),
    "optimizer_kwargs": (dict(optimizer_kwargs=dict(eps=0.1)), {},
                         dict(optimizer="rmsprop", optimizer_kwargs=dict(eps=0.1)), {}),
    "frames_vs_O": (dict(frames=5), {}, dict(frames=4), {}),
    "frames_zero": (dict(frames=0), {}, dict(frames=1), {}),
    "gaussian_A": (dict(action_dist="gaussian"), dict(A=17), dict(action_dist="gaussian"), dict(A=16)),
    "shared_torso_widths": (dict(shared_torso=True), dict(H_v=2 * H), dict(shared_torso=True), {}),
    "shared_torso_outputs": (dict(shared_torso=True), dict(A=32), dict(shared_torso=True), dict(A=31)),
    "replay_vs_B": (dict(replay_slabs=2, replay_columns=B), {}, dict(replay_slabs=2, replay_columns=B - 1), {}),
    "replay_vs_devices": (dict(replay_slabs=2, replay_columns=3), dict(world=2),
                          dict(replay_slabs=2, replay_columns=3), {}),
}


@pytest.mark.parametrize("name", CASES)
def test_same_refusal_everywhere(name, no_cuda):
    bad, bad_dims, good, good_dims = CASES[name]
    bad_dims, good_dims = {**DIMS, **bad_dims}, {**DIMS, **good_dims}
    want = _refusal(_checks, bad, bad_dims)
    assert want[0] is ValueError, want
    assert _refusal(_engine, bad, bad_dims) == want
    assert _refusal(_learner, bad, bad_dims) == want
    _checks(good, good_dims)
    _learner(good, good_dims)
    with pytest.raises(AssertionError, match="CUDA was touched"):  # a good value goes on to the device checks
        _engine(good, good_dims)


def test_unknown_option_is_a_type_error(no_cuda):
    with pytest.raises(TypeError, match="obs_type"):
        _engine(dict(obs_type="uint8"), DIMS)
    with pytest.raises(TypeError, match="obs_type"):
        _learner(dict(obs_type="uint8"), DIMS)


# every field away from its default; the Gaussian policy has 2A + 1 <= 32 outputs with the shared torso
AWAY = LearnerOptions(obs_dtype="uint8", frames=4, diagnostics=True, replay_slabs=2, replay_columns=3,
                      optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01, momentum=0.9), popart=True,
                      popart_beta=0.01, reward_clip="soft_asymmetric", action_dist="gaussian", shared_torso=True)


def test_json_round_trip():
    default = dataclasses.asdict(LearnerOptions())
    assert all(getattr(AWAY, k) != v for k, v in default.items())
    assert LearnerOptions(**json.loads(json.dumps(dataclasses.asdict(AWAY)))) == AWAY
    kw = dict(eps=0.01)
    o = LearnerOptions(optimizer="rmsprop", optimizer_kwargs=kw)
    kw["eps"] = 0.5
    assert o.optimizer_kwargs == dict(eps=0.01) and type(o.optimizer_kwargs) is dict
    assert LearnerOptions(optimizer_kwargs=None).optimizer_kwargs == {}


class _Recorder:
    calls = []

    def __init__(self, *args, **kw):
        _Recorder.calls.append((args, kw))

    def load_state(self, *a):
        pass


@pytest.mark.parametrize("devices", [DEVICES, DEVICES[:1]], ids=["two_devices", "one_device"])
def test_worker_builds_the_engine_of_rank_0(devices, tmp_path, monkeypatch, no_cuda):
    """Rank 0 (Learner._make_engine) and a worker rank (dp_worker: the JSON of the spec and the init-state file) make
    the same LearnerEngine call, with the Learner's options.  Replay runs on one device only, so two devices take
    every other field away from its default."""
    monkeypatch.setattr(engine, "LearnerEngine", _Recorder)
    _Recorder.calls = []
    opts = AWAY if len(devices) == 1 else dataclasses.replace(AWAY, replay_slabs=0, replay_columns=0)
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=30, log_path=None)
    lrn = Learner(0, hp, MlpPolicy(O, 2 * A, H), MlpValueFn(O, H), queue.Queue(), None, devices=devices,
                  lr_lambda=lambda e: 1.0 - e / 30, **dataclasses.asdict(opts))
    assert lrn.options == opts
    world = len(devices)
    lrn._make_engine(None, world)
    path = str(tmp_path / "init_state.npz")
    dp.write_init_state(path, lrn._init_state(), lrn.optim.lr_table, lrn._popart_init())
    _, table = dp.read_init_state(path)
    engine_from_cfg(json.loads(json.dumps(lrn._cfg())), world, devices[-1], None, table)
    (args0, kw0), (args1, kw1) = _Recorder.calls
    assert args0 == args1 == (T, B // world, O, A, H, H, hp)
    t0, t1 = kw0.pop("lr_table"), kw1.pop("lr_table")
    assert t0.size == 30 and np.array_equal(t0, t1) and np.array_equal(t0, lrn.optim.lr_table)
    assert (kw0.pop("device"), kw1.pop("device")) == (devices[0], devices[-1])
    assert kw0 == kw1
    fields = [f.name for f in dataclasses.fields(LearnerOptions)]
    assert set(kw0) == {"global_batch", "mode", "process_group"} | set(fields)
    for name in fields:
        assert kw0[name] == getattr(lrn.options, name), name
