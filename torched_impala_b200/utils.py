"""Boundary types of the learner hot path.

These are the three containers that cross the actor -> learner boundary in the
reference (`utils.py:17-45` Hyperparameters, `:48-77`
Trajectory, `:80-92` Counter).  The GPU learner consumes the reference's own
objects unchanged (it only duck-types on attribute names); the definitions
here exist so that the package, its tests and its benchmark are self-contained
on a machine that does not have the reference checked out.  Field names and
order are part of the wire contract and therefore identical.
"""
from __future__ import annotations

import collections
import multiprocessing as _mp

# Field order matters: train.py builds this positionally-by-keyword and logs
# `str(hparams)` (reference utils.py:17-45).
_HP_FIELDS = (
    "max_updates policy_hidden_dims value_fn_hidden_dims batch_size gamma rho_bar c_bar "
    "lr policy_loss_c v_loss_c entropy_c max_timesteps queue_lim max_norm n_actors "
    "env_name log_path save_every eval_every eval_eps verbose render"
).split()

Hyperparameters = collections.namedtuple("Hyperparameters", _HP_FIELDS)


def default_hparams(**overrides) -> Hyperparameters:
    """The literal values of reference train.py:11-36, overridable by keyword."""
    base = dict(
        max_updates=50, policy_hidden_dims=128, value_fn_hidden_dims=128, batch_size=32,
        gamma=0.99, rho_bar=1.0, c_bar=1.0, lr=1e-3, policy_loss_c=1, v_loss_c=0.5,
        entropy_c=0.0006, max_timesteps=1000, queue_lim=8, max_norm=10, n_actors=1,
        env_name="CartPole-v1", log_path=None, save_every=50, eval_every=None,
        eval_eps=20, verbose=0, render=False,
    )
    base.update(overrides)
    return Hyperparameters(**base)


class Trajectory:
    """One episode prefix as the actor ships it (reference utils.py:48-77).

    Five parallel python lists of tiny tensors: `obs` has one more entry than
    the others (the bootstrap observation), `a` holds (1,) int64 tensors, `r`
    0-d float64, `d` 0-d bool, `logits` (A,) float64 behaviour logits.
    """

    __slots__ = ("id", "obs", "a", "r", "d", "logits", "action_mask")

    def __init__(self, id, observations=None, actions=None, rewards=None, dones=None,
                 logits=None):
        self.id = id
        # masked policies (Learner(action_mask=True)): the legal-action mask (A,) / (N,) of each step, true = legal,
        # appended by the actor next to the step; None for the others
        self.action_mask = None
        self.obs = [] if observations is None else observations
        self.a = [] if actions is None else actions
        self.r = [] if rewards is None else rewards
        self.d = [] if dones is None else dones
        self.logits = [] if logits is None else logits

    def add(self, obs, a, r, d, logits):
        self.obs.append(obs)
        self.a.append(a)
        self.r.append(r)
        self.d.append(d)
        self.logits.append(logits)


class Counter:
    """Lock-protected shared int (reference utils.py:80-92)."""

    def __init__(self, init_val: int = 0):
        self._val = _mp.RawValue("i", init_val)
        self._lock = _mp.Lock()

    def increment(self):
        with self._lock:
            self._val.value += 1

    @property
    def value(self):
        with self._lock:
            return self._val.value
