"""Seeded synthetic trajectory batches in the learner's HBM layout.

The reference has no (T, B) tensor anywhere: a "batch" is `batch_size` python
`Trajectory` objects pulled one at a time from the queue
(`learner.py:89-117`).  The GPU learner's device layout is
time-major and dense:

    obs        (T+1, B, O) f32   index T is the bootstrap observation slot
    beh_logits (T,   B, A) f32   behaviour-policy logits shipped by the actor
    actions    (T,   B)    i32
    rewards    (T,   B)    f32
    done       (T,   B)    u8
    lens       (B,)        i32   L_b <= T valid steps; obs[L_b, b] is the bootstrap

Everything past L_b is zero padding.  This module generates such batches
(SURVEY.md section 8d: obs/logits/rewards ~ N(0,1), actions ~ Categorical(softmax
of the behaviour logits), done only on the last valid step) and converts them to
the reference wire format (lists of tiny float64 tensors) so the same numbers can
be pushed through the reference learner.  Values are drawn in float32 so that
the float64 oracle sees bit-identical inputs.
"""
from __future__ import annotations

import numpy as np

PARAM_ALIGN = 32  # floats; every parameter tensor starts on a 128-byte boundary


def make_batch(seed: int, T: int, B: int, O: int, A: int, ragged: bool = False,
               unit_reward: bool = False, done_last: bool = True) -> dict:
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((T + 1, B, O), dtype=np.float32)
    beh = rng.standard_normal((T, B, A), dtype=np.float32)
    # Categorical(softmax(beh)) by inverse-CDF on a float64 copy.
    z = beh.astype(np.float64)
    p = np.exp(z - z.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    u = rng.random((T, B, 1))
    actions = np.minimum((np.cumsum(p, -1) < u).sum(-1), A - 1).astype(np.int32)
    if unit_reward:
        rewards = np.ones((T, B), dtype=np.float32)
    else:
        rewards = rng.standard_normal((T, B), dtype=np.float32)
    if ragged:
        lens = rng.integers(1, T + 1, size=B).astype(np.int32)
    else:
        lens = np.full(B, T, dtype=np.int32)
    done = np.zeros((T, B), dtype=np.uint8)
    if done_last:
        # an episode that ended early terminated; a full-length one was cut by max_timesteps
        ended = lens < T if ragged else np.zeros(B, bool)
        done[lens[ended] - 1, np.nonzero(ended)[0]] = 1
    t_idx = np.arange(T)[:, None]
    pad = t_idx >= lens[None, :]
    beh[pad] = 0
    actions[pad] = 0
    rewards[pad] = 0
    done[pad] = 0
    pad_obs = np.arange(T + 1)[:, None] > lens[None, :]
    obs[pad_obs] = 0
    return dict(obs=obs, beh_logits=beh, actions=actions, rewards=rewards, done=done,
                lens=lens)


def shard_batch(batch: dict, rank: int, world: int) -> dict:
    """Contiguous B/world slice of every (.., B, ..) tensor (SURVEY.md section 8e)."""
    B = batch["lens"].shape[0]
    if B % world:
        raise ValueError(f"batch_size {B} does not divide over {world} ranks")
    lo, hi = rank * (B // world), (rank + 1) * (B // world)
    out = {}
    for k, v in batch.items():
        out[k] = np.ascontiguousarray(v[lo:hi] if k == "lens" else v[:, lo:hi])
    return out


def init_params(seed: int, O: int, A: int, H_pi: int, H_v: int | None = None) -> dict:
    """nn.Linear-style U(-1/sqrt(fan_in), 1/sqrt(fan_in)) init for both MLPs.

    Keys follow the reference state_dict names (`model.0.*`, `model.3.*`,
    reference models.py:13-18 / :41-46).
    """
    H_v = H_pi if H_v is None else H_v
    rng = np.random.default_rng(seed + 7919)

    def lin(fan_out, fan_in):
        k = 1.0 / np.sqrt(fan_in)
        w = rng.uniform(-k, k, size=(fan_out, fan_in)).astype(np.float32)
        b = rng.uniform(-k, k, size=(fan_out,)).astype(np.float32)
        return w, b

    pw1, pb1 = lin(H_pi, O)
    pw2, pb2 = lin(A, H_pi)
    vw1, vb1 = lin(H_v, O)
    vw2, vb2 = lin(1, H_v)
    return {
        "policy": {"model.0.weight": pw1, "model.0.bias": pb1,
                   "model.3.weight": pw2, "model.3.bias": pb2},
        "value_fn": {"model.0.weight": vw1, "model.0.bias": vb1,
                     "model.3.weight": vw2, "model.3.bias": vb2},
    }


def to_trajectories(batch: dict, torch_dtype=None) -> list:
    """Expand a dense batch into the reference wire format (one Trajectory per b).

    Shapes/dtypes follow what actor.py:72-92 appends: obs (O,) f64, a (1,) i64,
    r () f64, d () bool, logits (A,) f64.
    """
    import torch

    from .utils import Trajectory

    dt = torch.float64 if torch_dtype is None else torch_dtype
    obs = torch.from_numpy(batch["obs"]).to(dt)
    beh = torch.from_numpy(batch["beh_logits"]).to(dt)
    act = torch.from_numpy(batch["actions"]).to(torch.int64)
    rew = torch.from_numpy(batch["rewards"]).to(dt)
    don = torch.from_numpy(batch["done"]).to(torch.bool)
    out = []
    for b, L in enumerate(batch["lens"].tolist()):
        tr = Trajectory((0, b + 1))
        tr.obs.append(obs[0, b].clone())
        for t in range(L):
            tr.add(obs[t + 1, b].clone(), act[t, b].reshape(1).clone(), rew[t, b].clone(),
                   don[t, b].clone(), beh[t, b].clone())
        out.append(tr)
    return out
