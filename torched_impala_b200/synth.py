"""Seeded synthetic trajectory batches in the learner's HBM layout.

The reference has no (T, B) tensor anywhere: a "batch" is `batch_size` python
`Trajectory` objects pulled one at a time from the queue
(`learner.py:89-117`).  The GPU learner's device layout is
time-major and dense:

    obs        (T+1, B, O) f32   index T is the bootstrap observation slot (u8 for byte observations)
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
               unit_reward: bool = False, done_last: bool = True, obs_kind: str = "normal", frames: int = 1) -> dict:
    """obs_kind: "normal" - float32 N(0, 1); "bytes" - uint8 0..255 (Atari RAM); "planes" - uint8 0/1
    (MinAtar).  The integer kinds draw from a stream of their own, so every other field equals the
    "normal" batch of the same seed.  frames=k > 1: obs are the (T+k, B, O/k) frames of k-frame stacked
    observations (the layout of impala_batch_layout_frames), drawn from a stream of their own, zero from
    frame lens[b] + k on; `stack_frames` gives the dense batch."""
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((T + 1, B, O), dtype=np.float32)
    if obs_kind != "normal":
        irng = np.random.default_rng(seed + 104729)
        if obs_kind == "bytes":
            obs = irng.integers(0, 256, (T + 1, B, O), dtype=np.uint8)
        elif obs_kind == "planes":
            obs = (irng.random((T + 1, B, O)) < 0.3).astype(np.uint8)
        else:
            raise ValueError(f"obs_kind must be 'normal', 'bytes' or 'planes', got {obs_kind!r}")
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
    if frames > 1:
        if O % frames:
            raise ValueError(f"{O} observation features do not split into {frames} frames")
        frng = np.random.default_rng(seed + 15485863)
        shape = (T + frames, B, O // frames)
        if obs_kind == "normal":
            obs = frng.standard_normal(shape, dtype=np.float32)
        elif obs_kind == "bytes":
            obs = frng.integers(0, 256, shape, dtype=np.uint8)
        else:
            obs = (frng.random(shape) < 0.3).astype(np.uint8)
        obs[np.arange(T + frames)[:, None] >= lens[None, :] + frames] = 0
    return dict(obs=obs, beh_logits=beh, actions=actions, rewards=rewards, done=done,
                lens=lens)


def stack_frames(batch: dict, k: int) -> dict:
    """A frame batch (obs (T+k, B, F)) as the dense batch (obs (T+1, B, k F)) the frames stand for: row (t, b)
    is frames t .. t+k-1 of column b, oldest first.  Padded rows past lens[b] keep the frames they share with
    valid rows, as the device unstacking produces them."""
    fr = batch["obs"]
    T1 = fr.shape[0] - k + 1
    return {**batch, "obs": np.concatenate([fr[j:j + T1] for j in range(k)], axis=-1)}


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


def make_gaussian_batch(seed: int, T: int, B: int, O: int, A: int, ragged: bool = False, params: dict | None = None,
                        obs_kind: str = "normal", frames: int = 1) -> dict:
    """A batch of a diagonal Gaussian policy over A action dimensions (action_dist="gaussian"): obs, rewards, done
    and lens as make_batch(seed, ..., A=1); beh_logits (T, B, 2A) the behaviour outputs [m | s] and actions
    (T, B, A) float32 samples m + e^s eps.  With `params` (init_params(seed, O, 2A, H) layout) the behaviour is the
    policy's own output on the (dense) observations, moved 0.1-0.3 per entry (the off-policy lag of an actor);
    without, m ~ N(0, 1) and s ~ U(-1.5, 0.5).  Padded steps are zero."""
    b = make_batch(seed, T, B, O, 1, ragged=ragged, obs_kind=obs_kind, frames=frames)
    rng = np.random.default_rng(seed + 1299709)
    if params is None:
        beh = np.concatenate([rng.standard_normal((T, B, A)), rng.uniform(-1.5, 0.5, (T, B, A))], -1)
    else:
        x = (stack_frames(b, frames) if frames > 1 else b)["obs"][:-1].astype(np.float64)
        p = [np.asarray(params["policy"][k], np.float64) for k in ("model.0.weight", "model.0.bias",
                                                                      "model.3.weight", "model.3.bias")]
        beh = np.maximum(x @ p[0].T + p[1], 0.0) @ p[2].T + p[3]
        beh = beh + rng.uniform(0.1, 0.3, beh.shape) * rng.choice([-1.0, 1.0], beh.shape)
    act = beh[..., :A] + np.exp(beh[..., A:]) * rng.standard_normal((T, B, A))
    pad = np.arange(T)[:, None] >= b["lens"][None, :]
    beh[pad], act[pad] = 0.0, 0.0
    return dict(b, beh_logits=beh.astype(np.float32), actions=act.astype(np.float32))


def make_md_batch(seed: int, T: int, B: int, O: int, heads, ragged: bool = False, params: dict | None = None,
                  obs_kind: str = "normal", frames: int = 1) -> dict:
    """A batch of a multi-discrete policy with head sizes `heads` (action_dist="multi_discrete"): obs, rewards, done
    and lens as make_batch(seed, ..., A=2); beh_logits (T, B, N = sum heads) and actions (T, B, K) int32, one index per
    head sampled from the softmax of its slice.  With `params` (init_params(seed, O, N, H) layout) the behaviour is the
    policy's own output on the (dense) observations, moved 0.1-0.3 per entry (the off-policy lag of an actor);
    without, N(0, 1) logits.  Padded steps are zero."""
    heads = tuple(int(n) for n in heads)
    N, K = sum(heads), len(heads)
    b = make_batch(seed, T, B, O, 2, ragged=ragged, obs_kind=obs_kind, frames=frames)
    rng = np.random.default_rng(seed + 7919)
    if params is None:
        beh = rng.standard_normal((T, B, N))
    else:
        x = (stack_frames(b, frames) if frames > 1 else b)["obs"][:-1].astype(np.float64)
        p = [np.asarray(params["policy"][k], np.float64) for k in ("model.0.weight", "model.0.bias",
                                                                      "model.3.weight", "model.3.bias")]
        beh = np.maximum(x @ p[0].T + p[1], 0.0) @ p[2].T + p[3]
        beh = beh + rng.uniform(0.1, 0.3, beh.shape) * rng.choice([-1.0, 1.0], beh.shape)
    beh = beh.astype(np.float32)
    act = np.zeros((T, B, K), np.int32)
    s = 0
    for k, n in enumerate(heads):
        z = beh[..., s:s + n].astype(np.float64)
        q = np.exp(z - z.max(-1, keepdims=True))
        q /= q.sum(-1, keepdims=True)
        act[..., k] = np.minimum((np.cumsum(q, -1) < rng.random((T, B, 1))).sum(-1), n - 1)
        s += n
    pad = np.arange(T)[:, None] >= b["lens"][None, :]
    beh[pad], act[pad] = 0.0, 0
    return dict(b, beh_logits=beh, actions=act)


def draw_legal(rng, T: int, B: int, heads, density: float = 0.5, single: float = 0.1):
    """(T, B, N) bool legal-action masks over the heads (categorical: one head of N): each entry legal with probability
    `density`, at least one legal entry per head, and a fraction `single` of the steps with one legal entry per head."""
    heads = tuple(int(n) for n in heads)
    legal = rng.random((T, B, sum(heads))) < density
    one = rng.random((T, B)) < single
    s = 0
    for n in heads:
        h = legal[..., s:s + n]
        pick = rng.integers(0, n, (T, B))
        sole = np.arange(n) == pick[..., None]
        h[...] = np.where(one[..., None], sole, h | (~h.any(-1, keepdims=True) & sole))
        s += n
    return legal


def legal_words(legal) -> np.ndarray:
    """(..., N) bool legal masks -> (...) int32 legal words, bit j = entry j (the slab's last action column)."""
    legal = np.asarray(legal, bool)
    w = (legal.astype(np.uint64) << np.arange(legal.shape[-1], dtype=np.uint64)).sum(-1)
    return w.astype(np.uint32).view(np.int32)


def make_masked_batch(seed: int, T: int, B: int, O: int, A: int, heads=(), density: float = 0.5, ragged: bool = False,
                      params: dict | None = None, obs_kind: str = "normal", frames: int = 1) -> dict:
    """A batch of a masked policy (action_mask=True): categorical over A actions (heads=()) or multi-discrete with
    `heads` (sum = A).  obs, rewards, done and lens as make_batch; legal masks per step (draw_legal: `density`, at
    least one legal entry per head, some single-legal steps); behaviour logits as make_batch / make_md_batch, the
    actions drawn from the behaviour softmax renormalised over the legal entries, and garbage (+-1e30, -inf, NaN) in
    the illegal behaviour logits, as an actor may record.  actions (T, B, 2) [a, legal] or (T, B, K + 1)
    [a_0 .. a_{K-1}, legal] int32 (a multi-discrete batch of one head has the categorical layout); `legal` (T, B, A)
    bool rides along.  Padded steps are zero (legal word 0)."""
    md = bool(len(heads))
    heads = tuple(int(n) for n in heads) or (A,)
    if sum(heads) != A:
        raise ValueError(f"the heads {heads} do not have A = {A} outputs")
    b = make_batch(seed, T, B, O, 2, ragged=ragged, obs_kind=obs_kind, frames=frames)
    rng = np.random.default_rng(seed + 15485863)
    if params is None:
        beh = rng.standard_normal((T, B, A))
    else:
        x = (stack_frames(b, frames) if frames > 1 else b)["obs"][:-1].astype(np.float64)
        p = [np.asarray(params["policy"][k], np.float64) for k in ("model.0.weight", "model.0.bias",
                                                                      "model.3.weight", "model.3.bias")]
        beh = np.maximum(x @ p[0].T + p[1], 0.0) @ p[2].T + p[3]
        beh = beh + rng.uniform(0.1, 0.3, beh.shape) * rng.choice([-1.0, 1.0], beh.shape)
    legal = draw_legal(rng, T, B, heads, density)
    K = len(heads)
    act = np.zeros((T, B, K), np.int32)
    s = 0
    for k, n in enumerate(heads):
        z = np.where(legal[..., s:s + n], beh[..., s:s + n], -np.inf)
        q = np.exp(z - z.max(-1, keepdims=True))
        q /= q.sum(-1, keepdims=True)
        a = np.minimum((np.cumsum(q, -1) < 1.0 - rng.random((T, B, 1))).sum(-1), n - 1)
        while True:  # the cumulative sum may end a rounding short of 1: step back onto a legal entry
            off = ~np.take_along_axis(legal[..., s:s + n], a[..., None], -1)[..., 0]
            if not off.any():
                break
            a = np.where(off, a - 1, a)
        act[..., k] = a
        s += n
    beh = beh.astype(np.float32)
    garbage = np.array([1e30, -1e30, -np.inf, np.nan], np.float32)
    beh = np.where(legal, beh, garbage[rng.integers(0, 4, beh.shape)]).astype(np.float32)
    pad = np.arange(T)[:, None] >= b["lens"][None, :]
    beh[pad], act[pad], legal[pad] = 0.0, 0, False
    words = legal_words(legal)
    actions = np.concatenate([act, words[..., None]], -1).astype(np.int32)
    return dict(b, beh_logits=beh, actions=actions, legal=legal)


def to_trajectories(batch: dict, torch_dtype=None) -> list:
    """Expand a dense batch into the reference wire format (one Trajectory per b).

    Shapes/dtypes follow what actor.py:72-92 appends: obs (O,) f64, a (1,) i64,
    r () f64, d () bool, logits (A,) f64.  A Gaussian batch (actions (T, B, A)) gives a (A,) f64 and
    logits (2A,) f64; a multi-discrete batch (int32 actions (T, B, K)) a (K,) i64 and logits (N,) f64.  A masked
    batch (make_masked_batch: `legal` present, the legal word last in the actions) gives the indices without the word
    and traj.action_mask, (N,) bool per step.
    """
    import torch

    from .utils import Trajectory

    dt = torch.float64 if torch_dtype is None else torch_dtype
    obs = torch.from_numpy(batch["obs"]).to(dt)
    beh = torch.from_numpy(batch["beh_logits"]).to(dt)
    # (T, B, A) float actions: Gaussian samples; (T, B, K) integer actions: multi-discrete indices
    gauss = batch["actions"].ndim == 3 and np.issubdtype(batch["actions"].dtype, np.floating)
    multi = batch["actions"].ndim == 3 and not gauss
    masked = "legal" in batch
    act = torch.from_numpy(batch["actions"][..., :-1] if masked else batch["actions"]).to(dt if gauss else torch.int64)
    legal = torch.from_numpy(batch["legal"]) if masked else None
    rew = torch.from_numpy(batch["rewards"]).to(dt)
    don = torch.from_numpy(batch["done"]).to(torch.bool)
    out = []
    for b, L in enumerate(batch["lens"].tolist()):
        tr = Trajectory((0, b + 1))
        tr.obs.append(obs[0, b].clone())
        for t in range(L):
            tr.add(obs[t + 1, b].clone(), act[t, b].clone() if gauss or multi else act[t, b].reshape(1).clone(), rew[t, b].clone(),
                   don[t, b].clone(), beh[t, b].clone())
        if masked:
            tr.action_mask = [legal[t, b].clone() for t in range(L)]
        out.append(tr)
    return out
