"""Drop-in `Learner` for the reference's actor/learner split, running the update on the GPU.

Same constructor, lifecycle methods, events, checkpoint format and module-level loss
helpers as `learner.py` (constructor `:18-28`, `start/terminate/join`
`:55-65`, `_learn` `:67-275`, `save/load/policy_weights` `:277-295`, helpers `:298-321`),
so `train.py:69` and the unmodified `actor.py` (`:68,70,118,121`) work against it:

  * trajectories arrive as pickled `utils.Trajectory` objects through the same `mp.Queue`
    (or through `ring.RingQueue`, same `put()` call); `queue.Empty` after `timeout` seconds sets
    `completion` and re-raises (`:91-100`);
  * new policy weights are copied IN PLACE into the (shared-memory, float64) `policy` module the
    actors read through `learner.policy_weights` (`actor.py:70`);
  * `update_counter.increment()` once per update; TensorBoard scalars under the same tags;
    checkpoints with keys `policy_state_dict` / `value_fn_state_dict`.

What changes is where the arithmetic happens and that nothing on the host sits on the critical
path of the device (SURVEY 8f-2, 8f-4):

  * `_learn` packs each trajectory into a pinned, zero-padded time-major host slab (replacing the
    torch.stack calls at `:104-109,117`) and hands the batch to `engine.LearnerEngine`, i.e. to the
    sm_90a kernels behind include/impala_b200.h; batch i+1 is collected and DMA'd while the
    kernels of batch i run;
  * weight publication: only the POLICY is published (it is all `actor.py:70` reads; `train.py:67`
    shares only the policy): after the step an in-stream device copy freezes the policy block, a
    side stream brings it to a double-buffered pinned snapshot, and a publisher thread writes it
    into the shared tensors under a version counter (`policy_version`, odd while a write is in
    progress; `policy_snapshot()` returns a consistent copy).  `publish_every` thins it out.  The
    value function reaches its module at checkpoints and at the end;
  * the logged scalars of update n are read while update n + 1 runs;
  * evaluation (`learner.py:195-214`) runs on a frozen copy of the policy in a background thread,
    it no longer blocks updates and no longer flips the training module's mode;
  * `devices=[...]`: data-parallel over the GPUs of one node, still ONE learner object/process
    for the launcher (dp.py): rank 0 lives here, publishes weights and logs;
  * `replay_slabs=R, replay_columns=Br` (experience replay, off by default): every update consumes
    `batch_size - Br` trajectories from the queue and fills its other Br columns from the fresh batches of
    the last R updates, kept in HBM (engine.py, replay.py); one device only;
  * `optimizer="rmsprop"`, `optimizer_kwargs` (torch's RMSprop keywords) and `lr_lambda` (a LambdaLR
    lambda, tabulated over hp.max_updates updates): the IMPALA paper's recipe (optim.py); the default is
    the reference's Adam at 0.95 * hp.lr.  With a log_path and either one set, `optim/lr` is logged;
  * `popart=True`, `popart_beta` (PopArt value normalization, off by default): the value net trains on targets
    normalized by running statistics of vs, kept and updated on the device (engine.py).  Checkpoints and
    `value_fn` hold the FOLDED value function (reward units), plus the statistics under the key "popart";
    `popart/mu` and `popart/sigma` are logged;
  * `reward_clip="abs_one"` (clip(r, -1, 1), the paper's Atari setting) or `"soft_asymmetric"` (DMLab's
    5 tanh(r / 5), 1.5 tanh(r / 5) below 0): the V-trace kernel transforms the rewards it reads, so actors, the
    transport and replay keep raw rewards and `rewards/batch_mean_reward` stays the raw game score.  A
    hyperparameter, not state: checkpoints are unchanged;
  * `obs_norm=True`, `obs_norm_eps` (observation normalization, off by default): the networks train on observations
    normalized by running per-feature statistics kept on the device (engine.py).  `policy`, `value_fn` and
    checkpoints hold the networks FOLDED into raw-observation coordinates, plus the statistics under the key
    "obs_norm", so actors keep feeding raw observations.

CUDA is initialised inside the learner process only (`train.py:42` forces the fork start method,
so the parent must never touch the device); a policy / value_fn that already lives on a CUDA
device is rejected with instructions (the reference picks `cuda` at import when it is visible).

Dropout: the reference MLPs carry `Dropout(p=0.8)` (models.py:15,44) and never call `.eval()` on
the learner's nets before the first evaluation.  This learner implements the deterministic
(`.eval()`) forward, the setting every parity number is quoted in (SURVEY.md section 0.4) -
swapping the class therefore changes training dynamics, not only speed (INTEGRATION.md).
"""
from __future__ import annotations

import copy
import dataclasses
import queue
import sys
import threading
import time
from pathlib import Path

import numpy as np
import torch
import torch.multiprocessing as mp

from .engine import LearnerOptions, engine_from_cfg
from .optim import optim_config

PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")


def _np(t, dtype):
    """Stacked trajectory field -> numpy of `dtype` (tensors an actor left on a GPU are fetched)."""
    return t.detach().to(dtype).cpu().numpy()


def check_trajectory(traj, T: int) -> int:
    """Length checks of learner.py:104-109's implicit contract; returns the number of steps."""
    L = len(traj.r)
    if L < 1 or L > T:
        raise ValueError(f"trajectory {getattr(traj, 'id', '?')} has {L} steps; the learner was "
                         f"built for 1..{T} (hp.max_timesteps)")
    if len(traj.obs) != L + 1 or len(traj.a) != L or len(traj.d) != L or len(traj.logits) != L:
        raise ValueError("malformed trajectory: obs must have one more entry than a/r/d/logits")
    return L


def obs_array(traj, obs_dtype) -> np.ndarray:
    """The trajectory's stacked observations in the slab's observation type.  "uint8" takes them only
    when every value is an integer in [0, 255] (Atari RAM bytes, MinAtar planes) and raises ValueError
    otherwise: nothing is truncated or rescaled."""
    if np.dtype(obs_dtype) != np.uint8:
        return _np(torch.stack(traj.obs), torch.float32)
    v = torch.stack(traj.obs).detach().cpu()
    if v.dtype != torch.uint8:
        v = v.to(torch.float64)
        if not bool(((v >= 0) & (v <= 255) & (v == torch.floor(v))).all()):
            raise ValueError(f"trajectory {getattr(traj, 'id', '?')}: uint8 observations must be integers in "
                             "[0, 255] (the values enter the network as they are)")
    return v.to(torch.uint8).numpy()


def obs_frames(obs: np.ndarray, k: int, traj=None) -> np.ndarray:
    """Stacked observations (L+1, k F), oldest frame first -> the trajectory's frames (L+k, F): obs[0] split
    into its k frames, then the newest frame of each obs[t].  Raises ValueError, naming the trajectory and
    the step, where obs[t] does not continue obs[t-1] (obs[t][:(k-1)F] != obs[t-1][F:]): such a trajectory
    cannot be stored once per frame and is refused rather than misaligned."""
    n, O = obs.shape
    F = O // k
    if k > 1 and n > 1:
        bad = np.flatnonzero((obs[1:, :(k - 1) * F] != obs[:-1, F:]).any(axis=1))
        if bad.size:
            raise ValueError(f"trajectory {getattr(traj, 'id', '?')}: observation {int(bad[0]) + 1} does not continue "
                             f"observation {int(bad[0])} as {k} stacked frames (flattened, oldest frame first)")
    return np.concatenate([obs[0].reshape(k, F), obs[1:, (k - 1) * F:]], axis=0)


def gaussian_steps(traj, L: int, A: int):
    """A Gaussian trajectory's actions (L, A) and behaviour outputs (L, 2A) as float32.  Raises ValueError, naming
    the trajectory, for a step of another shape or a non-finite entry: one NaN sample or log std would turn the
    whole update's gradient into NaN (a categorical index cannot)."""
    tid = getattr(traj, "id", "?")
    out = []
    for name, seq, w in (("action", traj.a, A), ("behaviour [mean | log std]", traj.logits, 2 * A)):
        rows = [torch.as_tensor(x) for x in seq]
        bad = next((t for t, x in enumerate(rows) if tuple(x.shape) != (w,)), None)
        if bad is not None:
            raise ValueError(f"trajectory {tid}: step {bad} {name} has shape {tuple(rows[bad].shape)}, "
                             f"a Gaussian policy over {A} dimensions takes ({w},)")
        v = _np(torch.stack(rows), torch.float32) if rows else np.zeros((0, w), np.float32)
        if not np.isfinite(v).all():
            raise ValueError(f"trajectory {tid}: non-finite {name} at step {int(np.argwhere(~np.isfinite(v))[0, 0])}")
        out.append(v)
    return out


def check_gaussian_block(block: dict, T: int, n: int, A: int) -> None:
    """put_block's checks of a Gaussian block: (T, n, A) actions and (T, n, 2A) behaviour outputs, all finite."""
    for name, w in (("actions", A), ("beh_logits", 2 * A)):
        v = np.asarray(block[name])
        if v.shape != (T, n, w):
            raise ValueError(f"Gaussian block {name} of shape {v.shape}; this ring takes {(T, n, w)}")
        if not np.isfinite(v).all():
            raise ValueError(f"Gaussian block: non-finite {name} (column {int(np.argwhere(~np.isfinite(v))[0, 1])})")


def _is_int(x) -> bool:
    return not (x.is_floating_point() or x.is_complex() or x.dtype == torch.bool)


def md_steps(traj, L: int, heads):
    """A multi-discrete trajectory's actions (L, K) int32 and behaviour logits (L, N) float32, N = sum(heads).  Raises
    ValueError, naming the trajectory, the step and the head, for a step of another shape, a non-integer action or
    an index a_k outside [0, n_k): such an index would train the logit of another head's action without an error."""
    tid = getattr(traj, "id", "?")
    K, N = len(heads), sum(heads)
    acts = [torch.as_tensor(x) for x in traj.a]
    logits = [torch.as_tensor(x) for x in traj.logits]
    for t, x in enumerate(acts):
        if tuple(x.shape) != (K,):
            raise ValueError(f"trajectory {tid}: step {t} action has shape {tuple(x.shape)}, a multi-discrete policy "
                             f"of {K} heads takes ({K},)")
        if not _is_int(x):
            raise ValueError(f"trajectory {tid}: step {t} action has dtype {x.dtype}; the head indices must be integers")
    for t, x in enumerate(logits):
        if tuple(x.shape) != (N,):
            raise ValueError(f"trajectory {tid}: step {t} behaviour logits have shape {tuple(x.shape)}, the heads "
                             f"{tuple(heads)} take ({N},)")
    a = torch.stack(acts).to(torch.int64).numpy() if acts else np.zeros((0, K), np.int64)
    bad = np.argwhere((a < 0) | (a >= np.asarray(heads)))
    if bad.size:
        t, k = (int(v) for v in bad[0])
        raise ValueError(f"trajectory {tid}: step {t} head {k} action {int(a[t, k])} is outside [0, {heads[k]})")
    z = _np(torch.stack(logits), torch.float32) if logits else np.zeros((0, N), np.float32)
    return a.astype(np.int32), z


def check_md_block(block: dict, T: int, n: int, heads) -> None:
    """put_block's checks of a multi-discrete block: (T, n, K) integer actions with a_k in [0, n_k) and (T, n, N)
    behaviour logits."""
    K, N = len(heads), sum(heads)
    a, z = np.asarray(block["actions"]), np.asarray(block["beh_logits"])
    if a.shape != (T, n, K):
        raise ValueError(f"multi-discrete block actions of shape {a.shape}; this ring takes {(T, n, K)}")
    if not np.issubdtype(a.dtype, np.integer):
        raise ValueError(f"multi-discrete block actions of dtype {a.dtype}; the head indices must be integers")
    if z.shape != (T, n, N):
        raise ValueError(f"multi-discrete block beh_logits of shape {z.shape}; this ring takes {(T, n, N)}")
    bad = np.argwhere((a < 0) | (a >= np.asarray(heads)))
    if bad.size:
        t, col, k = (int(v) for v in bad[0])
        raise ValueError(f"multi-discrete block: column {col} step {t} head {k} action {int(a[t, col, k])} is outside "
                         f"[0, {heads[k]})")


def _mask_word_errors(m, a, heads):
    """The first problem of legal masks m (L, N) against action indices a (L, K) over `heads` as (step, head, what),
    or None: values other than 0 / 1, a head without a legal entry, an illegal taken action."""
    m = np.asarray(m)
    if m.dtype != bool:
        bad = np.argwhere((m != 0) & (m != 1))
        if bad.size:
            t, j = (int(v) for v in bad[0])
            return t, None, f"mask value {m[t, j]!r} at output {j} is not 0 / 1"
    m = m.astype(bool)
    s = 0
    for k, n in enumerate(heads):
        empty = np.argwhere(~m[:, s:s + n].any(-1))
        if empty.size:
            return int(empty[0, 0]), k, "has no legal action"
        off = np.argwhere(~np.take_along_axis(m[:, s:s + n], a[:, k:k + 1].astype(np.int64), -1)[:, 0])
        if off.size:
            t = int(off[0, 0])
            return t, k, f"action {int(a[t, k])} is illegal under its mask"
        s += n
    return None


def mask_steps(traj, L: int, heads, actions) -> np.ndarray:
    """The (L,) int32 legal words of a masked trajectory: traj.action_mask holds L masks of shape (N,), N = sum(heads)
    (a categorical policy: heads = (A,)), bool or 0 / 1, true meaning legal, as the mask that held when a_t was
    chosen; `actions` (L, K) the indices taken.  Raises ValueError, naming the trajectory, the step and the head, for a
    missing mask, a wrong width, values other than 0 / 1, a head without a legal entry or an illegal taken action."""
    tid = getattr(traj, "id", "?")
    N = sum(heads)
    masks = getattr(traj, "action_mask", None)
    if masks is None or len(masks) != L:
        raise ValueError(f"trajectory {tid}: a masked learner takes one action_mask per step, got "
                         f"{'none' if masks is None else len(masks)} for {L} steps")
    ms = [torch.as_tensor(x) for x in masks]
    for t, x in enumerate(ms):
        if tuple(x.shape) != (N,):
            raise ValueError(f"trajectory {tid}: step {t} action_mask has shape {tuple(x.shape)}, this policy takes "
                             f"({N},)")
    m = torch.stack(ms).numpy() if ms else np.zeros((0, N), bool)
    err = _mask_word_errors(m, np.asarray(actions).reshape(L, len(heads)), heads)
    if err is not None:
        t, k, what = err
        raise ValueError(f"trajectory {tid}: step {t}{'' if k is None else f' head {k}'} {what}")
    from .synth import legal_words

    return legal_words(m.astype(bool))


def check_mask_block(block: dict, T: int, n: int, heads) -> np.ndarray:
    """put_block's checks of a masked block: block["action_mask"] (T, n, N) legal masks against block["actions"]
    ((T, n) categorical, (T, n, K) multi-discrete) over the valid steps of each column; returns the (T, n) int32 legal
    words (0 on padded steps)."""
    N = sum(heads)
    if "action_mask" not in block:
        raise ValueError("a masked ring takes block['action_mask'] of shape (T, n, N)")
    m = np.asarray(block["action_mask"])
    if m.shape != (T, n, N):
        raise ValueError(f"block action_mask of shape {m.shape}; this ring takes {(T, n, N)}")
    a = np.asarray(block["actions"]).reshape(T, n, len(heads))
    lens = np.asarray(block["lens"])
    for col in range(n):
        L = int(lens[col])
        err = _mask_word_errors(m[:L, col], a[:L, col], heads)
        if err is not None:
            t, k, what = err
            raise ValueError(f"masked block: column {col} step {t}{'' if k is None else f' head {k}'} {what}")
    valid = np.arange(T)[:, None] < lens[None, :]
    from .synth import legal_words

    return np.where(valid, legal_words(m.astype(bool)), 0).astype(np.int32)


def pack_trajectory(views: dict, b: int, traj, T: int, obs=None, heads=(), masked: bool = False) -> float:
    """Write one reference-format trajectory into column `b` of a host batch slab.

    Replaces learner.py:104-109,117 (five torch.stack calls + `disc`): float64 -> float32 (or the
    checked uint8 of obs_array for a byte-observation slab), int64 -> int32, bool -> u8, zero padding
    past the trajectory's length.  `obs`: obs_array's result if the caller already has it.  A frame slab
    (obs (T+k, B, F), k > 1) receives obs_frames' L+k frames.  A Gaussian slab (actions (T, B, A)) takes
    (A,) actions and (2A,) behaviour outputs per step (gaussian_steps); a multi-discrete slab (`heads`: the head
    sizes, actions (T, B, K)) (K,) integer actions and (N,) logits (md_steps).  A masked slab (`masked`, actions
    (T, B, 2) or (T, B, K + 1)) takes traj.action_mask as well and stores its legal words last (mask_steps).
    Returns the trajectory's reward sum (learner.py:108)."""
    L = check_trajectory(traj, T)
    multi = bool(heads)
    if multi and tuple(views["actions"].shape[2:]) != (len(heads) + masked,):
        raise ValueError(f"a slab of actions {tuple(views['actions'].shape)} does not hold the heads {tuple(heads)}")
    gauss = views["actions"].ndim == 3 and not multi and not masked
    if gauss:
        act, beh = gaussian_steps(traj, L, views["actions"].shape[2])
    elif multi:
        act, beh = md_steps(traj, L, heads)
    if masked:
        if not multi:
            act = _np(torch.stack(traj.a).reshape(L), torch.int32) if L else np.zeros(0, np.int32)
        words = mask_steps(traj, L, heads or (views["beh_logits"].shape[2],), act)
        act = np.concatenate([act.reshape(L, -1), words[:, None]], -1)
    obs = obs_array(traj, views["obs"].dtype) if obs is None else obs
    k = views["obs"].shape[0] - T
    if k > 1:
        obs = obs_frames(obs, k, traj)
    views["obs"][:L + k, b] = obs
    views["obs"][L + k:, b] = 0
    views["beh_logits"][:L, b] = beh if gauss or multi else _np(torch.stack(traj.logits), torch.float32)
    views["beh_logits"][L:, b] = 0
    views["actions"][:L, b] = act if gauss or multi or masked else _np(torch.stack(traj.a).reshape(L), torch.int32)
    views["actions"][L:, b] = 0
    r = torch.stack(traj.r)
    views["rewards"][:L, b] = _np(r, torch.float32)
    views["rewards"][L:, b] = 0
    views["done"][:L, b] = _np(torch.stack(traj.d), torch.uint8)
    views["done"][L:, b] = 0
    views["lens"][b] = L
    return float(r.sum(dtype=torch.float64))  # summed as received (float64 from actor.py), like learner.py:108


def _dims(policy, value_fn, action_dist):
    """(O, A, H_pi, H_v) of the two modules: A actions (a multi-discrete policy: its N = sum n_k outputs), or the action
    dimensions of a Gaussian policy, whose 2A outputs are [mean | log std]."""
    sd_p, sd_v = policy.state_dict(), value_fn.state_dict()
    H_pi, O = sd_p[PKEYS[0]].shape
    A = int(sd_p[PKEYS[2]].shape[0])
    H_v = sd_v[PKEYS[0]].shape[0]
    if action_dist == "gaussian":
        if A % 2:
            raise ValueError(f"a Gaussian policy has 2A outputs [mean | log std]; this policy has {A}")
        A //= 2
    return int(O), A, int(H_pi), int(H_v)


def _check_ring(q, options, B_fresh: int) -> None:
    """A RingQueue (the queue with `collect_batch`) fills slabs the engine DMAs as they are, so it must hold what the
    options and B_fresh describe.  A plain queue carries reference trajectories, which the learner packs itself."""
    if not hasattr(q, "collect_batch"):
        return
    for want, have, what in ((options.action_dist, q.action_dist, "{} actions"),
                             (tuple(options.action_heads), tuple(getattr(q, "action_heads", ())), "action heads {}"),
                             (options.action_mask, getattr(q, "action_mask", False), "action_mask={}"),
                             (options.obs_dtype, q.obs_dtype, "{} observations"),
                             (options.frames, q.frames, "{} frames per observation"),
                             (B_fresh, q.B, "{} trajectories per update (batch_size - replay_columns)")):
        if want != have:
            raise ValueError(f"the learner takes {what.format(want)}, the RingQueue was built for {what.format(have)}")


class _Publisher:
    """Asynchronous policy-weight publication (SURVEY 8f-2; replaces the per-update full
    state_dict copy behind learner.py:293-295 / actor.py:70).

    post(n): [learner stream] policy block -> device staging buffer (freezes update n's weights
    without stalling the next update), [side stream] staging -> pinned host snapshot; the
    publisher thread waits for that copy and writes the float64 shared tensors under a seqlock.
    Two snapshot slots; publications coalesce when the host cannot keep up with the updates."""

    def __init__(self, eng, policy, version):
        self.eng, self.policy, self.version = eng, policy, version
        n = eng.n_pi
        self.stream = torch.cuda.Stream(device=eng.dev)
        self.stage = [torch.empty(n, dtype=torch.float32, device=eng.dev) for _ in range(2)]
        self.host = [torch.empty(n, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.free = [threading.Event(), threading.Event()]
        for e in self.free:
            e.set()
        # CUDA events of a slot are reused: a slot is posted again only after its previous publication
        # has been written (free[s] set after landed.synchronize())
        self.ev_frozen = [torch.cuda.Event() for _ in range(2)]
        self.ev_landed = [torch.cuda.Event() for _ in range(2)]
        self.views = []  # (flat offset, shared tensor) of the policy's four parameters
        sd = policy.state_dict()
        for grp, key, off, shp in eng._segments():
            if grp == "policy":
                self.views.append((off, int(np.prod(shp)), sd[key]))
        self.q: queue.SimpleQueue = queue.SimpleQueue()
        self.i = 0
        self.published = 0
        self.error = None
        self.thread = threading.Thread(target=self._run, name="impala-publisher", daemon=True)
        self.thread.start()

    def post(self, n: int, force: bool = False) -> bool:
        """Publish the weights of update n.  Coalescing: if the previous publication is still being
        written the call returns False at once (the next one carries newer weights anyway) - the
        actors always see the newest weights the host can deliver, the update loop never waits.
        force=True (evaluation / checkpoint points, last update) waits for a free snapshot slot."""
        s = self.i & 1
        if not self.free[s].is_set():
            if not force:
                return False
            self.free[s].wait()
        self.i += 1
        self.free[s].clear()
        eng = self.eng
        frozen, landed = self.ev_frozen[s], self.ev_landed[s]
        with eng._on_stream():
            # obs_norm: the policy folded into raw-observation coordinates, which the actors feed it
            self.stage[s].copy_((eng.folded if eng.obs_norm else eng.params)[:eng.n_pi], non_blocking=True)
            frozen.record(eng.stream)
        self.stream.wait_event(frozen)
        with torch.cuda.stream(self.stream):
            self.host[s].copy_(self.stage[s], non_blocking=True)
            landed.record(self.stream)
        self.q.put((s, n, landed))
        return True

    def _run(self) -> None:
        try:
            while True:
                item = self.q.get()
                if item is None:
                    return
                s, n, landed = item
                landed.synchronize()
                self._write(self.host[s])
                self.published = n
                self.free[s].set()
        except BaseException as e:  # noqa: BLE001 - surfaced by the learner loop
            self.error = e
            for ev in self.free:
                ev.set()

    def _write(self, flat: torch.Tensor) -> None:
        v = self.version
        with torch.no_grad():
            v.value += 1             # odd: a write is in progress
            for off, cnt, dst in self.views:
                dst.copy_(flat[off:off + cnt].view(dst.shape))  # float32 -> float64, in place
            v.value += 1

    def drain(self) -> None:
        """Block until everything posted so far is in the shared tensors."""
        for e in self.free:
            e.wait()
        if self.error is not None:
            raise self.error

    def close(self) -> None:
        self.q.put(None)
        self.thread.join(timeout=10)


class Learner:
    def __init__(self, id, hparams, policy, value_fn, q, update_counter, log_path=None,
                 timeout=200, device="cuda:0", mode="reference", devices=None, publish_every=1,
                 evaluator=None, lr_lambda=None, **options):
        self.id = id
        self.devices = [str(d) for d in devices] if devices else [str(device)]
        # the options, checked here, in the launching process, as every engine checks them; the schedule is
        # tabulated here (a lambda need not pickle; data-parallel worker ranks receive the table)
        o = self.options = LearnerOptions(**options)
        self.optim = optim_config(hparams, o.optimizer, o.optimizer_kwargs, lr_lambda)
        # experience replay: B_fresh trajectories per update come off the queue, replay_columns out of HBM
        self.B_fresh = o.check(hparams.batch_size, *_dims(policy, value_fn, o.action_dist), len(self.devices)).B_fresh
        _check_ring(q, o, self.B_fresh)
        self.popart_init = None  # {"mu", "nu"} of the folded value_fn (load() of a PopArt checkpoint sets it)
        self.obs_norm_init = None  # {"count", "mean", "var"} the folded first layers go with (obs_norm checkpoints)
        self.hp = hparams
        self.policy = policy
        self.value_fn = value_fn
        self.timeout = timeout
        self.q = q
        self.update_counter = update_counter
        self.device = self.devices[0]
        self.mode = mode
        self.publish_every = max(1, int(publish_every))
        for name, mod in (("policy", policy), ("value_fn", value_fn)):
            if any(p.is_cuda for p in mod.parameters()):
                raise ValueError(
                    f"{name} lives on a CUDA device: the reference's models.py / actor.py pick `cuda` at import "
                    "when a GPU is visible, which initialises CUDA in the launcher (fork start method, "
                    "train.py:42) and makes policy.share_memory() a no-op.  Hide the GPUs from the launcher "
                    "and the actors (CUDA_VISIBLE_DEVICES='' before importing the reference modules; see "
                    "INTEGRATION.md) - this learner restores visibility inside its own process "
                    "(IMPALA_LEARNER_VISIBLE_DEVICES)")
        self.log_path = log_path
        if self.log_path is not None:
            self.log_path = Path(log_path) / Path(f"l{self.id}")
            self.log_path.mkdir(parents=True, exist_ok=False)
        self.evaluator = evaluator  # optional callable(policy) -> (mean_reward, std); see _evaluate
        self._version = mp.Value("q", 0, lock=False)   # published-weights seqlock (shared with the actors)
        self._stage_ring = None
        self.completion = mp.Event()
        self.p = mp.Process(target=self._learn, name=f"learner_{self.id}")
        print(f"[main] learner_{self.id} Initialized")

    # -------------------------------------------------------------- lifecycle (learner.py:55-65)
    def start(self):
        self.completion.clear()
        if len(self.devices) > 1 and not hasattr(self.q, "collect_batch"):
            # data-parallel + reference wire format: rank 0 packs trajectories into a shared-memory
            # staging ring every rank can DMA its shard from (created before the fork)
            from .ring import RingQueue

            c, o = self._cfg(), self.options
            self._stage_ring = RingQueue(self.hp.max_timesteps, self.hp.batch_size, c["O"], c["A"], slabs=2,
                                         obs_dtype=o.obs_dtype, frames=o.frames, action_dist=o.action_dist,
                                         action_heads=o.action_heads, action_mask=o.action_mask)
        self.p.start()
        print(f"[main] Started learner_{self.id} with pid {self.p.pid}")

    def terminate(self):
        self.p.terminate()
        print(f"[main] Terminated learner_{self.id}")

    def join(self):
        self.p.join()
        if self._stage_ring is not None:
            self._stage_ring.close()
            self._stage_ring = None

    # ------------------------------------------------------------------ helpers
    def _cfg(self):
        """The JSON every rank builds its engine from (engine.engine_from_cfg): shapes, mode, hp and the fields of
        LearnerOptions.  The learning-rate table travels apart, in the init-state file (dp.write_init_state)."""
        O, A, H_pi, H_v = _dims(self.policy, self.value_fn, self.options.action_dist)
        hp = self.hp._asdict() if hasattr(self.hp, "_asdict") else dict(self.hp)
        hp["log_path"] = None if hp.get("log_path") is None else str(hp["log_path"])
        # action_heads, action_mask, obs_norm and obs_norm_eps are init-only options (engine.LearnerOptions), so they
        # ride next to the fields
        o = self.options
        return dict(T=self.hp.max_timesteps, B=self.hp.batch_size, O=O, A=A, H_pi=H_pi, H_v=H_v, mode=self.mode, hp=hp,
                    action_heads=list(o.action_heads), action_mask=o.action_mask, obs_norm=o.obs_norm,
                    obs_norm_eps=o.obs_norm_eps,
                    **dataclasses.asdict(self.options))

    def _make_engine(self, process_group=None, world=1):
        eng = engine_from_cfg(self._cfg(), world, self.device, process_group, self.optim.lr_table)
        eng.load_state(self._init_state(), self._popart_init(), self._obs_norm_init())
        return eng

    def _obs_norm_init(self):
        """The observation statistics the folded modules go with: those of a loaded checkpoint, else None (fresh)."""
        return dict(self.obs_norm_init) if self.options.obs_norm and self.obs_norm_init is not None else None

    def _popart_init(self):
        """The statistics the folded value_fn goes with: those of a loaded checkpoint, else None (mu 0, nu 1)."""
        return dict(self.popart_init) if self.options.popart and self.popart_init is not None else None

    def _init_state(self):
        return {"policy": {k: v.detach().cpu() for k, v in self.policy.state_dict().items()},
                "value_fn": {k: v.detach().cpu() for k, v in self.value_fn.state_dict().items()}}

    def _sync_modules(self, eng, pub):
        """Blocking: everything published so far is visible AND both float64 modules hold the current
        weights (checkpoints, end of run).  The per-update path is `_Publisher.post`."""
        pub.drain()
        st = eng.state()  # the value function folded into reward units under PopArt
        if self.options.popart:
            s = eng.popart_stats()
            self.popart_init = {"mu": s["mu"], "nu": s["nu"]}  # what save() writes next to the folded value_fn
        if self.options.obs_norm:
            self.obs_norm_init = eng.obs_norm_stats()  # what save() writes next to the folded first layers
        with torch.no_grad():
            self._version.value += 1
            for mod, grp in ((self.policy, "policy"), (self.value_fn, "value_fn")):
                for k, t in mod.state_dict().items():
                    t.copy_(st[grp][k].to(t.dtype))
            self._version.value += 1

    @property
    def policy_version(self) -> int:
        """Even: number of completed weight publications x 2; odd: a publication is in progress."""
        return int(self._version.value)

    def policy_snapshot(self):
        """(version, state_dict copy) that is guaranteed not to be torn by a concurrent publication
        (seqlock read; `policy_weights` keeps the reference's lock-free semantics, actor.py:70)."""
        while True:
            v0 = self._version.value
            if v0 & 1:
                continue
            sd = {k: t.clone() for k, t in self.policy.state_dict().items()}
            if self._version.value == v0:
                return v0, sd

    def _evaluate(self, policy):
        """learner.py:195-214 runs utils.test_policy (a gym rollout) inside the update loop.  Here it
        runs on a frozen copy in a background thread: `self.evaluator` if set, else the reference's
        own `utils.test_policy` when this class is deployed inside that repo."""
        if self.evaluator is not None:
            return self.evaluator(policy)
        if self.options.action_dist == "gaussian":  # the reference's test_policy refuses continuous environments
            print(f"[learner_{self.id}] evaluation skipped: a Gaussian policy is evaluated through evaluator= only")
            return None
        if self.options.action_dist == "multi_discrete":  # test_policy steps one Discrete index per action
            print(f"[learner_{self.id}] evaluation skipped: a multi-discrete policy is evaluated through evaluator= only")
            return None
        if self.options.action_mask:  # test_policy steps the environment without its legal-action masks
            print(f"[learner_{self.id}] evaluation skipped: a masked policy is evaluated through evaluator= only")
            return None
        try:
            import utils as ref_utils  # the reference's utils.py, if on sys.path

            return ref_utils.test_policy(policy, self.hp.env_name, self.hp.eval_eps, True, self.hp.max_timesteps)
        except Exception as e:  # no gym / not inside the reference tree
            print(f"[learner_{self.id}] evaluation skipped: {e!r}")
            return None

    def _start_evaluation(self, writer, n):
        """Evaluate the weights of update n without blocking update n + 1."""
        prev = getattr(self, "_eval_thread", None)
        if prev is not None and prev.is_alive():
            print(f"[learner_{self.id}] update {n}: previous evaluation still running - skipped")
            return
        _, sd = self.policy_snapshot()
        frozen = copy.deepcopy(self.policy)
        frozen.load_state_dict(sd)

        def work():
            res = self._evaluate(frozen)
            if res is None:
                return
            if self.hp.verbose >= 1:
                print(f"[learner_{self.id}] update {n}: evaluation reward {res[0]:.2f} +- {res[1]:.2f}")
            if writer is not None:
                writer.add_scalar(f"learner_{self.id}/rewards/evaluation_reward", res[0], n)

        self._eval_thread = threading.Thread(target=work, name="impala-eval", daemon=True)
        self._eval_thread.start()

    # ---------------------------------------------------------------- the update loop
    def _collect(self, views, writer):
        """Pull hp.batch_size trajectories (B_fresh of them with replay) off the queue into one host slab
        (learner.py:89-109)."""
        hp = self.hp
        reward = 0.0
        for b in range(self.B_fresh):
            try:
                traj = self.q.get(timeout=self.timeout)
            except queue.Empty:
                print(f"[learner_{self.id}] queue empty for {self.timeout} s - giving up")
                if writer is not None:
                    writer.close()
                self.completion.set()  # lets the actors leave their put() retry loop (actor.py:121)
                raise
            if hp.verbose >= 2:
                print(f"[learner_{self.id}] packing traj_{traj.id} into column {b}")
            reward += pack_trajectory(views, b, traj, hp.max_timesteps, heads=self.options.action_heads,
                                      masked=self.options.action_mask) / self.B_fresh
            del traj  # drop the shared-memory handles of its ~5T tensors right away
        return reward

    def _report(self, writer, n, reward, sc):
        """Console line + the five TensorBoard scalars of learner.py:188-192,217-240 (+ the off-policy
        diagnostics when they are on)."""
        if self.hp.verbose >= 1:
            diag = (f", rho clipped {100.0 * sc['rho_clip_fraction']:.1f} %, kl {sc['kl_behaviour_current']:.4f}"
                    if self.options.diagnostics else "")
            print(f"[learner_{self.id}] update {n}: batch mean reward {reward:.2f}, "
                  f"loss {sc['total_loss']:.2f}{diag}")
        if writer is None:
            return
        tag = f"learner_{self.id}"
        for name, val in (("rewards/batch_mean_reward", reward), ("loss/policy_loss", sc["policy_loss"]),
                          ("loss/value_fn_loss", sc["value_fn_loss"]),
                          ("loss/policy_entropy", sc["policy_entropy"]),
                          ("loss/total_loss", sc["total_loss"])):
            writer.add_scalar(f"{tag}/{name}", val, n)
        if self.options.diagnostics:
            for name in ("log_ratio_mean", "rho_clip_fraction", "c_clip_fraction", "kl_behaviour_current"):
                writer.add_scalar(f"{tag}/offpolicy/{name}", sc[name], n)
            writer.add_scalar(f"{tag}/value/explained_variance", sc["value_explained_variance"], n)
        if self.options.popart:
            writer.add_scalar(f"{tag}/popart/mu", sc["popart_mu"], n)
            writer.add_scalar(f"{tag}/popart/sigma", sc["popart_sigma"], n)

    def _due(self, n) -> bool:
        hp = self.hp
        return ((hp.eval_every is not None and n % hp.eval_every == 0)
                or (self.log_path is not None and n % hp.save_every == 0))

    def _periodic(self, writer, n, eng, pub):
        hp = self.hp
        if hp.eval_every is not None and n % hp.eval_every == 0:          # learner.py:195-214
            pub.drain()
            self._start_evaluation(writer, n)
        if self.log_path is not None and n % hp.save_every == 0:          # learner.py:243-251
            self._sync_modules(eng, pub)
            path = self.log_path / f"IMPALA_{hp.env_name}_l{self.id}_{n}.pt"
            self.save(path)
            print(f"[learner_{self.id}] checkpoint -> {path}")

    def _restore_gpu_visibility(self):
        """The launcher may have hidden the GPUs so that the reference's import-time device choice
        stays on the CPU (see __init__); the learner process gets them back before its first CUDA call."""
        import os

        vis = os.environ.get("IMPALA_LEARNER_VISIBLE_DEVICES")
        if vis is not None:
            os.environ["CUDA_VISIBLE_DEVICES"] = vis

    def _learn(self):
        """Process target (learner.py:67): loop until the shared counter reaches max_updates."""
        writer, pub, leader, eng = None, None, None, None
        try:
            import os

            if os.environ.get("IMPALA_DEBUG_STACKS"):  # dump every thread's stack if the process is still alive then
                import faulthandler

                faulthandler.dump_traceback_later(float(os.environ["IMPALA_DEBUG_STACKS"]), repeat=True, file=sys.stderr)
            # The forked child inherits the launcher's OpenMP state without its worker threads: the first
            # multi-threaded CPU op (e.g. zero-filling a multi-megabyte pinned slab) would wait forever
            # for them.  The learner's host work is tiny copies; one intra-op thread is also the fastest.
            torch.set_num_threads(1)
            self._restore_gpu_visibility()
            world = len(self.devices)
            ring = self.q if hasattr(self.q, "collect_batch") else None  # ring.RingQueue (SURVEY 8f-1)
            stage = self._stage_ring  # data-parallel + mp.Queue: shared staging slabs filled by this process
            pg = None
            if world > 1:
                from . import dp

                slabs = ring if ring is not None else stage
                leader = dp.DpLeader(self.devices, self._cfg(), self._init_state(), slabs.shm.name,
                                     slabs.slab_bytes, slabs.K, timeout=max(60.0, float(self.timeout)),
                                     lr_table=self.optim.lr_table, popart=self._popart_init(),
                                     obs_norm=self._obs_norm_init())
                torch.cuda.set_device(torch.device(self.device))
                pg = leader.init_process_group(self.device)
            eng = self._make_engine(pg, world)  # first CUDA call of this process (post-fork)
            pub = _Publisher(eng, self.policy, self._version)
            if self.log_path is not None:
                from torch.utils.tensorboard import SummaryWriter

                writer = SummaryWriter(self.log_path)
                writer.add_text("hyperparameters", f"{self.hp}")
            shared = ring if ring is not None else stage
            if shared is not None:
                if world == 1 and shared.slab_bytes != eng.slab_bytes:
                    raise ValueError("RingQueue and learner disagree on (T, B, obs, actions)")
                eng.register_host(shared.slab_address(0), shared.slab_bytes * shared.K)
            if leader is not None:
                leader.wait_ready()
            done, slot, pending, stage_k = 0, 0, None, 0
            eng.loop_stream(True)  # this thread's current stream is the engine's for the whole loop
            # IMPALA_LOOP_STATS=1: where the host time of the update loop goes (printed at the end)
            stats = {"release_wait": 0.0, "collect": 0.0, "enqueue": 0.0, "post": 0.0, "finish": 0.0} \
                if os.environ.get("IMPALA_LOOP_STATS") else None
            clock = time.perf_counter
            to_release = []  # (DMA-done event, ring slab): released one iteration later, off the critical path
            while done < self.hp.max_updates:
                # ---- batch i: collect (host), DMA (copy stream) - the kernels of batch i-1 are running
                # a slab goes back to the actors when its DMA has completed.  Do not WAIT for that here
                # unless the ring would otherwise run dry (or both device slabs' events are in use): the
                # next batch is collected and its DMA queued right behind the running one, so the copy
                # engine never idles for the host part of an iteration (IMPALA_LOOP_STATS=1 shows how long
                # an update still waits here)
                t0 = clock()
                while to_release:
                    ev, kk = to_release[0]
                    if not ev.query() and len(to_release) < min(ring.K - 1, 2):
                        break
                    ev.synchronize()
                    ring.release(kk)
                    to_release.pop(0)
                t1 = clock()
                if ring is not None:
                    try:
                        k, reward = ring.collect_batch(self.timeout)
                    except queue.Empty:
                        print(f"[learner_{self.id}] no trajectory for {self.timeout} s - giving up")
                        self.completion.set()
                        raise
                elif stage is not None:
                    k, stage_k = stage_k, (stage_k + 1) % stage.K
                    reward = self._collect(stage.views(k), writer)
                else:
                    k = None
                    reward = self._collect(eng.host_batch(slot), writer)
                t2 = clock()
                if world > 1:
                    step_no = leader.publish(k)                       # every rank: DMA your shard of slab k
                    eng.ingest_shard_from(shared.slab_address(k), 0, self.hp.batch_size, slot)
                    eng.slab_ready[slot].synchronize()
                    leader.ack_dma(0, step_no)
                    leader.wait_dma(step_no)
                    if ring is not None:
                        ring.release(k)
                elif ring is not None:
                    eng.ingest_from(ring.slab_address(k), slot)   # DMA straight out of shared memory
                    to_release.append((eng.slab_ready[slot], k))  # handed back to the actors once the DMA is done
                else:
                    eng.ingest(slot)
                eng.step(slot)
                t3 = clock()
                n = done + 1
                # the logged scalars: read back when somebody consumes them (TensorBoard / console), else
                # every 64th update (keeps the data-parallel error word checked)
                want_scalars = writer is not None or self.hp.verbose >= 1 or n % 64 == 0 or n >= self.hp.max_updates
                ticket = eng.post_scalars() if want_scalars else None
                due = self._due(n)  # evaluation / checkpoint of exactly update n
                if due and ticket is None:
                    ticket = eng.post_scalars()
                if due or n % self.publish_every == 0 or n >= self.hp.max_updates:
                    pub.post(n, force=due or n >= self.hp.max_updates)
                if pub.error is not None:
                    raise pub.error
                t4 = clock()
                # ---- while update n runs: log update n - 1
                if pending is not None:
                    self._finish_update(writer, eng, pub, *pending)
                    pending = None
                if due:
                    self._finish_update(writer, eng, pub, ticket, n, reward)  # waits for update n
                else:
                    pending = (ticket, n, reward)
                slot ^= 1
                self.update_counter.increment()                            # learner.py:254-255
                done = self.update_counter.value
                if stats is not None:
                    t5 = clock()
                    for key, dt in (("release_wait", t1 - t0), ("collect", t2 - t1), ("enqueue", t3 - t2),
                                    ("post", t4 - t3), ("finish", t5 - t4)):
                        stats[key] += dt
            if stats is not None:
                print(f"[learner_{self.id}] host time per update (us): "
                      + ", ".join(f"{k} {1e6 * v / max(1, done):.1f}" for k, v in stats.items()), file=sys.stderr, flush=True)
            if pending is not None:
                self._finish_update(writer, eng, pub, *pending)
            self._sync_modules(eng, pub)
            t = getattr(self, "_eval_thread", None)
            if t is not None:
                t.join(timeout=600)
            print(f"[learner_{self.id}] done after {done} updates")
            self.completion.set()
        except KeyboardInterrupt:
            print(f"[learner_{self.id}] interrupted")
            self.completion.set()
        except Exception:
            # The reference re-raises without setting `completion` (learner.py:271-275), which
            # leaves train.py:84 waiting forever; here the actors are released as well.
            print(f"[learner_{self.id}] failed")
            self.completion.set()
            raise
        finally:
            if pub is not None:
                pub.close()
            if leader is not None:
                leader.stop()
            if writer is not None:
                writer.close()

    def _finish_update(self, writer, eng, pub, ticket, n, reward):
        if ticket is not None:
            sc = eng.fetch_scalars(ticket)
            self._report(writer, n, reward, sc)
        if writer is not None and not self.optim.is_default:  # the rate update n used
            writer.add_scalar(f"learner_{self.id}/optim/lr", eng.lr_of(n), n)
        self._periodic(writer, n, eng, pub)

    # ------------------------------------------------------ checkpoints (learner.py:277-295)
    def save(self, path):
        """Reference checkpoint keys.  Shared torso: the two state dicts are the policy and value views of the one
        network (both hold the torso) and "shared_torso" is True; the policy view is an MlpPolicy state dict."""
        ckpt = {"policy_state_dict": self.policy.state_dict(), "value_fn_state_dict": self.value_fn.state_dict()}
        if self.options.shared_torso:
            ckpt["shared_torso"] = True
        if self.options.popart:  # value_fn is folded (reward units); the statistics that unfold it
            ckpt["popart"] = dict(self.popart_init or {"mu": 0.0, "nu": 1.0})
        if self.options.obs_norm:  # the first layers are folded (raw observations); the statistics that unfold them
            O = _dims(self.policy, self.value_fn, self.options.action_dist)[0]
            st = self.obs_norm_init or {"count": 0.0, "mean": np.zeros(O), "var": np.ones(O)}
            ckpt["obs_norm"] = {"count": float(st["count"]), "mean": torch.tensor(np.asarray(st["mean"], np.float64)),
                                "var": torch.tensor(np.asarray(st["var"], np.float64))}
        torch.save(ckpt, path)

    def load(self, path):
        """Restores a checkpoint of either kind into the two modules.  A shared-torso learner builds its network
        from the policy's torso and heads and the value function's head (engine.load_state), so a two-network
        checkpoint starts it from the policy's torso."""
        checkpoint = torch.load(path)
        self.policy.load_state_dict(checkpoint["policy_state_dict"])
        self.value_fn.load_state_dict(checkpoint["value_fn_state_dict"])
        if "popart" in checkpoint:
            self.popart_init = {k: float(checkpoint["popart"][k]) for k in ("mu", "nu")}
        if "obs_norm" in checkpoint:
            st = checkpoint["obs_norm"]
            self.obs_norm_init = {"count": float(st["count"]),
                                  **{k: np.asarray(torch.as_tensor(st[k]), np.float64) for k in ("mean", "var")}}

    @property
    def policy_weights(self):
        return self.policy.state_dict()


# ----------------------------------------------------------------------------------------------
# Module-level loss helpers with the reference's names, signatures and sign conventions
# (learner.py:298-321), backed by the C ABI.  Inputs are CUDA tensors (any float dtype; the
# kernels compute in float32 and reduce in float64); results come back in the input dtype and
# are differentiable with respect to the logits / advantages exactly where the reference's are.
# ----------------------------------------------------------------------------------------------
def _lib_and_stream():
    import ctypes as C

    from . import _cabi

    return _cabi, _cabi.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream), C


def _cuda_f32(t):
    from . import _cabi

    if not (torch.is_tensor(t) and t.is_cuda):
        raise _cabi.ImpalaCudaError("loss helpers need CUDA tensors (there is no CPU fallback)")
    return t.detach().to(torch.float32).contiguous()


class _PolicyTerms(torch.autograd.Function):
    """(logits, actions) -> (log pi(a), sum_k p_k log p_k) per row."""

    @staticmethod
    def forward(ctx, logits, actions):
        _cabi, lib, st, C = _lib_and_stream()
        z = _cuda_f32(logits).reshape(-1, logits.shape[-1])
        a = actions.detach().reshape(-1).to(torch.int32).contiguous()
        M, A = z.shape
        lp = torch.empty(M, dtype=torch.float32, device=z.device)
        ne = torch.empty(M, dtype=torch.float32, device=z.device)
        _cabi.check(lib.impala_policy_terms(C.c_void_p(z.data_ptr()), C.c_void_p(a.data_ptr()),
                                            C.c_void_p(lp.data_ptr()), C.c_void_p(ne.data_ptr()), M, A, st),
                    "impala_policy_terms")
        ctx.save_for_backward(z, a)
        ctx.in_shape, ctx.in_dtype = logits.shape, logits.dtype
        return lp.to(logits.dtype), ne.to(logits.dtype)

    @staticmethod
    def backward(ctx, g_lp, g_ne):
        _cabi, lib, st, C = _lib_and_stream()
        z, a = ctx.saved_tensors
        M, A = z.shape
        gl = None if g_lp is None else g_lp.to(torch.float32).contiguous()
        gn = None if g_ne is None else g_ne.to(torch.float32).contiguous()
        dz = torch.empty_like(z)
        _cabi.check(lib.impala_policy_terms_backward(
            C.c_void_p(z.data_ptr()), C.c_void_p(a.data_ptr()),
            C.c_void_p(gl.data_ptr()) if gl is not None else None,
            C.c_void_p(gn.data_ptr()) if gn is not None else None,
            C.c_void_p(dz.data_ptr()), M, A, st), "impala_policy_terms_backward")
        return dz.reshape(ctx.in_shape).to(ctx.in_dtype), None


class _Reduce(torch.autograd.Function):
    """float64-accumulated scalar reductions: mode 0 sum(a), 1 0.5*sum(a^2), 2 sum(a*b) (b constant)."""

    @staticmethod
    def forward(ctx, a, b, mode):
        _cabi, lib, st, C = _lib_and_stream()
        af = _cuda_f32(a).reshape(-1)
        bf = _cuda_f32(b).reshape(-1) if b is not None else None
        out = torch.empty(1, dtype=torch.float64, device=af.device)
        _cabi.check(lib.impala_reduce(C.c_void_p(af.data_ptr()),
                                      C.c_void_p(bf.data_ptr()) if bf is not None else None,
                                      af.numel(), mode, C.c_void_p(out.data_ptr()), st), "impala_reduce")
        ctx.mode, ctx.shape, ctx.dtype = mode, a.shape, a.dtype
        ctx.save_for_backward(af, bf if bf is not None else af)
        return out[0].to(a.dtype)

    @staticmethod
    def backward(ctx, g):
        af, bf = ctx.saved_tensors
        if ctx.mode == 0:
            ga = g.to(torch.float32).expand(af.shape)
        elif ctx.mode == 1:
            ga = g.to(torch.float32) * af
        else:
            ga = g.to(torch.float32) * bf
        return ga.reshape(ctx.shape).to(ctx.dtype), None, None


def action_log_probs(policy_logits, actions):
    """log pi(a|x) of the taken actions, shaped like `actions` (learner.py:298-303)."""
    return _PolicyTerms.apply(policy_logits, actions)[0].view_as(actions)


def compute_baseline_loss(advantages):
    """0.5 * sum(advantages ** 2)  (learner.py:306-307)."""
    return _Reduce.apply(advantages, None, 1)


def compute_entropy_loss(logits):
    """The NEGATIVE entropy sum(p * log p), as in the reference (learner.py:310-314)."""
    return _Reduce.apply(_PolicyTerms.apply(logits, torch.zeros(logits.shape[:-1], dtype=torch.int32,
                                                                 device=logits.device))[1], None, 0)


def compute_policy_gradient_loss(logits, actions, advantages):
    """sum(-log pi(a|x) * advantages.detach())  (learner.py:317-321)."""
    lp = _PolicyTerms.apply(logits, actions)[0]
    return _Reduce.apply(lp, -advantages.detach().reshape(-1), 2)
