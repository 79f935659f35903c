"""Shared-memory trajectory ring: SURVEY.md section 8(f)-1, the first "next" row after the hot path.

The reference ships every trajectory through `mp.Queue` as ~5T+1 separately pickled tiny tensors
(one file descriptor each, `utils.py:48-77`, `actor.py:116-124`): about 52 ms per trajectory at
the consumer and an fd-exhaustion failure mode (SURVEY section 6).  `RingQueue` keeps the queue
interface the unmodified `actor.py` uses (`q.put(traj, timeout=...)`, `queue.Full`), but nothing
travels through a pipe any more - payload AND bookkeeping live in one
`multiprocessing.shared_memory` segment:

  * K batch slabs, each in exactly the learner's device layout (time-major, float32,
    `impala_batch_layout` offsets);
  * a control block: one "column filled" byte, the reward sum and the trajectory id per
    (slab, column), a release counter per slab, and the next ticket number.

`put()` runs in the ACTOR process: under a lock it takes the next ticket n (slab (n // B) % K,
column n % B; only once the learner has released that slab often enough), packs the trajectory
straight into that column with the same `pack_trajectory` the learner uses, and sets the column's
byte.  The learner polls B bytes per batch - no per-trajectory message, no pickling - and, with a
GPU, registers the segment with `cudaHostRegister` once and DMAs each finished slab to the device
directly (no second host copy).

`train.py` changes one line (`q = RingQueue(...)` instead of `mp.Queue(...)`); `Learner` detects
the ring by its `collect_batch` method and otherwise speaks the reference wire format.
"""
from __future__ import annotations

import queue
import threading
import time
from multiprocessing import shared_memory

import numpy as np
import torch.multiprocessing as mp

_FIELDS = (("obs", np.float32), ("beh_logits", np.float32), ("actions", np.int32),
           ("rewards", np.float32), ("done", np.uint8), ("lens", np.int32))
_POLL_S = 2e-4      # back-off sleep once a wait has lasted longer than _SPIN_S
_SPIN_S = 2e-3      # busy-poll this long first: a sleep costs >= 60 us of scheduler latency per batch


def _pause(t_start: float) -> None:
    """Wait policy of the ring's polling loops: spin (yielding the GIL) while the wait is young."""
    if time.monotonic() - t_start < _SPIN_S:
        time.sleep(0)
    else:
        time.sleep(_POLL_S)


_OBS_BYTES = {"float32": 4, "uint8": 1}


_ACT_DISTS = ("categorical", "gaussian", "multi_discrete")


def _layout(T: int, B: int, O: int, A: int, obs_dtype: str = "float32", frames: int = 1,
            action_dist: str = "categorical", action_heads=(), action_mask: bool = False):
    """Same 256-byte aligned layout as include/impala_b200.h::impala_batch_layout_act with F = O / frames
    (impala_batch_layout_obs at frames = 1, categorical; pure python so actor processes do not need the CUDA
    library).  "gaussian": beh_logits (T, B, 2A) f32 and actions (T, B, A) f32 for A action dimensions.
    "multi_discrete": beh_logits (T, B, A) f32 for A = sum(action_heads) outputs and actions (T, B, K) i32.
    action_mask=True (categorical, multi_discrete): one more int32 per step in the actions, the legal word."""
    if action_dist not in _ACT_DISTS:
        raise ValueError(f"action_dist must be one of {list(_ACT_DISTS)}, got {action_dist!r}")
    g = action_dist == "gaussian"
    K = len(action_heads) if action_dist == "multi_discrete" else 1
    if obs_dtype not in _OBS_BYTES:
        raise ValueError(f"obs_dtype must be one of {sorted(_OBS_BYTES)}, got {obs_dtype!r}")
    if frames < 1 or O % frames:
        raise ValueError(f"{O} observation features do not split into {frames} frames")
    sizes = ((T + frames) * B * (O // frames) * _OBS_BYTES[obs_dtype], T * B * (2 * A if g else A) * 4,
             T * B * (A if g else K + bool(action_mask)) * 4, T * B * 4, T * B, B * 4)
    offs, off = [], 0
    for s in sizes:
        offs.append(off)
        off = (off + s + 255) // 256 * 256
    return offs, off


class RingQueue:
    """Drop-in for the `mp.Queue` between actors and learner, backed by shared-memory batch slabs."""

    def __init__(self, T: int, B: int, O: int, A: int, slabs: int = 3, obs_dtype: str = "float32", frames: int = 1,
                 action_dist: str = "categorical", action_heads=(), action_mask: bool = False):
        if slabs < 2:
            raise ValueError("need at least two slabs (one filling while one is consumed)")
        if action_dist == "gaussian" and not 1 <= A <= 16:
            raise ValueError(f"a Gaussian policy takes 1 to 16 action dimensions, got {A}")
        # "multi_discrete": K heads of action_heads[k] actions, A = sum(action_heads) outputs; K int32 indices per step
        if action_dist == "multi_discrete":
            from ._cabi import check_heads  # pure python: no library load

            action_heads = check_heads(action_heads)
            if sum(action_heads) != A:
                raise ValueError(f"the heads {action_heads} have {sum(action_heads)} outputs; this ring takes A = {A}")
        elif tuple(action_heads) != ():
            raise ValueError(f"action_heads is for action_dist='multi_discrete', not {action_dist!r}")
        self.action_heads = tuple(action_heads)
        # action_mask: the actors' legal-action masks (traj.action_mask, block["action_mask"]) travel as one int32
        # legal word per step after the action indices
        if not isinstance(action_mask, bool):
            raise ValueError(f"action_mask must be a bool, got {action_mask!r}")
        if action_mask and (action_dist == "gaussian" or A > 32):
            raise ValueError("action_mask is for categorical and multi-discrete policies of at most 32 outputs")
        self.action_mask = action_mask
        self.T, self.B, self.O, self.A, self.K = T, B, O, A, slabs
        # "uint8": byte observations (Atari RAM, MinAtar planes), a quarter of the float32 slab bytes
        self.offsets, self.slab_bytes = _layout(T, B, O, A, obs_dtype, frames, action_dist, self.action_heads,
                                                action_mask)
        # "gaussian": A action dimensions; the actors' [mean | log std] (2A) and float32 samples (A) per step
        self.action_dist = action_dist
        self.gaussian = action_dist == "gaussian"
        self.obs_dtype = obs_dtype
        # frames > 1: observations are `frames` stacked frames of O / frames features, each frame stored once
        # per column, (T + frames, B, O / frames); the learner rebuilds the stacked rows on the device
        self.frames = frames
        self._fields = (("obs", np.dtype(obs_dtype).type),) + _FIELDS[1:]
        if self.gaussian:
            self._fields = self._fields[:2] + (("actions", np.float32),) + self._fields[3:]
        # control block after the slabs: filled u8[K][B] | rsum f64[K][B] | tid i64[K][B] |
        # released i64[K] | next_ticket i64[1]   (8-byte aligned pieces)
        kb = slabs * B
        self._ctl_off = self.slab_bytes * slabs
        self._ctl = {"filled": (0, np.uint8, (slabs, B))}
        off = (kb + 7) // 8 * 8
        for name, dt, shape in (("rsum", np.float64, (slabs, B)), ("tid", np.int64, (slabs, B)),
                                ("released", np.int64, (slabs,)), ("ticket", np.int64, (1,))):
            self._ctl[name] = (off, dt, shape)
            off += int(np.prod(shape)) * 8
        self.shm = shared_memory.SharedMemory(create=True, size=self._ctl_off + off)
        self._owner = True
        self._lock = mp.Lock()          # serialises ticket allocation between actors
        self._views = None
        self._c = None
        self._fence = threading.Lock()  # acquire/release = a full memory fence on every platform
        self._next = 0
        self.ids = [np.full(B, -1, np.int64) for _ in range(slabs)]  # trajectory id per (slab, column), for logs; -1 = none
        c = self._control()
        c["filled"][:] = 0
        c["released"][:] = 0
        c["ticket"][0] = 0

    # ---- pickling: child processes attach to the same segment by name
    def __getstate__(self):
        d = self.__dict__.copy()
        d["_views"] = d["_c"] = None
        d["_owner"] = False
        d["shm_name"] = self.shm.name
        del d["shm"], d["_fence"]
        return d

    def __setstate__(self, d):
        name = d.pop("shm_name")
        self.__dict__.update(d)
        self._fence = threading.Lock()
        self.shm = shared_memory.SharedMemory(name=name)

    def _control(self) -> dict:
        if self._c is None:
            self._c = {name: np.ndarray(shape, dtype=dt, buffer=self.shm.buf, offset=self._ctl_off + off)
                       for name, (off, dt, shape) in self._ctl.items()}
        return self._c

    def views(self, k: int) -> dict:
        """Numpy views of slab k (the six batch tensors, learner layout)."""
        if self._views is None:
            N = 2 * self.A if self.gaussian else self.A
            Ka = (len(self.action_heads) or 1) + 1 if self.action_mask else len(self.action_heads)  # indices, legal word
            shapes = {"obs": (self.T + self.frames, self.B, self.O // self.frames), "beh_logits": (self.T, self.B, N),
                      "actions": ((self.T, self.B, self.A) if self.gaussian else
                                  (self.T, self.B, Ka) if Ka else (self.T, self.B)),
                      "rewards": (self.T, self.B), "done": (self.T, self.B), "lens": (self.B,)}
            self._views = []
            for kk in range(self.K):
                base = kk * self.slab_bytes
                self._views.append({name: np.ndarray(shapes[name], dtype=dt, buffer=self.shm.buf, offset=base + off)
                                    for (name, dt), off in zip(self._fields, self.offsets)})
        return self._views[k]

    def slab_address(self, k: int) -> int:
        """Address of slab k in THIS process (for cudaHostRegister / impala_ingest)."""
        return np.ndarray((1,), dtype=np.uint8, buffer=self.shm.buf, offset=k * self.slab_bytes).ctypes.data

    def _barrier(self) -> None:
        with self._fence:
            pass

    # ---- actor side (same call shape as mp.Queue.put used at actor.py:118)
    def put(self, traj, block: bool = True, timeout: float | None = None):
        from .learner import check_trajectory, obs_array, pack_trajectory

        check_trajectory(traj, self.T)  # BEFORE a column is taken: a malformed trajectory must not leave a hole
        obs = obs_array(traj, self.obs_dtype)  # the same: raises on obs a uint8 ring cannot hold
        if self.action_heads:  # the same: wrong widths, non-integer or out-of-range head indices
            from .learner import md_steps

            md_steps(traj, len(traj.r), self.action_heads)
        if self.action_mask:  # the same: missing, malformed or empty masks, illegal taken actions
            from .learner import mask_steps, md_steps

            L = len(traj.r)
            a = (md_steps(traj, L, self.action_heads)[0] if self.action_heads else
                 np.asarray([int(np.asarray(x).reshape(-1)[0]) for x in traj.a], np.int64).reshape(L, 1))
            mask_steps(traj, L, self.action_heads or (self.A,), a)
        c = self._control()
        end = None if (timeout is None or not block) else time.monotonic() + timeout
        t_wait = time.monotonic()
        while True:
            with self._lock:
                n = int(c["ticket"][0])
                k, b, gen = (n // self.B) % self.K, n % self.B, n // (self.B * self.K)
                if int(c["released"][k]) >= gen:  # the learner has handed slab k out `gen` times
                    c["ticket"][0] = n + 1
                    break
            if not block or (end is not None and time.monotonic() >= end):
                raise queue.Full  # like mp.Queue.put on a full queue; actor.py:120 retries
            _pause(t_wait)
        try:
            rsum = pack_trajectory(self.views(k), b, traj, self.T, obs=obs, heads=self.action_heads,
                                   masked=self.action_mask)
        except BaseException:
            # never leave the column unfilled (the learner would stall on it until its timeout):
            # publish it as an empty trajectory - neutral padding for the update - and re-raise
            v = self.views(k)
            for name in ("obs", "beh_logits", "actions", "rewards", "done"):
                v[name][:, b] = 0
            v["lens"][b] = 0
            c["rsum"][k, b] = 0.0
            c["tid"][k, b] = -1
            self._barrier()
            c["filled"][k, b] = 1
            raise
        tid = getattr(traj, "id", None)
        c["rsum"][k, b] = rsum
        c["tid"][k, b] = int(tid) if isinstance(tid, (int, np.integer)) else -1
        self._barrier()  # payload before the flag
        c["filled"][k, b] = 1

    def put_block(self, block: dict, block_rsum=None, timeout: float | None = None) -> None:
        """Pre-stacked payload (SURVEY section 7: synthetic actors push stacked arrays through the same
        queue): `block` holds n trajectories in the learner layout - obs (T+1, n, O) f32 (frames
        (T+frames, n, O/frames) on a frame ring), beh_logits
        (T, n, A) f32, actions (T, n) i32, rewards (T, n) f32, done (T, n) u8, lens (n,) i32 - and is
        copied into n consecutive columns of the slab being filled (n must divide B, so a block never
        straddles two slabs).  One lock round trip and five strided copies per block instead of
        ~5T tiny tensors per trajectory."""
        n = int(block["lens"].shape[0])
        if n < 1 or self.B % n:
            raise ValueError(f"block of {n} trajectories: n must divide the batch size {self.B}")
        if self.obs_dtype == "uint8" and np.asarray(block["obs"]).dtype != np.uint8:
            raise ValueError(f"a uint8-observation ring takes uint8 obs blocks, got {np.asarray(block['obs']).dtype}")
        want = (self.T + self.frames, n, self.O // self.frames)
        if self.frames > 1 and tuple(np.shape(block["obs"])) != want:
            raise ValueError(f"obs block of shape {tuple(np.shape(block['obs']))}; this ring takes {want}")
        if self.gaussian:
            from .learner import check_gaussian_block

            check_gaussian_block(block, self.T, n, self.A)
        if self.action_heads:
            from .learner import check_md_block

            check_md_block(block, self.T, n, self.action_heads)
        words = None
        if self.action_mask:
            from .learner import check_mask_block

            words = check_mask_block(block, self.T, n, self.action_heads or (self.A,))
        c = self._control()
        end = None if timeout is None else time.monotonic() + timeout
        t_wait = time.monotonic()
        while True:
            with self._lock:
                t0 = int(c["ticket"][0])
                k, b, gen = (t0 // self.B) % self.K, t0 % self.B, t0 // (self.B * self.K)
                if b % n == 0 and int(c["released"][k]) >= gen:
                    c["ticket"][0] = t0 + n
                    break
                if b % n:  # trajectory-wise writers left a partial block: skip to the next aligned column
                    raise ValueError("put_block cannot be mixed with put on the same ring at unaligned columns")
            if end is not None and time.monotonic() >= end:
                raise queue.Full
            _pause(t_wait)
        v = self.views(k)
        for name in ("obs", "beh_logits", "rewards", "done"):
            v[name][:, b:b + n] = block[name]
        if words is None:
            v["actions"][:, b:b + n] = block["actions"]
        else:  # the indices, then the legal word
            v["actions"][:, b:b + n, :-1] = np.asarray(block["actions"]).reshape(self.T, n, -1)
            v["actions"][:, b:b + n, -1] = words
        v["lens"][b:b + n] = block["lens"]
        rs = block["rewards"].sum(0, dtype=np.float64) if block_rsum is None else block_rsum
        c["rsum"][k, b:b + n] = rs
        c["tid"][k, b:b + n] = -1
        self._barrier()  # payload before the flags
        c["filled"][k, b:b + n] = 1

    # ---- learner side
    def collect_batch(self, timeout: float | None = None):
        """Blocks until the next slab (in round-robin order) has all B columns; returns
        (slab index, batch-mean reward).  Raises queue.Empty when no new trajectory has arrived
        for `timeout` seconds, like `mp.Queue.get` does for the reference learner
        (learner.py:91-100)."""
        c, k = self._control(), self._next
        seen, last = -1, time.monotonic()
        while True:
            n = int(np.count_nonzero(c["filled"][k]))
            if n == self.B:
                break
            now = time.monotonic()
            if n != seen:
                seen, last = n, now
            elif timeout is not None and now - last >= timeout:
                raise queue.Empty
            _pause(last)
        self._barrier()  # flags before the payload reads
        reward = float(c["rsum"][k].sum()) / self.B
        self.ids[k] = c["tid"][k].copy()  # one vector copy - a python loop over B columns costs more than the DMA
        self._next = (k + 1) % self.K
        return k, reward

    def release(self, k: int) -> None:
        """The learner is done with slab k (its DMA has completed): hand its columns out again."""
        c = self._control()
        c["filled"][k] = 0
        self._barrier()
        c["released"][k] += 1

    def close(self):
        try:
            self._views = self._c = None
            self.shm.close()
            if self._owner:
                self.shm.unlink()
        except (FileNotFoundError, BufferError):
            pass


def wait_until(pred, timeout: float, poll: float = 0.01) -> bool:
    end = time.time() + timeout
    while time.time() < end:
        if pred():
            return True
        time.sleep(poll)
    return pred()
