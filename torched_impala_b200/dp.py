"""Data-parallel learner behind ONE `Learner` object: one process per GPU of an NVLink node.

SURVEY 8e / reference `train.py:69`, `learner.py:52`: the launcher creates exactly one learner.
With `Learner(..., devices=["cuda:0", ..., "cuda:N-1"])` that learner process is rank 0 of an
N-rank group: after the fork it starts N - 1 worker processes (fresh interpreters,
`python -m torched_impala_b200.dp_worker`), every rank builds a `LearnerEngine` on its own GPU
with the global batch size, and per update

  * rank 0 waits for a complete batch slab in host shared memory (the `RingQueue` the actors fill,
    or the staging ring rank 0 packs `mp.Queue` trajectories into) and publishes its index in a
    small shared-memory control block;
  * EVERY rank DMAs its own contiguous B/N column range of that slab to its own GPU over its own
    PCIe link (`impala_ingest_shard`, strided 2-D copies out of the registered segment) and
    acknowledges the DMA, so rank 0 can hand the slab back to the actors;
  * every rank enqueues the same captured step; the gradient exchange is the push all-reduce of
    engine.py / csrc/optim.cu; replicas stay bit-identical;
  * rank 0 alone reads the logged scalars and publishes policy weights to the actors.

The control block is a handful of int64 words polled by the workers (they own a core each, like
the actors); nothing is pickled per update.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import tempfile
import time
from multiprocessing import shared_memory

import numpy as np

# control block layout (int64 words)
_CMD, _SLAB, _STOP, _ERR = 0, 1, 2, 3
_DMA_ACK, _STEP_ACK, _READY = 8, 16, 24   # + rank (<= 8 ranks each)
_WORDS = 32
_POLL_S = 2e-5


_OWNED: set = set()  # segments created by THIS process (their tracker registration must stay)


def attach_untracked(name: str) -> shared_memory.SharedMemory:
    """Attach to an existing segment WITHOUT registering it with this interpreter's resource tracker
    (Python < 3.13 registers on attach and would unlink the owner's segment when a worker exits)."""
    shm = shared_memory.SharedMemory(name=name)
    if shm.name in _OWNED:
        return shm
    try:
        from multiprocessing import resource_tracker

        resource_tracker.unregister(shm._name, "shared_memory")  # noqa: SLF001
    except Exception:  # noqa: BLE001
        pass
    return shm


class ShardControl:
    """int64[32] in shared memory: command word, slab index, stop/error flags, per-rank acks."""

    def __init__(self, name: str | None = None):
        if name is None:
            self.shm = shared_memory.SharedMemory(create=True, size=_WORDS * 8)
            _OWNED.add(self.shm.name)
            self.owner = True
        else:
            self.shm = attach_untracked(name)
            self.owner = False
        self.w = np.ndarray((_WORDS,), dtype=np.int64, buffer=self.shm.buf)
        if self.owner:
            self.w[:] = 0

    @property
    def name(self) -> str:
        return self.shm.name

    def close(self):
        try:
            self.w = None
            self.shm.close()
            if self.owner:
                self.shm.unlink()
        except (FileNotFoundError, BufferError):
            pass


def free_port() -> int:
    import socket

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _wait(pred, timeout: float, what: str, ctl: ShardControl | None = None):
    end = time.monotonic() + timeout
    while not pred():
        if ctl is not None and ctl.w[_ERR]:
            raise RuntimeError(f"data-parallel learner: a rank reported an error while waiting for {what}")
        if time.monotonic() > end:
            raise TimeoutError(f"data-parallel learner: timed out after {timeout:.0f} s waiting for {what}")
        time.sleep(_POLL_S)


LR_TABLE_KEY = "optim/lr_table"  # init_state.npz entry of the learning-rate table (absent: the default)


def write_init_state(path: str, init_state: dict, lr_table=None, popart=None, obs_norm=None) -> None:
    """The worker ranks' start: both networks' parameters and the learning-rate table (tabulated on rank 0: a
    lambda need not pickle, and a command-line argument is capped at 128 KiB on Linux).  popart = {"mu", "nu"}:
    the PopArt statistics the (folded) value function goes with, read back as state["popart"]; obs_norm =
    {"count", "mean", "var"}: the observation statistics the (folded) first layers go with, as state["obs_norm"]."""
    arrays = {f"{g}/{k}": np.asarray(v) for g, d in init_state.items() for k, v in d.items()}
    if lr_table is not None:
        arrays[LR_TABLE_KEY] = np.asarray(lr_table, np.float32)
    if popart is not None:
        arrays["popart/mu"], arrays["popart/nu"] = np.float64(popart["mu"]), np.float64(popart["nu"])
    if obs_norm is not None:
        for k in ("count", "mean", "var"):
            arrays[f"obs_norm/{k}"] = np.asarray(obs_norm[k], np.float64)
    np.savez(path, **arrays)


def read_init_state(path: str):
    """(state, lr_table or None) from the init_state.npz DpLeader writes."""
    z = np.load(path)
    state, table = {"policy": {}, "value_fn": {}}, None
    for key in z.files:
        if key == LR_TABLE_KEY:
            table = z[key]
            continue
        g, k = key.split("/", 1)
        state.setdefault(g, {})[k] = z[key]  # "popart", "obs_norm": the statistics, when written
    return state, table


class DpLeader:
    """Rank 0's handle on the worker ranks (lives inside the learner process, post-fork)."""

    def __init__(self, devices, cfg: dict, init_state: dict, slab_shm_name: str, slab_bytes: int,
                 n_slabs: int, timeout: float = 200.0, lr_table=None, popart=None, obs_norm=None):
        self.world = len(devices)
        self.devices = list(devices)
        self.timeout = timeout
        self.ctl = ShardControl()
        self.port = free_port()
        self.step_no = 0
        self._tmp = tempfile.mkdtemp(prefix="impala_dp_")
        state_path = os.path.join(self._tmp, "init_state.npz")
        write_init_state(state_path, init_state, lr_table, popart, obs_norm)
        self.procs = []
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        for r in range(1, self.world):
            spec = dict(rank=r, world=self.world, device=str(devices[r]), port=self.port, cfg=cfg,
                        state=state_path, ctl=self.ctl.name, slab_shm=slab_shm_name, slab_bytes=slab_bytes,
                        n_slabs=n_slabs, parent=os.getpid())
            env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
            for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT"):
                env.pop(k, None)
            self.procs.append(subprocess.Popen([sys.executable, "-m", "torched_impala_b200.dp_worker", json.dumps(spec)],
                                               env=env))

    def init_process_group(self, device):
        import torch
        import torch.distributed as dist

        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{self.port}", rank=0, world_size=self.world,
                                device_id=torch.device(device))
        return dist.group.WORLD

    def wait_ready(self):
        _wait(lambda: all(self.ctl.w[_READY + r] for r in range(1, self.world)) or self._dead(), self.timeout,
              "the worker ranks to build their engines", self.ctl)
        if self._dead():
            raise RuntimeError("data-parallel learner: a worker rank exited during start-up")

    def _dead(self) -> bool:
        return any(p.poll() is not None for p in self.procs)

    def publish(self, slab: int) -> int:
        """Tell every rank that batch slab `slab` is complete; returns the step number."""
        self.step_no += 1
        self.ctl.w[_SLAB] = slab
        self.ctl.w[_CMD] = self.step_no   # after the slab word (x86 store order; numpy stores are plain)
        return self.step_no

    def ack_dma(self, rank: int, step: int):
        self.ctl.w[_DMA_ACK + rank] = step

    def wait_dma(self, step: int):
        """All ranks have copied their shard of the slab of `step` (the slab can go back to the actors)."""
        _wait(lambda: all(self.ctl.w[_DMA_ACK + r] >= step for r in range(self.world)) or self._dead(),
              self.timeout, f"the shard DMAs of step {step}", self.ctl)
        if self._dead():
            raise RuntimeError("data-parallel learner: a worker rank died")

    def stop(self):
        try:
            self.ctl.w[_STOP] = 1
            for p in self.procs:
                try:
                    p.wait(timeout=30)
                except subprocess.TimeoutExpired:
                    p.kill()
        finally:
            self.ctl.close()
            try:
                import shutil

                shutil.rmtree(self._tmp, ignore_errors=True)
            except Exception:  # noqa: BLE001
                pass
