"""Experience replay, the host side that needs no CUDA: argument checks and the sampling plan.

With `replay_slabs = R` and `replay_columns = Br`, update n (1-based) trains on B = Bf + Br columns: columns
[0, Bf) are its own fresh trajectories, every column j in [Bf, B) is a copy of column c_j of the fresh batch of
update u_j, with (u_j, c_j) drawn independently and uniformly, with replacement, from
{max(1, n - R) .. n - 1} x [0, Bf).  The fresh batch of update u lives in store slot u mod (R + 2): R slots are
the pool, one holds the batch being trained on and one receives the next batch while that happens.
"""
from __future__ import annotations

import numpy as np


def check_replay_args(batch_size: int, replay_slabs: int, replay_columns: int) -> int:
    """Validate the two replay arguments against the batch size; returns Bf, the fresh columns per update
    (batch_size when replay is off: both arguments 0)."""
    R, Br = int(replay_slabs), int(replay_columns)
    if R == 0 and Br == 0:
        return int(batch_size)
    if R < 1 or Br < 1:
        raise ValueError(f"replay_slabs and replay_columns are both 0 (off) or both positive, got "
                         f"replay_slabs={replay_slabs}, replay_columns={replay_columns}")
    if Br >= batch_size:
        raise ValueError(f"replay_columns={Br} must leave fresh columns in a batch of {batch_size}")
    return int(batch_size) - Br


class ReplaySampler:
    """plan(n): the (B, 2) int32 array of (store slot, column) that update n trains on.  A pure function of
    (seed, n), so any process can recompute the plan of any update."""

    def __init__(self, seed: int, replay_slabs: int, fresh_columns: int, replay_columns: int):
        if min(replay_slabs, fresh_columns, replay_columns) < 1:
            raise ValueError(f"a sampler needs replay_slabs, fresh_columns, replay_columns >= 1, got "
                             f"{replay_slabs}, {fresh_columns}, {replay_columns}")
        self.seed, self.R, self.Bf, self.Br = int(seed), int(replay_slabs), int(fresh_columns), int(replay_columns)
        self.slots = self.R + 2

    def sources(self, n: int):
        """(updates, columns) of the Br replayed columns of update n; two empty arrays at update 1."""
        if n < 1:
            raise ValueError(f"updates are numbered from 1, got {n}")
        pool = min(self.R, n - 1)
        if pool == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.int64)
        rng = np.random.default_rng([self.seed, n])
        return n - 1 - rng.integers(0, pool, self.Br), rng.integers(0, self.Bf, self.Br)

    def plan(self, n: int) -> np.ndarray:
        plan = np.empty((self.Bf + self.Br, 2), np.int32)
        plan[:self.Bf, 0] = n % self.slots
        plan[:self.Bf, 1] = np.arange(self.Bf)
        u, c = self.sources(n)
        if u.size:
            plan[self.Bf:, 0], plan[self.Bf:, 1] = u % self.slots, c
        else:  # nothing to replay yet: empty columns
            plan[self.Bf:] = (-1, 0)
        return plan
