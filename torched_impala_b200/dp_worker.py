"""Worker rank (1..N-1) of the data-parallel learner; started by dp.DpLeader.

    python -m torched_impala_b200.dp_worker '<json spec>'

Builds the same `LearnerEngine` as rank 0 on its own GPU, maps the actors' shared-memory batch
slabs, then follows rank 0's commands: for every published step it DMAs its B/N column range of
the named slab to its GPU, acknowledges the DMA and enqueues the step (whose gradient exchange is
the push all-reduce).  Exits when rank 0 sets the stop word or disappears.
"""
from __future__ import annotations

import json
import os
import sys
import time
import numpy as np


def main():
    spec = json.loads(sys.argv[1])
    import torch
    import torch.distributed as dist

    from . import dp
    from .engine import engine_from_cfg

    rank, world, dev = spec["rank"], spec["world"], spec["device"]
    ctl = dp.ShardControl(spec["ctl"])
    try:
        torch.cuda.set_device(torch.device(dev))
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{spec['port']}", rank=rank, world_size=world,
                                device_id=torch.device(dev))
        c = spec["cfg"]
        state, lr_table = dp.read_init_state(spec["state"])
        eng = engine_from_cfg(c, world, dev, dist.group.WORLD, lr_table)
        popart = state.pop("popart", None)  # rank 0's statistics: every rank starts identical
        obs_norm = state.pop("obs_norm", None)
        eng.load_state(state, {k: float(v) for k, v in popart.items()} if popart else None, obs_norm)
        shm = dp.attach_untracked(spec["slab_shm"])
        base = np.ndarray((1,), dtype=np.uint8, buffer=shm.buf).ctypes.data
        eng.register_host(base, spec["slab_bytes"] * spec["n_slabs"])
        ctl.w[dp._READY + rank] = 1
        last, b0 = 0, rank * (c["B"] // world)
        while True:
            while ctl.w[dp._CMD] <= last and not ctl.w[dp._STOP]:
                if os.getppid() != spec["parent"]:
                    return  # the learner process is gone
                time.sleep(dp._POLL_S)
            if ctl.w[dp._CMD] <= last:
                break  # stop without a new command
            last += 1
            k, slot = int(ctl.w[dp._SLAB]), last & 1
            eng.ingest_shard_from(base + k * spec["slab_bytes"], b0, c["B"], slot)
            eng.slab_ready[slot].synchronize()
            ctl.w[dp._DMA_ACK + rank] = last
            eng.step(slot)
        eng.synchronize()
        dist.destroy_process_group()
    except BaseException:
        ctl.w[dp._ERR] = 1
        raise
    finally:
        ctl.close()


if __name__ == "__main__":
    main()
