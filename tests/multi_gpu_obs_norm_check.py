"""torchrun target: N-rank sharded learner steps with observation normalization.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_obs_norm_check.py

Every rank builds the engine with obs_norm=True from the same folded networks and statistics; the observation sums
ride `comm` (the peer push, or the NCCL all-reduce under IMPALA_ALLREDUCE=nccl).  The replicas' parameters,
optimizer state, statistics and folded blocks must stay bit-identical, and rank 0 compares with a single-GPU engine
of the same configuration on the full batch: parameters to 1e-5 (float32 sum order differs), statistics to 1e-12.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import numpy as np  # noqa: E402

from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, B, O, A, H = 20, 512, 24, 4, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=4)
    kw = dict(obs_norm=True)
    stats = {"count": 1000.0, "mean": np.linspace(-2.0, 3.0, O), "var": np.linspace(0.5, 4.0, O)}
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(10 + u, T, B, O, A, ragged=(u % 2 == 1)) for u in range(5)]
    for u, b in enumerate(batches):
        b["obs"] = (b["obs"] * np.linspace(0.1, 10.0, O) + np.linspace(-50.0, 50.0, O)).astype(np.float32)
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, **kw)
    eng.load_state(params, obs_norm=stats)
    for u, b in enumerate(batches):
        eng.fill_host(synth.shard_batch(b, rank, world), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        eng.read_scalars()
    mine = torch.cat([eng.params, eng.adam_m, eng.adam_v]).detach().double()
    mine = torch.cat([mine, eng.obs_stats, eng.folded.double()]).clone()
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    for g in gathered:
        assert torch.equal(g, gathered[0]), "ranks diverged"
    if rank == 0:
        ref = LearnerEngine(T, B, O, A, H, H, hp, device=f"cuda:{local}", **kw)
        ref.load_state(params, obs_norm=stats)
        for u, b in enumerate(batches):
            ref.fill_host(b, u % 2)
            ref.ingest(u % 2)
            ref.step(u % 2)
        ref.synchronize()
        d = (eng.params - ref.params).abs().max().item()
        assert d < 1e-5, d
        s0, s1 = eng.obs_norm_stats(), ref.obs_norm_stats()
        assert s0["count"] == s1["count"] == stats["count"] + sum(int(b["lens"].sum()) for b in batches)
        for k in ("mean", "var"):
            np.testing.assert_allclose(s0[k], s1[k], rtol=1e-12, atol=0, err_msg=k)
        mode = ("peer(fused)" if eng.peer["fused"] else "peer(standalone)") if eng.peer else "nccl"
        print(f"MULTI_GPU_OBS_NORM_OK world={world} allreduce={mode} max|dparam|={d:.2e} count={s0['count']:.0f}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
