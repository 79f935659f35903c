"""torchrun target: N-rank sharded learner steps with PopArt.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_popart_check.py

Every rank builds the engine with popart=True from the same folded value function and statistics (through the
peer push, or the NCCL all-reduce under IMPALA_ALLREDUCE=nccl); the replicas' parameters, optimizer state and
statistics must stay bit-identical, and rank 0 compares with a single-GPU engine of the same configuration on
the full batch (float32 sum order differs -> ~1e-6, as tests/multi_gpu_check.py).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, B, O, A, H = 20, 512, 24, 4, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=4)
    kw = dict(popart=True, popart_beta=0.2)
    stats = {"mu": 0.5, "nu": 4.0}
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(10 + u, T, B, O, A, ragged=(u % 2 == 1)) for u in range(5)]
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, **kw)
    eng.load_state(params, stats)
    for u, b in enumerate(batches):
        eng.fill_host(synth.shard_batch(b, rank, world), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        eng.read_scalars()
    mine = torch.cat([eng.params, eng.adam_m, eng.adam_v]).detach().double()
    mine = torch.cat([mine, eng.popart_buf]).clone()
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    for g in gathered:
        assert torch.equal(g, gathered[0]), "ranks diverged"
    if rank == 0:
        ref = LearnerEngine(T, B, O, A, H, H, hp, device=f"cuda:{local}", **kw)
        ref.load_state(params, stats)
        for u, b in enumerate(batches):
            ref.fill_host(b, u % 2)
            ref.ingest(u % 2)
            ref.step(u % 2)
        ref.synchronize()
        d = (eng.params - ref.params).abs().max().item()
        assert d < 2e-5, d
        s0, s1 = eng.popart_stats(), ref.popart_stats()
        for k in ("mu", "nu"):
            assert abs(s0[k] - s1[k]) <= 1e-6 * max(1.0, abs(s1[k])), (k, s0, s1)
        assert s0["mu"] != stats["mu"]
        mode = ("peer(fused)" if eng.peer["fused"] else "peer(standalone)") if eng.peer else "nccl"
        print(f"MULTI_GPU_POPART_OK world={world} allreduce={mode} max|dparam|={d:.2e} mu={s0['mu']:.5f}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
