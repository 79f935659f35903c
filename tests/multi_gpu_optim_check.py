"""torchrun target: N-rank sharded learner steps with RMSprop and a learning-rate schedule.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_optim_check.py

Every rank builds the engine with optimizer="rmsprop" and a linear schedule (through the peer push, or the NCCL
all-reduce under IMPALA_ALLREDUCE=nccl); the replicas must stay bit-identical, and rank 0 compares with a
single-GPU engine of the same configuration on the full batch (float32 sum order differs -> ~1e-6, as
tests/multi_gpu_check.py).
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
    kw = dict(optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01, momentum=0.9), lr_lambda=lambda e: 1.0 - e / 4)
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(10 + u, T, B, O, A, ragged=(u % 2 == 1)) for u in range(5)]
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, **kw)
    eng.load_state(params)
    for u, b in enumerate(batches):  # past the table's end
        eng.fill_host(synth.shard_batch(b, rank, world), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        eng.read_scalars()
    mine = torch.cat([eng.params, eng.adam_m, eng.adam_v]).detach().clone()
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    for g in gathered:
        assert torch.equal(g, gathered[0]), "ranks diverged"
    if rank == 0:
        ref = LearnerEngine(T, B, O, A, H, H, hp, device=f"cuda:{local}", **kw)
        ref.load_state(params)
        for u, b in enumerate(batches):
            ref.fill_host(b, u % 2)
            ref.ingest(u % 2)
            ref.step(u % 2)
        ref.synchronize()
        d = (eng.params - ref.params).abs().max().item()
        # RMSprop moves every entry by up to ~lr / sqrt(1 - alpha) per step whatever the gradient's size, so the
        # tolerance of the Adam check (2e-5) is scaled by the steps' magnitude rather than kept absolute
        assert d < 2e-5 * max(1.0, 10 * hp.lr * len(batches) / 1e-3), d
        mode = ("peer(fused)" if eng.peer["fused"] else "peer(standalone)") if eng.peer else "nccl"
        print(f"MULTI_GPU_OPTIM_OK world={world} allreduce={mode} max|dparam|={d:.2e}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
