"""torchrun target: the off-policy sums of N-rank sharded steps (diagnostics=True) vs one full-batch GPU.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_diag_check.py

The eight sums ride the all-reduce with the loss scalars (push or IMPALA_ALLREDUCE=nccl): counts must
equal the single-GPU full-batch counts exactly, float sums to 1e-9 relative, replicas stay bit-identical.
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


def sums(eng):
    eng.synchronize()
    return eng.comm[eng.n_total + 4:eng.n_total + 12].cpu().tolist()


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, B, O, A, H = 20, 512, 24, 4, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=0.9, c_bar=0.8)
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(10 + u, T, B, O, A, ragged=(u == 1)) for u in range(3)]
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, diagnostics=True)
    eng.load_state(params)
    got = []
    for u, b in enumerate(batches):
        eng.fill_host(synth.shard_batch(b, rank, world), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        got.append(sums(eng))
    mine = eng.params.detach().clone()
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    for g in gathered:
        assert torch.equal(g, gathered[0]), "ranks diverged"
    if rank == 0:
        ref = LearnerEngine(T, B, O, A, H, H, hp, device=f"cuda:{local}", diagnostics=True)
        ref.load_state(params)
        for u, b in enumerate(batches):
            ref.fill_host(b, u % 2)
            ref.ingest(u % 2)
            ref.step(u % 2)
            want = sums(ref)
            for i in (0, 2, 3):  # n and the clip counts
                assert got[u][i] == want[i], (u, i, got[u][i], want[i])
            for i in (1, 4, 5, 6, 7):
                assert abs(got[u][i] - want[i]) <= 1e-9 * max(1.0, abs(want[i])), (u, i, got[u][i], want[i])
        path = ('peer(fused)' if eng.peer['fused'] else 'peer(standalone)') if eng.peer else 'nccl'
        print(f"MULTI_GPU_DIAG_OK world={world} allreduce={path} n={got[-1][0]:.0f} rho_clipped={got[-1][2]:.0f}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
