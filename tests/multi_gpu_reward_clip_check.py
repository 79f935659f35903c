"""torchrun target: N-rank sharded learner steps with reward clipping.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_reward_clip_check.py

Every rank builds the engine with reward_clip="abs_one" (and diagnostics, so the clipped-unit sums ride the
exchange too) and trains on its shard of raw-reward batches (through the peer push, or the NCCL all-reduce under
IMPALA_ALLREDUCE=nccl).  The first step's loss scalars must match the float64 oracle on the full batch, with
batch_mean_reward the raw mean; the replicas' parameters and optimizer state must stay bit-identical; rank 0
compares with a single-GPU engine of the same configuration on the full batch (float32 sum order differs ->
~1e-6, as tests/multi_gpu_check.py).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import reward_clip_oracle as rorc  # noqa: E402
from conftest import PKEYS  # noqa: E402
from oracle import impala_oracle as orc  # noqa: E402
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, B, O, A, H = 20, 512, 24, 4, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=4)
    kw = dict(reward_clip="abs_one", diagnostics=True)
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(10 + u, T, B, O, A, ragged=(u % 2 == 1)) for u in range(5)]
    for b in batches:
        b["rewards"] = b["rewards"] * np.float32(3.0)
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, **kw)
    eng.load_state(params)
    for u, b in enumerate(batches):
        eng.fill_host(synth.shard_batch(b, rank, world), u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        sc = eng.read_scalars()
        if u == 0:  # the first step against the float64 oracle on the full batch
            obs = b["obs"].astype(np.float64)
            f64 = {g: [np.asarray(params[g][k], np.float64) for k in PKEYS] for g in ("policy", "value_fn")}
            logits, _ = orc.mlp_forward(obs[:-1], *f64["policy"])
            v = orc.mlp_forward(obs, *f64["value_fn"])[0][..., 0]
            want = rorc.vtrace_loss(v, logits, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], hp,
                                    B, "abs_one")
            for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
                assert abs(sc[k] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, sc[k], want[k])
    mine = torch.cat([eng.params, eng.adam_m, eng.adam_v]).detach().double().clone()
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
        assert d < 2e-5, d
        mode = ("peer(fused)" if eng.peer["fused"] else "peer(standalone)") if eng.peer else "nccl"
        print(f"MULTI_GPU_REWARD_CLIP_OK world={world} allreduce={mode} max|dparam|={d:.2e}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
