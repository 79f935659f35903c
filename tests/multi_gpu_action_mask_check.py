"""torchrun target: N-rank sharded learner steps of a masked multi-discrete-policy engine.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_action_mask_check.py

Every rank builds LearnerEngine(action_dist="multi_discrete", action_heads=(3, 3, 2, 2, 5, 5), action_mask=True,
diagnostics=True) and pulls its shard of a full-batch host slab with ingest_shard_from (impala_ingest_shard_act: K
int32 indices and the legal word per step), then trains through the peer push at N = 20 policy outputs (or the NCCL
all-reduce under IMPALA_ALLREDUCE=nccl).  The first step's loss scalars must match the float64 oracle on
the full batch; the replicas' parameters and optimizer state must stay bit-identical; rank 0 compares with a
single-GPU engine on the full batch (float32 sum order differs -> ~1e-6).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import action_mask_oracle as aorc  # noqa: E402
from oracle import impala_oracle as orc  # noqa: E402
from torched_impala_b200 import _cabi, synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, B, O, heads, H = 20, 512, 28, (3, 3, 2, 2, 5, 5), 256
    A = sum(heads)
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=4, rho_bar=1.0, c_bar=0.9)
    kw = dict(action_dist="multi_discrete", action_heads=heads, action_mask=True, diagnostics=True)
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_masked_batch(10 + u, T, B, O, A, heads, density=0.5, ragged=(u % 2 == 1), params=params)
               for u in range(4)]
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, **kw)
    eng.load_state(params)
    offs, nbytes = _cabi.batch_layout(T, B, O, A, "float32", 1, "multi_discrete", heads, True)
    host = torch.zeros(nbytes, dtype=torch.uint8).pin_memory()
    arr = host.numpy()
    for u, b in enumerate(batches):
        for (name, _), off in zip(eng.fields, offs):
            v = np.ascontiguousarray(b[name])
            arr[off:off + v.nbytes] = v.view(np.uint8).reshape(-1)
        eng.ingest_shard_from(host.data_ptr(), rank * (B // world), B, u % 2)
        eng.step(u % 2)
        sc = eng.read_scalars()
        eng.synchronize()  # the host slab is rewritten for the next update
        if u == 0:  # the first step against the float64 oracle on the full batch
            lo, hi = rank * (B // world), (rank + 1) * (B // world)
            assert np.array_equal(eng.d["actions"].cpu().numpy(), b["actions"][:, lo:hi])
            obs = b["obs"].astype(np.float64)
            f64 = {g: [np.asarray(params[g][k], np.float64) for k in orc.PKEYS] for g in ("policy", "value_fn")}
            z = orc.mlp_forward(obs[:-1], *f64["policy"])[0]
            v = orc.mlp_forward(obs, *f64["value_fn"])[0][..., 0]
            want = aorc.vtrace_loss(v, z, b["beh_logits"], b["actions"][..., :-1], b["legal"], b["rewards"], b["done"],
                                    b["lens"], hp, B, heads)
            for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
                assert abs(sc[k] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, sc[k], want[k])
            assert sc["valid_steps"] == want["diag"][0]
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
        print(f"MULTI_GPU_MASK_OK world={world} allreduce={mode} max|dparam|={d:.2e}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
