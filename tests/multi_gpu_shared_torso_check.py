"""torchrun target: N-rank sharded learner steps of a shared-torso engine.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_shared_torso_check.py

Every rank builds LearnerEngine(shared_torso=True, diagnostics=True, popart=True) and pulls its shard of a
full-batch host slab with ingest_shard_from, then trains through the flat-gradient push after
impala_mlp_backward_shared (or the NCCL all-reduce under IMPALA_ALLREDUCE=nccl).  The first step's loss scalars
and PopArt statistics must match the float64 oracle on the full batch; the replicas' parameters and optimizer state
must stay bit-identical; rank 0 compares with a single-GPU engine on the full batch.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import shared_torso_oracle as sorc  # noqa: E402
from torched_impala_b200 import _cabi, synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, B, O, A, H = 20, 512, 24, 4, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=4, rho_bar=1.0, c_bar=0.9)
    kw = dict(shared_torso=True, diagnostics=True, popart=True, popart_beta=0.1)
    params = synth.init_params(3, O, A, H)
    batches = [synth.make_batch(10 + u, T, B, O, A, ragged=(u % 2 == 1)) for u in range(4)]
    eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=f"cuda:{local}",
                        process_group=dist.group.WORLD, **kw)
    eng.load_state(params)
    assert not (eng.peer and eng.peer["fused"])  # the fused push is the paired backward's
    offs, nbytes = _cabi.batch_layout(T, B, O, A)
    host = torch.zeros(nbytes, dtype=torch.uint8).pin_memory()
    arr = host.numpy()
    lrn = sorc.SharedLearner(params, hp, popart=True, beta=0.1)
    for u, b in enumerate(batches):
        for (name, _), off in zip(eng.fields, offs):
            v = np.ascontiguousarray(b[name])
            arr[off:off + v.nbytes] = v.view(np.uint8).reshape(-1)
        eng.ingest_shard_from(host.data_ptr(), rank * (B // world), B, u % 2)
        eng.step(u % 2)
        sc = eng.read_scalars()
        eng.synchronize()  # the host slab is rewritten for the next update
        if u == 0:  # the first step against the float64 oracle on the full batch
            want = lrn.update(b)
            for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward"):
                assert abs(sc[k] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, sc[k], want[k])
            assert abs(sc["norm_policy"] - want["norm_policy"]) <= 5e-5 * want["norm_policy"]
            assert sc["norm_value"] == 0.0
            st = eng.popart_stats()
            assert abs(st["mu"] - lrn.mu) < 1e-5 and abs(st["nu"] - lrn.nu) < 1e-5, (st, lrn.mu, lrn.nu)
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
        print(f"MULTI_GPU_SHARED_OK world={world} allreduce={mode} max|dparam|={d:.2e}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
