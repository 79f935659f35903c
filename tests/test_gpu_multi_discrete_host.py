"""GPU: multi-discrete policies beyond the kernel - uint8 frames=4 slabs equal to the dense engine, a forked Learner
behind a multi-discrete RingQueue against the float64 oracle learner, and two GPUs (peer push and NCCL)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import impala_oracle as orc
from torched_impala_b200 import synth
from torched_impala_b200.engine import LearnerEngine
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu


def test_u8_frames_equal_dense():
    """uint8 frames=4 multi-discrete slabs train bit for bit as the dense uint8 engine on the unstacked rows
    (MinAtar-like 0/1 planes; the behaviour is the policy's own output on those observations)."""
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    T, B, F, k, heads, H = 20, 256, 64, 4, (3, 3, 2, 2, 5, 5), 256
    O, N = F * k, sum(heads)
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    kw = dict(action_dist="multi_discrete", action_heads=heads, obs_dtype="uint8")
    fr = LearnerEngine(T, B, O, N, H, H, hp, frames=k, **kw)
    dn = LearnerEngine(T, B, O, N, H, H, hp, **kw)
    params = synth.init_params(6, O, N, H)
    for e in (fr, dn):
        e.load_state(params)
    for u in range(3):
        b = synth.make_md_batch(90 + u, T, B, O, heads, ragged=True, params=params, obs_kind="planes", frames=k)
        for e, bb in ((fr, b), (dn, synth.stack_frames(b, k))):
            e.fill_host(bb, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
        sf, sd = fr.read_scalars(), dn.read_scalars()
        assert all(np.isfinite(v) for v in sf.values()), sf
        assert sf == sd, (u, sf, sd)
    fr.synchronize()
    dn.synchronize()
    for name in ("params", "adam_m", "adam_v"):
        assert torch.equal(getattr(fr, name), getattr(dn, name)), name


def test_forked_learner(tmp_path):
    """A forked Learner behind a multi-discrete RingQueue, fed synthetic actors, ends within tolerance of the float64
    oracle learner run on the same batches."""
    import md_learner_process_check as chk

    out = tmp_path / "weights.npz"
    res = subprocess.run([sys.executable, chk.__file__, str(tmp_path / "logs"), str(out)], capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MD_LEARNER_OK" in res.stdout
    got = np.load(out)
    want = chk.oracle_run()
    for g in ("policy", "value_fn"):
        for key in orc.PKEYS:
            d = np.abs(got[f"{g}/{key}"] - want[g][key]).max()
            assert d < 1e-4, (g, key, d)


@pytest.mark.parametrize("allreduce", ["peer", "nccl"])
def test_two_gpus(allreduce):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs (data-parallel path)")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_multi_discrete_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240, env=dict(os.environ, IMPALA_ALLREDUCE=allreduce))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_MD_OK" in res.stdout
