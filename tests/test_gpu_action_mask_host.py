"""GPU: invalid-action masking beyond the kernel - a forked Learner behind a masked RingQueue and behind a plain
mp.Queue of trajectories with action_mask, against the float64 oracle learner, and two GPUs (peer push and NCCL)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import impala_oracle as orc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["ring", "queue"])
def test_forked_learner(tmp_path, kind):
    """A forked masked Learner, fed synthetic actors, ends within 1e-4 of the float64 oracle learner after 4 updates."""
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    import mask_learner_process_check as chk

    out = tmp_path / "weights.npz"
    res = subprocess.run([sys.executable, chk.__file__, str(tmp_path / "logs"), str(out), kind], capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MASK_LEARNER_OK" in res.stdout
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
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_action_mask_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240, env=dict(os.environ, IMPALA_ALLREDUCE=allreduce))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_MASK_OK" in res.stdout
