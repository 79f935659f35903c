"""CPU: the built library accepts wide observations (128 < O <= 1024, O % 4 == 0, H = 128 k <= 1024, N2 <= 32)
and refuses what lies outside, and its K-streamed tensor-core kernels use HGMMA with one wait per batch of
them and no local memory."""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

from torched_impala_b200 import _cabi


@pytest.mark.parametrize("M,O,H,N2", [(81920, 512, 256, 18), (86016, 512, 256, 1), (5, 132, 128, 1),
                                      (1, 1024, 1024, 32), (20480, 400, 256, 6)])
def test_obs_workspace_supported(M, O, H, N2):
    assert _cabi.lib().impala_mlp_backward_workspace(M, O, H, N2) > 0


@pytest.mark.parametrize("O,H,N2,env", [(130, 256, 6, {}), (1028, 256, 6, {}), (512, 320, 6, {}),
                                        (512, 1152, 6, {}), (512, 256, 33, {}),
                                        (512, 256, 6, {"IMPALA_MLP_TC": "0"}),
                                        (512, 256, 6, {"IMPALA_MLP_TCW": "0"})])
def test_obs_workspace_refused(monkeypatch, O, H, N2, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert _cabi.lib().impala_mlp_backward_workspace(1000, O, H, N2) == -2


def test_obs_workspace_is_dominated_by_dpt():
    """At 4 stacked RAM frames (T20 B4096 O512 A18 H256) DP^T (H x rows x 4 B) is most of the workspace."""
    lib = _cabi.lib()
    for M, N2 in ((20 * 4096, 18), (21 * 4096, 1)):
        dpt = 256 * M * 4
        ws = lib.impala_mlp_backward_workspace(M, 512, 256, N2)
        assert dpt < ws < 1.25 * dpt, (M, ws, dpt)


@pytest.fixture(scope="module")
def sass_by_kernel():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([exe, "-sass", _cabi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, cur = {}, None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            kernels[cur] = Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)((?:\.[A-Z0-9_]+)*)", ln)
        if m and cur:
            kernels[cur][m.group(1)] += 1
            kernels[cur][m.group(1) + m.group(2)] += 1
    return kernels


NEW_KERNELS = ["mlp_fwd_obs_kernelILi1E", "mlp_fwd_obs_kernelILi4E", "mlp_fwd_obs_kernelILi32E",
               "mlp_bwd_obs_pre_kernelILi1E", "mlp_bwd_obs_pre_kernelILi4E", "mlp_bwd_obs_pre_kernelILi32E",
               "mlp_bwd_obs_dw1_kernel"]


@pytest.mark.parametrize("frag", NEW_KERNELS)
def test_obs_kernels_use_hgmma_without_local_memory(sass_by_kernel, frag):
    hits = {name: ops for name, ops in sass_by_kernel.items() if frag in name}
    assert hits, f"no kernel named *{frag}* in the library"
    for name, ops in hits.items():
        # every form of the warpgroup wait (WARPGROUP.DEPBAR.LE ...)
        waits = sum(n for k, n in ops.items() if k.startswith("WARPGROUP.DEPBAR"))
        assert ops["HGMMA"] > 0, name
        assert ops["HGMMA"] >= 8 * waits, (name, ops["HGMMA"], waits)
        assert ops["LDL"] == 0 and ops["STL"] == 0, (name, ops["LDL"], ops["STL"])
