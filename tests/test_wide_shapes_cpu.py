"""CPU: the built library accepts Atari-RAM-sized networks (O <= 128, N2 <= 32) and its new kernels are
the ones the design claims - tensor-core forwards and backwards with HGMMA and one wait per batch of
them, and no local memory in any of the new tensor-core, FP32 MLP or V-trace instantiations."""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

from torched_impala_b200 import _cabi


def test_backward_workspace_limits():
    lib = _cabi.lib()
    assert lib.impala_mlp_backward_workspace(1000, 128, 256, 18) > 0
    assert lib.impala_mlp_backward_workspace(1000, 65, 128, 32) > 0
    assert lib.impala_mlp_backward_workspace(1000, 129, 256, 18) == -2
    assert lib.impala_mlp_backward_workspace(1000, 128, 256, 33) == -2


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


# mangled-name fragments of the instantiations added for O in 65..128 / N2 in 17..32 / A in 17..32
NEW_TC = ["mlp_fwd_tc_kernelILi1ELi4E", "mlp_fwd_tc_kernelILi4ELi4E", "mlp_fwd_tc_kernelILi32ELi1E",
          "mlp_fwd_tc_kernelILi32ELi2E", "mlp_fwd_tc_kernelILi32ELi4E",
          "mlp_bwd_tcw_kernelILi1ELi4E", "mlp_bwd_tcw_kernelILi4ELi4E", "mlp_bwd_tcw_kernelILi32ELi4E"]
NEW_FP32 = ([f"mlp_fwd_kernelILi1ELi128ELi{n}ELi256E" for n in (1, 4, 16, 32)] +
            [f"mlp_bwd_kernelILi1ELi128ELi{n}ELi256ELi4E" for n in (1, 4, 16, 32)] +
            [f"mlp_fwd_kernelILi1ELi{o}ELi32ELi256E" for o in (8, 24, 32, 64)] +
            [f"mlp_bwd_kernelILi1ELi{o}ELi32ELi256ELi2E" for o in (8, 24, 32)] +
            ["mlp_bwd_kernelILi1ELi64ELi32ELi256ELi4E", "vtrace_lane_kernelILi32E"])


def _hits(sass, frag):
    hits = {name: ops for name, ops in sass.items() if frag in name}
    assert hits, f"no kernel named *{frag}* in the library"
    return hits


@pytest.mark.parametrize("frag", NEW_TC)
def test_new_tensor_core_kernels_use_hgmma(sass_by_kernel, frag):
    for name, ops in _hits(sass_by_kernel, frag).items():
        assert ops["HGMMA"] > 0, name
        # one wait per batch of wgmma, not one per MMA (ptxas serializes them when the accumulators are touched)
        assert ops["HGMMA"] >= 8 * ops["WARPGROUP.DEPBAR"], (name, ops["HGMMA"], ops["WARPGROUP.DEPBAR"])
        assert ops["LDL"] == 0 and ops["STL"] == 0, (name, ops["LDL"], ops["STL"])


@pytest.mark.parametrize("frag", NEW_FP32)
def test_new_kernels_have_no_local_memory(sass_by_kernel, frag):
    for name, ops in _hits(sass_by_kernel, frag).items():
        assert ops["LDL"] == 0 and ops["STL"] == 0, (name, ops["LDL"], ops["STL"])
