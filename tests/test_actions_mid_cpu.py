"""CPU: policies with 5..16 actions (Atari minimal action sets) have tensor-core MLP kernels of their own.

The 16-output instantiations - forward at one, two and four K atoms, backward (layer 2 through shared
memory) at one and two - are in the sm_90a library, issue HGMMA with one wait per batch of them (ptxas
did not serialize), keep no local memory, and the one-atom forward issues the m64n64 form.  The backward
workspace query covers the new shapes and still refuses the ones it refused before.
"""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

from torched_impala_b200 import _cabi

UNSUPPORTED = -2  # IMPALA_ERR_UNSUPPORTED_SHAPE

# mangled-name fragments of the 16-output instantiations
NEW_FWD = {ka: f"mlp_fwd_tc_kernelILi16ELi{ka}E" for ka in (1, 2, 4)}
NEW_BWD = {ka: f"mlp_bwd_tcw_kernelILi16ELi{ka}E" for ka in (1, 2)}

# (M, O, H, N2) of the tensor-core grid in test_gpu_actions_mid.py
SHAPES = [(20 * 1024, 128, 256, 6), (5000, 100, 512, 9), (3001, 24, 256, 6), (60001, 28, 128, 5),
          (777, 64, 512, 16), (1000, 32, 1024, 8), (5, 128, 128, 16), (4097, 4, 128, 7)]


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
        m = re.search(r"\b(HGMMA\.[0-9x]+\.[A-Z0-9]+\.[A-Z0-9]+)", ln)  # the MMA shape, e.g. HGMMA.64x64x8.F32.TF32
        if m and cur:
            kernels[cur][m.group(1)] += 1
    return kernels


def _one(sass, frag):
    hits = {name: ops for name, ops in sass.items() if frag in name}
    assert len(hits) == 1, f"{len(hits)} kernels named *{frag}* in the library"
    return next(iter(hits.items()))


@pytest.mark.parametrize("frag", list(NEW_FWD.values()) + list(NEW_BWD.values()))
def test_16_output_kernels_issue_hgmma_without_local_memory(sass_by_kernel, frag):
    name, ops = _one(sass_by_kernel, frag)
    assert ops["HGMMA"] > 0, name
    assert ops["HGMMA"] >= 8 * ops["WARPGROUP.DEPBAR"], (name, ops["HGMMA"], ops["WARPGROUP.DEPBAR"])
    assert ops["LDL"] == 0 and ops["STL"] == 0, (name, ops["LDL"], ops["STL"])


def test_one_atom_16_output_forward_issues_m64n64(sass_by_kernel):
    name, ops = _one(sass_by_kernel, NEW_FWD[1])
    assert ops["HGMMA.64x64x8.F32.TF32"] > 0, (name, {k: v for k, v in ops.items() if k.startswith("HGMMA")})


@pytest.mark.parametrize("M,O,H,N2", SHAPES)
def test_backward_workspace_covers_new_shapes(M, O, H, N2):
    assert _cabi.lib().impala_mlp_backward_workspace(M, O, H, N2) > 0


@pytest.mark.parametrize("M,O,H,N2", [(0, 24, 256, 6), (1000, 129, 256, 6), (1000, 128, 256, 33),
                                      (1000, 24, 256, 0), (1000, 0, 256, 6)])
def test_backward_workspace_still_refuses(M, O, H, N2):
    assert _cabi.lib().impala_mlp_backward_workspace(M, O, H, N2) == UNSUPPORTED
