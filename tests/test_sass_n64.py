"""CPU: the narrow tensor-core MLP kernels issue the 64-column warpgroup MMA.

At one K atom the forward (fwd_rs_body: the pair kernel and every one-atom single-network forward)
issues two 32-unit hidden slices as one m64n64k8 chain, and the narrow backward (bwd_blk_body) runs its
recompute GEMM over the tile's 64 batch rows as m64n64k8 MMAs.
In `cuobjdump -sass` of the sm_90a library that is the HGMMA.64x64x8.F32.TF32 form; a kernel left on
pairs of m64n32 MMAs would only show HGMMA.64x32x8.F32.TF32.
"""
from collections import Counter
import os
import re
import shutil
import subprocess

import pytest

from torched_impala_b200 import _cabi

N64 = "HGMMA.64x64x8.F32.TF32"
N32 = "HGMMA.64x32x8.F32.TF32"
# kernel name patterns (mangled) -> the narrow bodies they run
NARROW = {
    "forward pair": r"mlp_fwd_tc_pair_kernel",
    "forward, one K atom": r"mlp_fwd_tc_kernelILi\d+ELi1EE",
    "backward pair": r"mlp_bwd_tc_pair_kernel",
    "backward": r"mlp_bwd_tc_kernelILi\d+EE",
}


@pytest.fixture(scope="module")
def hgmma_forms():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([exe, "-sass", _cabi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    forms, cur = {}, None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            forms[cur] = Counter()
            continue
        m = re.search(r"\b(HGMMA\.[0-9x]+\.[A-Z0-9]+\.[A-Z0-9]+)", ln)
        if m and cur:
            forms[cur][m.group(1)] += 1
    return forms


@pytest.mark.parametrize("what", sorted(NARROW))
def test_narrow_kernels_issue_64_column_mma(hgmma_forms, what):
    hits = {name: f for name, f in hgmma_forms.items() if re.search(NARROW[what], name)}
    assert hits, f"no {what} kernel in the library"
    for name, f in hits.items():
        assert f[N64] > 0, (name, dict(f))
