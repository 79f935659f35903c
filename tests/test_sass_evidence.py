"""CPU: the built library really contains the Hopper-native instruction streams the design claims.

`cuobjdump -sass` of torched_impala_b200/lib/libimpala_b200.so (sm_90a) is scanned per kernel for the
SASS mnemonics of wgmma.mma_async (HGMMA) and its warpgroup synchronisation (WARPGROUP.ARRIVE /
DEPBAR around it): a kernel that silently fell back to FFMA / mma.sync code would fail here before it
ever reaches a GPU.  The DEPBAR count also shows whether ptxas serialized the MMAs (one wait per wgmma
instead of one per batch of them).
"""
from collections import Counter
import os
import re
import shutil
import subprocess

import pytest

from torched_impala_b200 import _cabi

WANT = {
    # kernel name fragment -> mnemonics that must appear in it
    "mlp_fwd_tc_pair_kernel": ("HGMMA", "WARPGROUP"),
    "mlp_bwd_tc_pair_kernel": ("HGMMA", "WARPGROUP"),
    "mlp_bwd_tc_kernel": ("HGMMA", "WARPGROUP"),
    "mlp_fwd_tc_kernel": ("HGMMA", "WARPGROUP"),  # narrow and wide (two K atoms) instantiations
    "mlp_bwd_tcw_kernel": ("HGMMA", "WARPGROUP"),
}


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


@pytest.mark.parametrize("fragment", sorted(WANT))
def test_kernel_contains_hopper_instructions(sass_by_kernel, fragment):
    hits = {name: ops for name, ops in sass_by_kernel.items() if fragment in name}
    assert hits, f"no kernel named *{fragment}* in the library"
    for name, ops in hits.items():
        missing = [w for w in WANT[fragment] if w not in ops]
        assert not missing, (name, missing)


@pytest.mark.parametrize("fragment", sorted(WANT))
def test_wgmma_batches_are_not_serialized(sass_by_kernel, fragment):
    """Each batch of wgmma ends in one wait; a WARPGROUP.DEPBAR per HGMMA means ptxas serialized them
    (warning C7515: the accumulators were defined by other instructions inside a batch)."""
    for name, ops in sass_by_kernel.items():
        if fragment in name:
            assert ops["HGMMA"] >= 8 * ops["WARPGROUP.DEPBAR"], (name, ops["HGMMA"], ops["WARPGROUP.DEPBAR"])


def test_library_is_sm90a_only(sass_by_kernel):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([exe, "-lelf", _cabi.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs
