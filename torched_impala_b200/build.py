"""In-tree build of libimpala_b200.so for sm_90a (H100) (nvcc, no torch extension machinery).

`python -m torched_impala_b200.build` (or `__graft_entry__.build()`) compiles every
translation unit under csrc/ in parallel and links them into
`torched_impala_b200/lib/libimpala_b200.so`.  The runtime is linked statically
(`-cudart static`) so the library loads with nothing but the driver present; objects
are cached by source mtime so an incremental rebuild only recompiles what changed.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# IMPALA_LIB_DIR: build somewhere else (compile checks while a snapshot of the tree is in flight)
_LIB_DIR = os.environ.get("IMPALA_LIB_DIR", os.path.join(HERE, "lib"))
# IMPALA_PHASE_CLOCKS=1: compile the phase clocks of the narrow tensor-core MLP kernels in
# (csrc/phase_clocks.cuh, scripts/phase_mlp.py); build such a library into an IMPALA_LIB_DIR of its own
_DEFS = ["-DIMPALA_PHASE_CLOCKS"] if os.environ.get("IMPALA_PHASE_CLOCKS") == "1" else []
OBJ = os.path.join(_LIB_DIR, "obj")
LIB = os.path.join(_LIB_DIR, "libimpala_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
MLP_WIDTHS = (8, 24, 32, 64, 128)


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built")


def _units():
    units = [("mlp", "mlp.cu", []), ("vtrace_loss", "vtrace_loss.cu", []),
             ("vtrace_loss_rclip", "vtrace_loss_rclip.cu", []), ("vtrace_loss_gauss", "vtrace_loss_gauss.cu", []),
             ("vtrace_loss_md", "vtrace_loss_md.cu", []),
             ("vtrace_loss_mask", "vtrace_loss_mask.cu", []),
             ("optim", "optim.cu", []), ("abi", "abi.cu", []),
             ("mlp_fwd_tc", "mlp_fwd_tc.cu", []), ("mlp_bwd_tc", "mlp_bwd_tc.cu", []),
             ("loss_terms", "loss_terms.cu", []), ("mlp_obs_tc", "mlp_obs_tc.cu", []),
             ("obs_frames", "obs_frames.cu", []), ("batch_compose", "batch_compose.cu", []),
             ("obs_norm", "obs_norm.cu", [])]
    for op in MLP_WIDTHS:
        for bwd in (0, 1):
            units.append((f"mlp_inst_op{op}_{'bwd' if bwd else 'fwd'}", "mlp_inst.cu",
                          [f"-DIMPALA_OP={op}", f"-DIMPALA_BWD={bwd}"]))
    return units


def _newest_source_mtime() -> float:
    paths = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    paths.append(os.path.join(HERE, "..", "include", "impala_b200.h"))
    paths.append(os.path.abspath(__file__))
    return max(os.path.getmtime(p) for p in paths)


def _compile(nvcc, name, src, defs, stamp):
    obj = os.path.join(OBJ, name + ".o")
    log = os.path.join(OBJ, name + ".ptxas.log")
    if os.path.exists(obj) and os.path.getmtime(obj) >= stamp:
        return name, 0, "cached"
    cmd = [nvcc, *ARCH, *COMMON, *_DEFS, *defs, "-c", os.path.join(CSRC, src), "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    with open(log, "w") as f:
        f.write(res.stderr)
    return name, res.returncode, res.stderr if res.returncode else "built"


def build(verbose: bool = False, jobs: int | None = None) -> str:
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    stamp = _newest_source_mtime()
    # the objects of a directory were built with one set of defines, recorded beside them: other (or unknown)
    # defines rebuild every unit, so a default and an IMPALA_PHASE_CLOCKS build never share an object
    defs_file = os.path.join(OBJ, "defines.txt")
    defs = " ".join(_DEFS)
    built_with = open(defs_file).read() if os.path.exists(defs_file) else None
    if built_with != defs:
        stamp = float("inf")
        if built_with is not None:
            os.remove(defs_file)
    units = _units()
    jobs = jobs or min(len(units), os.cpu_count() or 4)
    with cf.ThreadPoolExecutor(jobs) as ex:
        results = list(ex.map(lambda u: _compile(nvcc, *u, stamp), units))
    for name, rc, msg in results:
        if rc:
            raise RuntimeError(f"nvcc failed on {name}:\n{msg}")
        if verbose:
            print(f"[build] {name}: {msg}")
    with open(defs_file, "w") as f:
        f.write(defs)
    objs = [os.path.join(OBJ, u[0] + ".o") for u in units]
    if (not os.path.exists(LIB)) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [nvcc, *ARCH, "-shared", "-cudart", "static", "-o", LIB, *objs]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode:
            raise RuntimeError(f"link failed:\n{res.stderr}")
        if verbose:
            print(f"[build] linked {LIB}")
    return LIB


if __name__ == "__main__":
    print(build(verbose=True))
    sys.exit(0)
