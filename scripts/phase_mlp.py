"""Phase clocks of the narrow tensor-core MLP kernels: where a warpgroup's cycles go in the paired forward
(`fwd_rs_body`) and backward (`bwd_blk_body`) launches of one learner step.

Builds the library with IMPALA_PHASE_CLOCKS=1 into its own directory (csrc/phase_clocks.cuh; the default
library is not touched), runs the c3 or c4 forward pair and backward pair, L2 flushed before each launch,
and prints cycles per warpgroup-tile for every phase, the tensor-busy fraction and the overlap fraction:

    python scripts/phase_mlp.py [--config c4] [--iters 200] [--lib-dir DIR]

tensor-busy = issued MMA cycles / SM cycles, from the tensor-core rate of the H100 SXM data sheet (dense
TF32: 2 048 FLOP per cycle per SM, so an m64n64k8 takes 32 cycles and an m64n32k8 16); overlap = share of GEMM
windows (issue -> wait return) opened while the other warpgroup of the CTA was inside one; it does not see
the other CTA of an SM.  The instrumented kernels are not the default ones: the clocks add shared-memory
updates per phase and change the register allocation (the backward pair compiles to 241 registers instead
of 255), so they show where a warpgroup's cycles go, not how fast the default kernels run; time those with
CUDA events (bench.py's `kernels`).  Needs a GPU; there is nothing to measure without one.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIGS = {"c3": dict(T=20, B=1024, O=24, A=4, H=256), "c4": dict(T=20, B=4096, O=24, A=4, H=256)}
# phase sums [0, 8) of each body, in the order of its PHASE_MARK indices
PHASES = {
    "bwd": ["stage barrier wait", "staging", "GEMM1 issue->wait", "epilogue + DP split", "GEMM2 issue->wait",
            "ping-pong token wait"],
    "fwd": ["batch issue->wait", "epilogue", "x split", "row write", "ping-pong token wait", "weight staging"],
}
SLOTS = 16  # phase::kSlots
K_TILES, K_OVERLAP, K_WINDOWS, K_WG_CYCLES, K_CTA_NS, K_CTAS, K_FIRST_NS, K_LAST_NS = range(8, 16)
WG_PER_SM = {"bwd": 2, "fwd": 4}  # backward: one CTA of 2 warpgroups per SM; forward pair: two CTAs


def tensor_cycles(kind, O, H):
    """Issued MMA cycles of one warpgroup-tile at the data-sheet rate (3xTF32: three products per K step)."""
    ksteps = (O + 7) // 8
    if kind == "bwd":  # GEMM1 m64n64 per product and K step, GEMM2 8 K steps x 3 products of m64n32
        return 3 * ksteps * 32 + 24 * 16
    return (H // 64) * 3 * ksteps * 32 + (H % 64 // 32) * 3 * ksteps * 16


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="c4", choices=sorted(CONFIGS))
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--lib-dir", default=os.path.join(tempfile.gettempdir(), "impala_phase_clocks"),
                    help="directory of the instrumented library (brought up to date with this tree first)")
    ap.add_argument("--json", default=None, help="also write the table here")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        sys.exit("phase_mlp.py needs a CUDA device: phase clocks are read from the GPU")
    lib_dir = os.path.abspath(args.lib_dir)
    # incremental: units older than the tree's sources, or built with other defines, are rebuilt
    env = dict(os.environ, IMPALA_PHASE_CLOCKS="1", IMPALA_LIB_DIR=lib_dir)
    subprocess.run([sys.executable, "-m", "torched_impala_b200.build"], cwd=ROOT, env=env, check=True,
                   stdout=subprocess.DEVNULL)
    os.environ["IMPALA_LIB_DIR"] = lib_dir  # before _cabi is imported
    sys.path.insert(0, ROOT)
    from torched_impala_b200 import synth
    from torched_impala_b200.engine import LearnerEngine, _ptr
    from torched_impala_b200.utils import default_hparams

    w = CONFIGS[args.config]
    hp = default_hparams(batch_size=w["B"], max_timesteps=w["T"])
    eng = LearnerEngine(w["T"], w["B"], w["O"], w["A"], w["H"], w["H"], hp, use_graph=False)
    eng.load_state(synth.init_params(0, w["O"], w["A"], w["H"]))
    eng.load_device_batch(synth.make_batch(1, w["T"], w["B"], w["O"], w["A"]))
    eng.step()
    eng.synchronize()
    lib = eng.lib
    if not hasattr(lib, "impala_phase_read"):
        sys.exit(f"{lib_dir}/libimpala_b200.so was built without IMPALA_PHASE_CLOCKS")
    lib.impala_phase_read.restype = C.c_int
    lib.impala_phase_read.argtypes = [C.c_void_p, C.c_int]

    O, A, H = eng.O, eng.A, eng.H_pi
    st = C.c_void_p(eng.stream.cuda_stream)
    p_pi = C.c_void_p(eng.params.data_ptr())
    p_vf = C.c_void_p(eng.params.data_ptr() + 4 * eng.n_pi)
    g_pi = C.c_void_p(eng.comm.data_ptr())
    g_vf = C.c_void_p(eng.comm.data_ptr() + 8 * eng.n_pi)
    obs = _ptr(eng.d["obs"])
    launch = {
        "fwd": lambda: lib.impala_mlp_forward_pair(obs, p_pi, p_vf, _ptr(eng.logits), _ptr(eng.values), eng.M_pi,
                                                   eng.M_vf, O, eng.H_pi, eng.H_v, A, st),
        "bwd": lambda: lib.impala_mlp_backward_pair(obs, p_pi, p_vf, _ptr(eng.dlogits), _ptr(eng.dv), g_pi, g_vf,
                                                    _ptr(eng.ws_pi), eng.ws_pi_bytes, _ptr(eng.ws_vf),
                                                    eng.ws_vf_bytes, eng.M_pi, eng.M_vf, O, eng.H_pi, eng.H_v, A, st),
    }
    buf = torch.empty(256 << 20, dtype=torch.uint8, device=eng.dev)
    raw = (C.c_ulonglong * (2 * SLOTS))()

    def read(reset):
        torch.cuda.synchronize(eng.dev)
        if lib.impala_phase_read(C.addressof(raw), int(reset)):
            raise RuntimeError("impala_phase_read failed")
        return {"bwd": list(raw[:SLOTS]), "fwd": list(raw[SLOTS:])}

    def run(kind):
        with torch.cuda.stream(eng.stream):
            buf.zero_()  # L2 cold, as in bench.py's kernel breakdown
            rc = launch[kind]()
        if rc:
            raise RuntimeError(f"{kind} pair launch returned {rc}")

    for _ in range(10):
        run("fwd"), run("bwd")
    # launch span and CTA spans, one launch at a time
    spans = {"fwd": [], "bwd": []}
    for _ in range(20):
        for kind in ("fwd", "bwd"):
            read(True)
            run(kind)
            c = read(False)[kind]
            spans[kind].append(((c[K_LAST_NS] - c[K_FIRST_NS]) / 1e3, c[K_CTA_NS] / c[K_CTAS] / 1e3))
    read(True)
    for _ in range(args.iters):
        run("fwd"), run("bwd")
    cnt = read(True)

    report = {"config": args.config, "gpu": torch.cuda.get_device_name(eng.dev), "iters": args.iters}
    for kind, name in (("fwd", "mlp_forward_pair"), ("bwd", "mlp_backward_pair")):
        c = cnt[kind]
        tiles = c[K_TILES]
        per_tile = c[K_WG_CYCLES] / tiles
        phases = {p: c[i] / tiles for i, p in enumerate(PHASES[kind])}
        tc = tensor_cycles(kind, O, H)
        span = sorted(s[0] for s in spans[kind])[len(spans[kind]) // 2]
        cta = sorted(s[1] for s in spans[kind])[len(spans[kind]) // 2]
        r = {"wg_tiles_per_launch": tiles / args.iters, "cycles_per_wg_tile": per_tile, "phases": phases,
             "tensor_cycles_per_wg_tile": tc, "tensor_busy": tc * WG_PER_SM[kind] / per_tile,
             "overlap": c[K_OVERLAP] / c[K_WINDOWS], "launch_span_us": span, "mean_cta_span_us": cta}
        report[name] = r
        print(f"{name} ({args.config}, {tiles / args.iters:.0f} warpgroup-tiles per launch, median launch span "
              f"{span:.1f} us, mean CTA span {cta:.1f} us)")
        for p, v in phases.items():
            print(f"  {p:24s} {v:8.0f} cycles / warpgroup-tile")
        print(f"  {'whole body':24s} {per_tile:8.0f} cycles / warpgroup-tile (prologue and tail included)")
        print(f"  tensor-busy {r['tensor_busy']:.2f} ({tc} MMA cycles per warpgroup-tile, {WG_PER_SM[kind]} "
              f"warpgroups per SM), overlap {r['overlap']:.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
