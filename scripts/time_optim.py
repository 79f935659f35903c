"""Time impala_clip_optim (RMSprop with momentum 0 and 0.9, Adam under a learning-rate table) against
impala_clip_adam, and the learner step of a default engine against an RMSprop engine with a schedule.

    python scripts/time_optim.py [--launches 200] [--steps 200] [--configs c4,c5]

Kernels: at the c4 size (14 144 parameters), the c5 size (69 312) and the largest parameter vector the MLP route
table allows (O = H = 1024, 32 actions); median of `--launches` launches per arm, the arms alternating launch by
launch, L2 flushed before each, CUDA events around the launch.  Steps: device-resident engine steps (CUDA graph),
the two engines alternating step by step, L2 flushed before each.  The GPU name, power limit and maximum SM clock
are read in the same run.  Nothing is written to the tree."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from torched_impala_b200 import _cabi, ops, synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402

CFG = {"c4": dict(T=20, B=4096, O=24, A=4, H=256), "c5": dict(T=100, B=8192, O=64, A=4, H=512)}


def n_params(O, H, A):
    return _cabi.param_layout(O, H, A)[1] + _cabi.param_layout(O, H, 1)[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--configs", default="c4,c5")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_optim.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    lr = 0.95 * 1e-3
    table = torch.full((1000,), lr, dtype=torch.float32, device="cuda")
    arms = {"impala_clip_adam": None, "clip_optim adam+table": ("adam", 0.9, 0.999, 1e-8),
            "clip_optim rmsprop m=0": ("rmsprop", 0.99, 0.0, 0.01),
            "clip_optim rmsprop m=0.9": ("rmsprop", 0.99, 0.9, 0.01)}
    sizes = {"c4": n_params(24, 256, 4), "c5": n_params(64, 512, 4), "largest": n_params(1024, 1024, 32)}
    for label, n in sizes.items():
        gen = torch.Generator(device="cuda").manual_seed(n)
        grad = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen) * 1e-3
        bufs = {k: [torch.randn(n, device="cuda", generator=gen), torch.zeros(n, device="cuda"),
                    torch.zeros(n, device="cuda"), torch.zeros(3, dtype=torch.int64, device="cuda")] for k in arms}
        ts = {k: [] for k in arms}
        for i in range(a.launches + 10):
            for k, h in arms.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                p, m, v, st = bufs[k]
                if h is None:
                    ops.clip_adam(p, grad, m, v, st, n // 2, 10.0, lr)
                else:
                    ops.clip_optim(p, grad, m, v, st, n // 2, 10.0, table, *h)
                e1.record()
                e1.synchronize()
                if i >= 10:
                    ts[k].append(e0.elapsed_time(e1) * 1e3)
        base = statistics.median(ts["impala_clip_adam"])
        print(f"kernel n={n} ({label}): " + ", ".join(
            f"{k} {statistics.median(v):.2f} us ({statistics.median(v) - base:+.2f})" for k, v in ts.items()))
    for cfg in a.configs.split(","):
        w = CFG[cfg]
        hp = default_hparams(batch_size=w["B"], max_timesteps=w["T"], max_updates=100000)
        batch = synth.make_batch(1, w["T"], w["B"], w["O"], w["A"])
        engines = {"default (adam)": {}, "rmsprop+schedule": dict(optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01),
                                                                  lr_lambda=lambda e: 1.0 - e / 100000)}
        for k, kw in list(engines.items()):
            eng = LearnerEngine(w["T"], w["B"], w["O"], w["A"], w["H"], w["H"], hp, **kw)
            eng.load_state(synth.init_params(0, w["O"], w["A"], w["H"]))
            eng.load_device_batch(batch, 0)
            engines[k] = eng
        ts = {k: [] for k in engines}
        for i in range(a.steps + 5):
            for k, eng in engines.items():
                with torch.cuda.stream(eng.stream):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(eng.stream)
                    eng.step(0)
                    e1.record(eng.stream)
                    e1.synchronize()
                    if i >= 5:
                        ts[k].append(e0.elapsed_time(e1) * 1e3)
        base = statistics.median(ts["default (adam)"])
        for k, eng in engines.items():
            med = statistics.median(ts[k])
            print(f"step {cfg} {w} [{k}]: median {med:.1f} us/step ({med - base:+.1f} us), "
                  f"{eng.launches_per_step} launches, loss {eng.read_scalars()['total_loss']:.5f}")
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"GPU (nvidia-smi): {q}")


if __name__ == "__main__":
    main()
