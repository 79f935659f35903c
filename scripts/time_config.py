"""Device-resident learner step time for any BASELINE config (c2..c5) or the Atari-RAM / MinAtar shapes: CUDA events,
L2 flushed, with the GPU name, power limit and maximum SM clock read in the same run.  --compare-tc also times the FP32 FFMA MLP path (IMPALA_MLP_TC=0) in the same process,
alternating step by step with the default path, so both numbers see the same clocks and neighbours.
--compare-obs alternates a float32-slab engine and a uint8-slab engine (byte observations 0..255) the same way
and reports, for both, the device-resident step time and the pinned-slab end-to-end step time (the DMA of
slab i+1 runs under step i; a step's window also waits for that DMA), with the GPU name, power limit and
maximum SM clock read in the same run.
--compare-frames alternates the dense engine and a frame engine (--frames k stacked frames stored once per frame,
--obs-dtype) on the same values the same way, and times the unstacking launch alone (median of 200 launches,
L2 flushed before each) against its HBM floor (frame bytes read + dense bytes written at 3.35 TB/s).
--compare-diag alternates a diagnostics=False and a diagnostics=True engine on the same batch the same way, and
times impala_vtrace_loss against impala_vtrace_loss_diag alone on the engine's buffers (median of 200 launches
each, alternating, L2 flushed before each).
--compare-replay alternates a plain engine and a replay engine (--replay-slabs R, --replay-columns Br, default
B/2; --obs-dtype, --frames k if given) the same way: the replay engine's pool is filled first, and the plain
engine trains on the very slab the replay engine composed, so both steps see the same values.  It also times
impala_batch_compose alone (median of 200 launches, L2 flushed before each) against its HBM floor (one training
slab read and written at 3.35 TB/s).
--compare-popart alternates a popart=False and a popart=True engine on the same batch the same way (the same
launch count; the PopArt arm adds one FMA per value load, the 1 / sigma scaling and the optimizer's head
epilogue), and times impala_vtrace_loss_diag against impala_vtrace_loss_popart and impala_clip_optim against
impala_clip_optim_popart alone on the engine's buffers (median of 200 launches each, alternating, L2 flushed
before each).
--compare-reward-clip alternates engines with reward_clip None, "abs_one" and "soft_asymmetric" on the same batch
(rewards N(0, 5^2), so both transforms act) the same way, and times impala_vtrace_loss against
impala_vtrace_loss_rclip in both modes alone on the engine's buffers (median of 200 launches each, alternating,
L2 flushed before each).
--compare-shared alternates a two-network engine and a shared-torso engine (shared_torso=True: one hidden layer
feeding the policy and the value head) on the same batch the same way, and reports both steps' launches.  Byte
observations for the Atari RAM and MinAtar shapes, as --compare-popart.
--compare-heads (configs md_c4, md_ram) alternates a categorical engine at A = N and a multi-discrete engine
(action_dist="multi_discrete" with the config's heads, N = sum of them) on batches of the same shapes the same way,
and times impala_vtrace_loss against impala_vtrace_loss_md alone on each engine's buffers (median of 200 launches
each, alternating, L2 flushed before each).
--compare-mask (configs mask_c4, mask_ram, md_mask_c4) alternates the unmasked engine and the masked one
(action_mask=True: legal words in the actions, about half the entries legal) on batches of the same shapes the same
way, and times the unmasked V-trace + loss kernel (impala_vtrace_loss, or impala_vtrace_loss_md for md_mask_c4)
against impala_vtrace_loss_mask alone on each engine's buffers (median of 200 launches each, alternating, L2 flushed
before each).
--compare-obs-norm alternates an obs_norm=False and an obs_norm=True engine (observation normalization) on the same
batch the same way (--obs-dtype for the slab; the halfcheetah config is a Gaussian policy), reports both steps'
launches, and times impala_obs_normalize alone on the engine's buffers (median of 200 launches, L2 flushed before
each) against its HBM floor (slab observations read + float32 rows written at 3.35 TB/s)."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.engine import LearnerEngine  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402

CFG = {"c4": dict(T=20, B=4096, O=24, A=4, H=256),
       # multi-discrete policies (--compare-heads): A = N = sum(heads) policy outputs
       "md_c4": dict(T=20, B=4096, O=24, A=8, H=256, heads=(3, 3, 2)),
       "md_ram": dict(T=20, B=4096, O=128, A=20, H=256, heads=(3, 3, 2, 2, 5, 5)), "c5": dict(T=100, B=8192, O=64, A=4, H=512),
       # invalid-action masks (--compare-mask): categorical at c4 and Atari-RAM shapes (byte observations), and md_c4's heads
       "mask_c4": dict(T=20, B=4096, O=24, A=8, H=256, mask=()), "mask_ram": dict(T=20, B=4096, O=128, A=18, H=256, mask=()),
       "md_mask_c4": dict(T=20, B=4096, O=24, A=8, H=256, mask=(3, 3, 2)),
       "c3": dict(T=20, B=1024, O=24, A=4, H=256), "c2": dict(T=20, B=256, O=4, A=2, H=32),
       # c4 with 512 hidden units: the wide forward at one K atom (two passes of 256) and the wide backward
       "c4h512": dict(T=20, B=4096, O=24, A=4, H=512),
       # Atari from RAM (128-byte observation, 18 actions): P = 70 931 parameters, 50 675 712 input bytes
       # and 24.4 GFLOP of MLP work per step (SURVEY 8d formulas)
       "ram": dict(T=20, B=4096, O=128, A=18, H=256),
       # 4 stacked Atari RAM frames: P = 267 539 parameters, 4x the layer-1 work of "ram": 88 GFLOP per step
       # (forward + dW1 of both networks), ~400 GFLOP executed on the tensor cores (3xTF32, the backward's
       # recompute), 176 MB of observations
       "ram4": dict(T=20, B=4096, O=512, A=18, H=256),
       # MinAtar Breakout / Asterix, flattened 10x10x4 binary grids: P = 207 111 parameters
       "minatar": dict(T=20, B=4096, O=400, A=6, H=256),
       # 8 stacked Atari RAM frames
       "ram8": dict(T=20, B=4096, O=1024, A=18, H=256),
       # minimal Atari action sets (Pong, Space Invaders, Q*bert: 6; Ms. Pac-Man, Enduro, Beam Rider: 9): the
       # 16-output tensor-core epilogue.  ram_a9h512 has no FP32 arm (that forward refuses H > 256 at O > 64)
       "ram_a6": dict(T=20, B=4096, O=128, A=6, H=256),
       "c4a6": dict(T=20, B=4096, O=24, A=6, H=256),
       "ram_a9h512": dict(T=20, B=4096, O=128, A=9, H=512),
       # MuJoCo HalfCheetah-shaped continuous control (--compare-obs-norm): 17 features, 6 action dimensions
       "halfcheetah": dict(T=20, B=4096, O=17, A=6, H=256, gaussian=True)}
ap = argparse.ArgumentParser()
ap.add_argument("--config", default="c5")
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--compare-tc", action="store_true", help="alternate with IMPALA_MLP_TC=0 and report both")
ap.add_argument("--compare-obs", action="store_true", help="alternate float32 and uint8 observation slabs")
ap.add_argument("--compare-frames", action="store_true", help="alternate dense and frame-stacked observation slabs")
ap.add_argument("--frames", type=int, default=None, help="stacked frames of --compare-frames (default 4) / --compare-replay (default 1)")
ap.add_argument("--obs-dtype", default="float32", choices=["float32", "uint8"], help="slab obs type of --compare-frames")
ap.add_argument("--compare-diag", action="store_true", help="alternate engines without / with off-policy diagnostics")
ap.add_argument("--compare-popart", action="store_true", help="alternate engines without / with PopArt")
ap.add_argument("--compare-replay", action="store_true", help="alternate engines without / with experience replay")
ap.add_argument("--compare-reward-clip", action="store_true", help="alternate engines without / with reward clipping")
ap.add_argument("--compare-shared", action="store_true", help="alternate two networks and a shared-torso network")
ap.add_argument("--compare-heads", action="store_true",
                help="alternate a categorical engine at A = N and a multi-discrete engine (configs md_c4, md_ram)")
ap.add_argument("--compare-mask", action="store_true",
                help="alternate an unmasked and a masked engine (configs mask_c4, mask_ram, md_mask_c4)")
ap.add_argument("--compare-obs-norm", action="store_true",
                help="alternate engines without / with observation normalization (--obs-dtype for the slab)")
ap.add_argument("--replay-slabs", type=int, default=2, help="past fresh batches in the pool of --compare-replay")
ap.add_argument("--replay-columns", type=int, default=None, help="replayed columns of --compare-replay (default B/2)")
a = ap.parse_args()
w = CFG[a.config]
if a.frames is None:
    a.frames = 1 if a.compare_replay else 4
hp = default_hparams(batch_size=w["B"], max_timesteps=w["T"])
arms = {"default": os.environ.get("IMPALA_MLP_TC", "1")}
obs_dt = {"default": "float32"}
if a.compare_tc:
    arms = {"tc": "1", "fp32 (IMPALA_MLP_TC=0)": "0"}
if a.compare_obs:
    arms = {"obs float32": arms["default"], "obs uint8": arms["default"]}
    obs_dt = {"obs float32": "float32", "obs uint8": "uint8"}
n_frames = {}
diag_arm = {}
if a.compare_diag:
    arms = {"diagnostics off": arms["default"], "diagnostics on": arms["default"]}
    diag_arm = {"diagnostics on": True}
    # byte observations where the flagship users of the shape have them (Atari RAM, MinAtar)
    obs_dt = {name: "uint8" if a.config in ("ram", "ram4", "ram8", "minatar", "ram_a6") else "float32" for name in arms}
if a.compare_frames:
    arms = {f"dense {a.obs_dtype}": arms["default"], f"frames={a.frames} {a.obs_dtype}": arms["default"]}
    obs_dt = {name: a.obs_dtype for name in arms}
    n_frames = {f"frames={a.frames} {a.obs_dtype}": a.frames}
popart_arm = {}
if a.compare_popart:
    arms = {"popart off": arms["default"], "popart on": arms["default"]}
    popart_arm = {"popart on": dict(popart=True)}
    obs_dt = {name: "uint8" if a.config in ("ram", "ram4", "ram8", "minatar", "ram_a6") else "float32" for name in arms}
rclip_arm = {}
if a.compare_reward_clip:
    arms = {"reward_clip None": arms["default"], "reward_clip abs_one": arms["default"],
            "reward_clip soft_asymmetric": arms["default"]}
    rclip_arm = {name: dict(reward_clip=name.split()[1]) for name in list(arms)[1:]}
    obs_dt = {name: "uint8" if a.config in ("ram", "ram4", "ram8", "minatar", "ram_a6") else "float32" for name in arms}
shared_arm = {}
if a.compare_shared:
    arms = {"two networks": arms["default"], "shared torso": arms["default"]}
    shared_arm = {"shared torso": dict(shared_torso=True)}
    obs_dt = {name: "uint8" if a.config in ("ram", "ram4", "ram8", "minatar", "ram_a6") else "float32" for name in arms}
heads_arm = {}
if a.compare_heads:
    if "heads" not in w:
        raise SystemExit(f"--compare-heads takes a multi-discrete config (md_c4, md_ram), not {a.config}")
    md_name = f"multi-discrete heads {w['heads']}"
    arms = {f"categorical A={w['A']}": arms["default"], md_name: arms["default"]}
    heads_arm = {md_name: dict(action_dist="multi_discrete", action_heads=w["heads"])}
mask_arm = {}
if a.compare_mask:
    if "mask" not in w:
        raise SystemExit(f"--compare-mask takes a masked config (mask_c4, mask_ram, md_mask_c4), not {a.config}")
    md_kw = dict(action_dist="multi_discrete", action_heads=w["mask"]) if w["mask"] else {}
    mask_name = "masked"
    arms = {"unmasked": arms["default"], mask_name: arms["default"]}
    heads_arm = {name: md_kw for name in arms} if md_kw else {}
    mask_arm = {mask_name: dict(action_mask=True)}
    obs_dt = {name: "uint8" if a.config == "mask_ram" else "float32" for name in arms}
obs_norm_arm = {}
if a.compare_obs_norm:
    arms = {"obs_norm off": arms["default"], "obs_norm on": arms["default"]}
    obs_norm_arm = {"obs_norm on": dict(obs_norm=True)}
    obs_dt = {name: a.obs_dtype for name in arms}
    if w.get("gaussian"):
        heads_arm = {name: dict(action_dist="gaussian") for name in arms}
replay_arm = {}
if a.compare_replay:
    Br = w["B"] // 2 if a.replay_columns is None else a.replay_columns
    on = f"replay R={a.replay_slabs} Br={Br}"
    arms = {"replay off": arms["default"], on: arms["default"]}
    obs_dt = {name: a.obs_dtype for name in arms}
    n_frames = {name: a.frames for name in arms}
    replay_arm = {on: dict(replay_slabs=a.replay_slabs, replay_columns=Br)}
engines = {}
for name, tc in arms.items():
    os.environ["IMPALA_MLP_TC"] = tc  # read by the C library at every launch (and at graph capture)
    dt = obs_dt.get(name, "float32")
    k = n_frames.get(name, 1)
    eng = LearnerEngine(w["T"], w["B"], w["O"], w["A"], w["H"], w["H"], hp, obs_dtype=dt, frames=k,
                        diagnostics=diag_arm.get(name, False), **replay_arm.get(name, {}), **popart_arm.get(name, {}),
                        **rclip_arm.get(name, {}), **shared_arm.get(name, {}), **heads_arm.get(name, {}),
                        **mask_arm.get(name, {}), **obs_norm_arm.get(name, {}))
    eng.load_state(synth.init_params(0, w["O"], 2 * w["A"] if w.get("gaussian") else w["A"], w["H"]))
    byte_obs = (a.compare_obs or ((a.compare_frames or a.compare_replay) and dt == "uint8")
                or ((a.compare_diag or a.compare_popart or a.compare_reward_clip or a.compare_shared or a.compare_mask)
                    and dt == "uint8"))
    if a.compare_replay:
        engines[name] = eng
        continue
    if a.compare_frames:  # the same observation values in both arms: the dense arm gets the stacked frames
        batch = synth.make_batch(1, w["T"], w["B"], w["O"], w["A"], obs_kind="bytes" if byte_obs else "normal",
                                 frames=a.frames)
        if k == 1:
            batch = synth.stack_frames(batch, a.frames)
    elif name in mask_arm:
        batch = synth.make_masked_batch(1, w["T"], w["B"], w["O"], w["A"], w["mask"], density=0.5,
                                        obs_kind="bytes" if byte_obs else "normal")
        batch.pop("legal")
    elif w.get("gaussian"):
        batch = synth.make_gaussian_batch(1, w["T"], w["B"], w["O"], w["A"])
    elif a.compare_obs_norm:
        batch = synth.make_batch(1, w["T"], w["B"], w["O"], w["A"], obs_kind="bytes" if dt == "uint8" else "normal")
    elif name in heads_arm:
        batch = (synth.make_md_batch(1, w["T"], w["B"], w["O"], w["heads"]) if "heads" in w else
                 synth.make_md_batch(1, w["T"], w["B"], w["O"], w["mask"]))
    else:
        batch = synth.make_batch(1, w["T"], w["B"], w["O"], w["A"], obs_kind="bytes" if byte_obs else "normal")
    if dt == "float32":
        batch["obs"] = batch["obs"].astype("float32")
    if a.compare_reward_clip:
        batch["rewards"] = batch["rewards"] * 5.0
    eng.load_device_batch(batch)
    if a.compare_obs or a.compare_frames:
        eng.load_device_batch(batch, 1)
    engines[name] = eng
if a.compare_replay:  # fill the pool (R fresh batches, then the one trained on), then hand the composed slab over
    eng = engines[on]
    for n in range(a.replay_slabs + 1):
        eng.load_device_batch(synth.make_batch(1 + n, w["T"], eng.B_fresh, w["O"], w["A"], frames=a.frames,
                                               obs_kind="bytes" if a.obs_dtype == "uint8" else "normal"))
        eng.step(0)
        eng.synchronize()
    assert (eng.replay_plan[:, 0] >= 0).all()
    engines["replay off"].d_slabs[0].copy_(eng.d_slabs[0])
    torch.cuda.synchronize()
    engines["replay off"].slab_ready[0].record(engines["replay off"].copy_stream)
    eng.load_state(synth.init_params(0, w["O"], w["A"], w["H"]))  # both arms start the timed steps from the same weights
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
ts = {name: [] for name in arms}
for i in range(a.steps + 5):
    for name, eng in engines.items():
        os.environ["IMPALA_MLP_TC"] = arms[name]
        with torch.cuda.stream(eng.stream):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(eng.stream)
            eng.step(0)
            e1.record(eng.stream)
            e1.synchronize()
            if i >= 5:
                ts[name].append(e0.elapsed_time(e1) * 1e3)
te = {name: [] for name in arms}
if a.compare_obs or a.compare_frames:  # pinned-slab end to end: ingest(slab i+1) on the copy stream under step(slab i)
    for i in range(a.steps + 5):
        for name, eng in engines.items():
            with torch.cuda.stream(eng.stream):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(eng.stream)
                eng.copy_stream.wait_event(e0)
                eng.ingest((i + 1) % 2)
                eng.step(i % 2)
                eng.stream.wait_event(eng.slab_ready[(i + 1) % 2])
                e1.record(eng.stream)
                e1.synchronize()
                if i >= 5:
                    te[name].append(e0.elapsed_time(e1) * 1e3)
dev = torch.cuda.get_device_name()
if a.compare_frames:  # the unstacking launch alone, back to back
    import ctypes

    from torched_impala_b200 import _cabi

    eng = engines[f"frames={a.frames} {a.obs_dtype}"]
    out_code = _cabi.OBS_U8 if eng.obs_dense.dtype == torch.uint8 else _cabi.OBS_F32
    args = (ctypes.c_void_p(eng.d["obs"].data_ptr()), eng.obs_code, ctypes.c_void_p(eng.obs_dense.data_ptr()),
            out_code, w["T"] + 1, w["B"], eng.F, a.frames)
    with torch.cuda.stream(eng.stream):
        st = ctypes.c_void_p(eng.stream.cuda_stream)
        tu = []
        for i in range(220):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(eng.stream)
            _cabi.check(eng.lib.impala_obs_unstack(*args, st), "impala_obs_unstack")
            e1.record(eng.stream)
            e1.synchronize()
            if i >= 20:
                tu.append(e0.elapsed_time(e1) * 1e3)
    us = statistics.median(tu)
    nbytes = eng.d["obs"].numel() * eng.d["obs"].element_size() + eng.obs_dense.numel() * eng.obs_dense.element_size()
    print(f"impala_obs_unstack {a.config} frames={a.frames} {a.obs_dtype} -> {eng.obs_dense.dtype}: {us:.1f} us, "
          f"{nbytes / 1e6:.1f} MB moved, HBM floor {nbytes / 3.35e12 * 1e6:.1f} us at 3.35 TB/s "
          f"({nbytes / 3.35e12 * 1e6 / us:.0%} of it)")
if a.compare_replay:  # the compose launch alone
    import ctypes

    from torched_impala_b200 import _cabi

    eng = engines[on]
    args = (ctypes.c_void_p(eng.d_slabs[0].data_ptr()), ctypes.c_void_p(eng.store.data_ptr()), eng.slab_bytes,
            ctypes.c_void_p(eng.d_plans[0].data_ptr()), w["T"], w["B"], eng.B_fresh, eng.F, a.frames, w["A"], eng.obs_code)
    with torch.cuda.stream(eng.stream):
        st = ctypes.c_void_p(eng.stream.cuda_stream)
        tu = []
        for i in range(220):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(eng.stream)
            _cabi.check(eng.lib.impala_batch_compose(*args, st), "impala_batch_compose")
            e1.record(eng.stream)
            e1.synchronize()
            if i >= 20:
                tu.append(e0.elapsed_time(e1) * 1e3)
    us, nbytes = statistics.median(tu), 2 * eng.d_slabs[0].numel()
    print(f"impala_batch_compose {a.config} frames={a.frames} {a.obs_dtype} {on}: {us:.1f} us, {nbytes / 1e6:.1f} MB moved "
          f"(training slab {nbytes / 2e6:.1f} MB read and written, fresh slab {eng.slab_bytes / 1e6:.1f} MB, store "
          f"{eng.store.numel() / 1e6:.1f} MB), HBM floor {nbytes / 3.35e12 * 1e6:.1f} us at 3.35 TB/s "
          f"({nbytes / 3.35e12 * 1e6 / us:.0%} of it)")
if a.compare_diag:  # the V-trace + loss kernel alone, plain and diag entry points alternating
    import ctypes

    eng = engines["diagnostics on"]
    d = eng.d_views[0]
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    ins = (P(eng.logits), P(d["beh_logits"]), P(d["actions"]), P(d["rewards"]), P(d["done"]), P(d["lens"]),
           P(eng.values), P(eng.vs), P(eng.pg_adv), P(eng.dlogits), P(eng.dv))
    scal = ctypes.c_void_p(eng.comm.data_ptr() + 8 * eng.n_total)
    diag = ctypes.c_void_p(eng.comm.data_ptr() + 8 * (eng.n_total + 4))
    ws_plain = torch.zeros(int(eng.lib.impala_vtrace_loss_workspace(w["T"], w["B"], w["A"])), dtype=torch.uint8,
                           device="cuda")
    tail = (w["T"], w["B"], w["A"], hp.gamma, hp.rho_bar, hp.c_bar, hp.v_loss_c, hp.policy_loss_c, hp.entropy_c,
            1.0 / w["B"], 0)
    calls = {"impala_vtrace_loss": lambda st: eng.lib.impala_vtrace_loss(*ins, scal, P(ws_plain), ws_plain.numel(),
                                                                        *tail, st),
             "impala_vtrace_loss_diag": lambda st: eng.lib.impala_vtrace_loss_diag(*ins, scal, diag, P(eng.ws_vt),
                                                                                  eng.ws_vt_bytes, *tail, st)}
    tk = {name: [] for name in calls}
    with torch.cuda.stream(eng.stream):
        st = ctypes.c_void_p(eng.stream.cuda_stream)
        for i in range(220):
            for name, fn in calls.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(eng.stream)
                rc = fn(st)
                e1.record(eng.stream)
                e1.synchronize()
                assert rc == 0, (name, rc)
                if i >= 20:
                    tk[name].append(e0.elapsed_time(e1) * 1e3)
    k0, k1 = statistics.median(tk["impala_vtrace_loss"]), statistics.median(tk["impala_vtrace_loss_diag"])
    print(f"V-trace + loss kernel {a.config}: impala_vtrace_loss {k0:.1f} us, impala_vtrace_loss_diag {k1:.1f} us "
          f"(+{k1 - k0:.1f} us, {100 * (k1 / k0 - 1):+.1f} %)")
if a.compare_popart:  # the two launches PopArt changes, alone, plain and PopArt entry points alternating
    import ctypes

    from torched_impala_b200 import _cabi

    eng = engines["popart on"]
    d = eng.d_views[0]
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    ins = (P(eng.logits), P(d["beh_logits"]), P(d["actions"]), P(d["rewards"]), P(d["done"]), P(d["lens"]),
           P(eng.values), P(eng.vs), P(eng.pg_adv), P(eng.dlogits), P(eng.dv))
    scal = ctypes.c_void_p(eng.comm.data_ptr() + 8 * eng.n_total)
    diag = ctypes.c_void_p(eng.comm.data_ptr() + 8 * (eng.n_total + 4))
    tail = (w["T"], w["B"], w["A"], hp.gamma, hp.rho_bar, hp.c_bar, hp.v_loss_c, hp.policy_loss_c, hp.entropy_c,
            1.0 / w["B"], 0)
    # the optimizer on copies of the engine's state, so the timed launches do not move the engine
    cp = {k: getattr(eng, k).clone() for k in ("params", "adam_m", "adam_v", "adam_step", "popart_buf")}
    o = eng.optim
    rule = (P(eng.lr_table), eng.lr_table.numel(), o.rule_code, o.h0, o.h1, o.eps)
    opt_head = (P(cp["params"]), P(eng.comm), P(cp["adam_m"]), P(cp["adam_v"]), P(cp["adam_step"]), eng.n_pi,
                eng.n_total, float(hp.max_norm))
    calls = {"impala_vtrace_loss_diag": lambda st: eng.lib.impala_vtrace_loss_diag(*ins, scal, diag, P(eng.ws_vt),
                                                                                  eng.ws_vt_bytes, *tail, st),
             "impala_vtrace_loss_popart": lambda st: eng.lib.impala_vtrace_loss_popart(
                 *ins, scal, diag, P(eng.ws_vt), eng.ws_vt_bytes, *tail, P(eng.popart_buf), st),
             "impala_clip_optim": lambda st: eng.lib.impala_clip_optim(*opt_head, *rule, P(eng.norms), st),
             "impala_clip_optim_popart": lambda st: eng.lib.impala_clip_optim_popart(
                 *opt_head, *rule, P(eng.norms), P(cp["popart_buf"]), eng.n_total + 4, eng.w2_at, w["H"], eng.b2_at,
                 float(eng.popart_beta), st)}
    tk = {name: [] for name in calls}
    with torch.cuda.stream(eng.stream):
        st = ctypes.c_void_p(eng.stream.cuda_stream)
        for i in range(220):
            for name, fn in calls.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(eng.stream)
                rc = fn(st)
                e1.record(eng.stream)
                e1.synchronize()
                assert rc == 0, (name, rc)
                if i >= 20:
                    tk[name].append(e0.elapsed_time(e1) * 1e3)
    for plain, pop in (("impala_vtrace_loss_diag", "impala_vtrace_loss_popart"),
                       ("impala_clip_optim", "impala_clip_optim_popart")):
        k0, k1 = statistics.median(tk[plain]), statistics.median(tk[pop])
        print(f"{a.config}: {plain} {k0:.1f} us, {pop} {k1:.1f} us (+{k1 - k0:.1f} us, {100 * (k1 / k0 - 1):+.1f} %)")
if a.compare_reward_clip:  # the V-trace + loss kernel alone, without and with either transform, alternating
    import ctypes

    from torched_impala_b200 import _cabi

    eng = engines["reward_clip abs_one"]
    d = eng.d_views[0]
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    ins = (P(eng.logits), P(d["beh_logits"]), P(d["actions"]), P(d["rewards"]), P(d["done"]), P(d["lens"]),
           P(eng.values), P(eng.vs), P(eng.pg_adv), P(eng.dlogits), P(eng.dv),
           ctypes.c_void_p(eng.comm.data_ptr() + 8 * eng.n_total), P(eng.ws_vt), eng.ws_vt_bytes)
    tail = (w["T"], w["B"], w["A"], hp.gamma, hp.rho_bar, hp.c_bar, hp.v_loss_c, hp.policy_loss_c, hp.entropy_c,
            1.0 / w["B"], 0)
    calls = {"impala_vtrace_loss": lambda st: eng.lib.impala_vtrace_loss(*ins, *tail, st)}
    for rc_name, code in _cabi.REWARD_CLIPS.items():
        calls[f"impala_vtrace_loss_rclip {rc_name}"] = (
            lambda st, code=code: eng.lib.impala_vtrace_loss_rclip(*ins, *tail, None, None, code, st))
    tk = {name: [] for name in calls}
    with torch.cuda.stream(eng.stream):
        st = ctypes.c_void_p(eng.stream.cuda_stream)
        for i in range(220):
            for name, fn in calls.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(eng.stream)
                rc = fn(st)
                e1.record(eng.stream)
                e1.synchronize()
                assert rc == 0, (name, rc)
                if i >= 20:
                    tk[name].append(e0.elapsed_time(e1) * 1e3)
    k0 = statistics.median(tk["impala_vtrace_loss"])
    print(f"V-trace + loss kernel {a.config}: impala_vtrace_loss {k0:.1f} us", end="")
    for name in list(calls)[1:]:
        k1 = statistics.median(tk[name])
        print(f", {name} {k1:.1f} us ({k1 - k0:+.1f} us, {100 * (k1 / k0 - 1):+.1f} %)", end="")
    print()
if a.compare_heads:  # the V-trace + loss kernel alone, categorical against multi-discrete, each on its engine's buffers
    import ctypes

    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    tail = (w["T"], w["B"], w["A"], hp.gamma, hp.rho_bar, hp.c_bar, hp.v_loss_c, hp.policy_loss_c, hp.entropy_c,
            1.0 / w["B"], 0)

    def _ins(e):
        d = e.d_views[0]
        return (P(e.logits), P(d["beh_logits"]), P(d["actions"]), P(d["rewards"]), P(d["done"]), P(d["lens"]),
                P(e.values), P(e.vs), P(e.pg_adv), P(e.dlogits), P(e.dv), ctypes.c_void_p(e.comm.data_ptr() + 8 * e.n_total),
                P(e.ws_vt), e.ws_vt_bytes)

    ec, em = engines[list(arms)[0]], engines[md_name]
    hh = (ctypes.c_int32 * len(w["heads"]))(*w["heads"])
    calls = {"impala_vtrace_loss": lambda st: ec.lib.impala_vtrace_loss(*_ins(ec), *tail, st),
             "impala_vtrace_loss_md": lambda st: em.lib.impala_vtrace_loss_md(*_ins(em), *tail[:-1], tail[-1], None,
                                                                              None, 0, hh, len(w["heads"]), st)}
    tk = {name: [] for name in calls}
    with torch.cuda.stream(em.stream):
        st = ctypes.c_void_p(em.stream.cuda_stream)
        for i in range(220):
            for name, fn in calls.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(em.stream)
                rc = fn(st)
                e1.record(em.stream)
                e1.synchronize()
                assert rc == 0, (name, rc)
                if i >= 20:
                    tk[name].append(e0.elapsed_time(e1) * 1e3)
    k0, k1 = statistics.median(tk["impala_vtrace_loss"]), statistics.median(tk["impala_vtrace_loss_md"])
    print(f"V-trace + loss kernel {a.config}: impala_vtrace_loss (A={w['A']}) {k0:.1f} us, impala_vtrace_loss_md "
          f"(heads {w['heads']}) {k1:.1f} us ({k1 - k0:+.1f} us, {100 * (k1 / k0 - 1):+.1f} %)")
if a.compare_mask:  # the V-trace + loss kernel alone, unmasked against masked, each on its engine's buffers
    import ctypes

    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    tail = (w["T"], w["B"], w["A"], hp.gamma, hp.rho_bar, hp.c_bar, hp.v_loss_c, hp.policy_loss_c, hp.entropy_c,
            1.0 / w["B"], 0)

    def _ins(e):
        d = e.d_views[0]
        return (P(e.logits), P(d["beh_logits"]), P(d["actions"]), P(d["rewards"]), P(d["done"]), P(d["lens"]),
                P(e.values), P(e.vs), P(e.pg_adv), P(e.dlogits), P(e.dv), ctypes.c_void_p(e.comm.data_ptr() + 8 * e.n_total),
                P(e.ws_vt), e.ws_vt_bytes)

    eu, em = engines["unmasked"], engines[mask_name]
    K = len(w["mask"])
    hh = (ctypes.c_int32 * K)(*w["mask"]) if K else None
    plain_name = "impala_vtrace_loss_md" if K else "impala_vtrace_loss"
    calls = {plain_name: (lambda st: eu.lib.impala_vtrace_loss_md(*_ins(eu), *tail[:-1], tail[-1], None, None, 0, hh, K,
                                                                  st)) if K else
             (lambda st: eu.lib.impala_vtrace_loss(*_ins(eu), *tail, st)),
             "impala_vtrace_loss_mask": lambda st: em.lib.impala_vtrace_loss_mask(*_ins(em), *tail[:-1], tail[-1], None,
                                                                                  None, 0, hh, K, st)}
    tk = {name: [] for name in calls}
    with torch.cuda.stream(em.stream):
        st = ctypes.c_void_p(em.stream.cuda_stream)
        for i in range(220):
            for name, fn in calls.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(em.stream)
                rc = fn(st)
                e1.record(em.stream)
                e1.synchronize()
                assert rc == 0, (name, rc)
                if i >= 20:
                    tk[name].append(e0.elapsed_time(e1) * 1e3)
    k0, k1 = statistics.median(tk[plain_name]), statistics.median(tk["impala_vtrace_loss_mask"])
    print(f"V-trace + loss kernel {a.config}: {plain_name} {k0:.1f} us, impala_vtrace_loss_mask {k1:.1f} us "
          f"({k1 - k0:+.1f} us, {100 * (k1 / k0 - 1):+.1f} %)")
if a.compare_obs_norm:  # the normalize launch alone, on the engine's slab and buffers
    import ctypes

    from torched_impala_b200 import _cabi

    eng = engines["obs_norm on"]
    d = eng.d_views[0]
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    sums = ctypes.c_void_p(eng.comm.data_ptr() + 8 * eng.obs_sums_at)
    with torch.cuda.stream(eng.stream):
        st = ctypes.c_void_p(eng.stream.cuda_stream)
        tu = []
        for i in range(220):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(eng.stream)
            _cabi.check(eng.lib.impala_obs_normalize(P(d["obs"]), eng.obs_code, w["T"], w["B"], eng.F, eng.frames,
                                                     P(d["lens"]), P(eng.obs_norm_dev), P(eng.obs_normed), sums,
                                                     P(eng.obs_norm_ws), eng.obs_norm_ws.numel(), st),
                        "impala_obs_normalize")
            e1.record(eng.stream)
            e1.synchronize()
            if i >= 20:
                tu.append(e0.elapsed_time(e1) * 1e3)
    us = statistics.median(tu)
    nbytes = d["obs"].numel() * d["obs"].element_size() + eng.obs_normed.numel() * 4
    print(f"impala_obs_normalize {a.config} {a.obs_dtype}: {us:.1f} us, {nbytes / 1e6:.1f} MB moved, HBM floor "
          f"{nbytes / 3.35e12 * 1e6:.1f} us at 3.35 TB/s ({nbytes / 3.35e12 * 1e6 / us:.0%} of it)")
q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                    "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"GPU (nvidia-smi): {q}")
for name, eng in engines.items():
    med = statistics.median(ts[name])
    e2e = f", pinned-slab end to end {statistics.median(te[name]):.1f} us/step, slab {eng.slab_bytes / 1e6:.1f} MB" \
        if te[name] else ""
    print(f"{a.config} {w} [{name}] on {dev}: median {med:.1f} us/step ({1e6 / med:.0f} steps/s){e2e}, "
          f"loss {eng.read_scalars()['total_loss']:.5f}")
if a.compare_replay:
    m0, m1 = statistics.median(ts["replay off"]), statistics.median(ts[on])
    print(f"replay overhead {a.config}: {m1 - m0:+.1f} us/step ({100 * (m1 / m0 - 1):+.1f} %), one launch more "
          f"({engines[on].launches_per_step} against {engines['replay off'].launches_per_step})")
if a.compare_diag:
    m0, m1 = statistics.median(ts["diagnostics off"]), statistics.median(ts["diagnostics on"])
    sc = engines["diagnostics on"].read_scalars()
    print(f"diagnostics overhead {a.config}: {m1 - m0:+.1f} us/step ({100 * (m1 / m0 - 1):+.1f} %); "
          f"rho clipped {100 * sc['rho_clip_fraction']:.1f} %, kl {sc['kl_behaviour_current']:.4f}, "
          f"explained variance {sc['value_explained_variance']:.4f}")
if a.compare_popart:
    m0, m1 = statistics.median(ts["popart off"]), statistics.median(ts["popart on"])
    st = engines["popart on"].popart_stats()
    print(f"popart overhead {a.config}: {m1 - m0:+.1f} us/step ({100 * (m1 / m0 - 1):+.1f} %), launches "
          f"{engines['popart on'].launches_per_step} against {engines['popart off'].launches_per_step}; "
          f"mu {st['mu']:.4f}, sigma {st['sigma']:.4f}")
if a.compare_reward_clip:
    m0 = statistics.median(ts["reward_clip None"])
    for name in list(arms)[1:]:
        m1 = statistics.median(ts[name])
        print(f"{name} overhead {a.config}: {m1 - m0:+.1f} us/step ({100 * (m1 / m0 - 1):+.1f} %), launches "
              f"{engines[name].launches_per_step} against {engines['reward_clip None'].launches_per_step}")
if a.compare_shared:
    m0, m1 = statistics.median(ts["two networks"]), statistics.median(ts["shared torso"])
    print(f"shared torso {a.config}: {m1:.1f} us/step against {m0:.1f} ({m1 - m0:+.1f} us, {100 * (m1 / m0 - 1):+.1f} %), "
          f"launches {engines['shared torso'].launches_per_step} against {engines['two networks'].launches_per_step}")
if a.compare_heads:
    m0, m1 = statistics.median(ts[list(arms)[0]]), statistics.median(ts[md_name])
    print(f"multi-discrete {a.config}: {m1:.1f} us/step against {m0:.1f} ({m1 - m0:+.1f} us, {100 * (m1 / m0 - 1):+.1f} %), "
          f"launches {engines[md_name].launches_per_step} against {engines[list(arms)[0]].launches_per_step}")
if a.compare_mask:
    m0, m1 = statistics.median(ts["unmasked"]), statistics.median(ts[mask_name])
    print(f"masked {a.config}: {m1:.1f} us/step against {m0:.1f} ({m1 - m0:+.1f} us, {100 * (m1 / m0 - 1):+.1f} %), "
          f"launches {engines[mask_name].launches_per_step} against {engines['unmasked'].launches_per_step}")
if a.compare_obs_norm:
    m0, m1 = statistics.median(ts["obs_norm off"]), statistics.median(ts["obs_norm on"])
    st = engines["obs_norm on"].obs_norm_stats()
    print(f"obs_norm {a.config} {a.obs_dtype}: {m1:.1f} us/step against {m0:.1f} ({m1 - m0:+.1f} us, "
          f"{100 * (m1 / m0 - 1):+.1f} %), launches {engines['obs_norm on'].launches_per_step} against "
          f"{engines['obs_norm off'].launches_per_step}; rows counted {st['count']:.0f}")
