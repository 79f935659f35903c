"""GPU: frame-stacked observations stored once per frame, held to value identity with the dense path.

impala_obs_unstack against numpy for every dtype pair; whole learner updates with graph replay of a frame
engine against the dense engine fed synth.stack_frames of the same batch; the first step against the float64
oracle; shard ingest of a frame slab; and the forked Learner on a frame ring against a dense ring, whose
padded observation rows differ (zero there, shared frames here) and must not matter."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.check import first_step_parity
from test_gpu_wide_shapes import check_engine_mlp, check_grad_end_to_end
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


PAIRS = [(torch.uint8, torch.uint8), (torch.uint8, torch.float32), (torch.float32, torch.float32)]


@pytest.mark.parametrize("k", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("F", [1, 3, 6, 16, 32, 100, 128])
@pytest.mark.parametrize("pair", PAIRS, ids=["u8-u8", "u8-f32", "f32-f32"])
def test_unstack_equals_numpy(ops, pair, F, k):
    R, B = 21, 37
    rng = np.random.default_rng(F * 10 + k)
    fr = rng.integers(0, 256, (R + k - 1, B, F), dtype=np.uint8) if pair[0] == torch.uint8 else \
        rng.standard_normal((R + k - 1, B, F), dtype=np.float32)
    want = torch.from_numpy(synth.stack_frames({"obs": fr}, k)["obs"]).to(pair[1])
    got = ops.obs_unstack(torch.from_numpy(fr).cuda(), k, pair[1])
    assert torch.equal(got.cpu(), want)


def test_unstack_unaligned_pointers_take_the_element_path(ops):
    fr = torch.randint(0, 256, (1 + 5 * 33 * 32,), dtype=torch.uint8, device="cuda")[1:].view(5, 33, 32)
    want = torch.from_numpy(synth.stack_frames({"obs": fr.cpu().numpy()}, 4)["obs"])
    for dt in (torch.uint8, torch.float32):
        assert torch.equal(ops.obs_unstack(fr, 4, dt).cpu(), want.to(dt))


# name: (T, B, O, frames, A, H, ragged, obs_dtype, env)
ENGINE_CASES = {
    "ram4_u8": (20, 4096, 512, 4, 18, 256, False, "uint8", {}),
    "ram4_f32": (20, 4096, 512, 4, 18, 256, False, "float32", {}),
    "ram8_u8_B1024": (20, 1024, 1024, 8, 18, 256, False, "uint8", {}),
    "o128_u8_ragged": (20, 1024, 128, 4, 18, 256, True, "uint8", {}),
    "o24_f32_ragged": (20, 1024, 24, 4, 4, 256, True, "float32", {}),
    "o128_u8_fp32_kernels": (20, 512, 128, 4, 18, 256, True, "uint8", {"IMPALA_MLP_TC": "0"}),
}


def _run_engine(frames, obs_dtype, T, B, O, A, H, hp, params, batches):
    from torched_impala_b200.engine import LearnerEngine

    eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=True, obs_dtype=obs_dtype, frames=frames)
    eng.load_state(params)
    scal, outs = [], []
    for u in range(4):
        eng.fill_host(batches[u % 2], u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        scal.append(eng.read_scalars())
        outs.append([t.clone() for t in (eng.logits, eng.values, eng.vs, eng.pg_adv)])
    eng.synchronize()
    return eng, eng.params.clone(), scal, outs


@pytest.mark.parametrize("name", list(ENGINE_CASES))
def test_frame_engine_equals_dense_engine(ops, monkeypatch, name):
    T, B, O, k, A, H, ragged, obs_dtype, env = ENGINE_CASES[name]
    for key, v in env.items():
        monkeypatch.setenv(key, v)
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(31, O, A, H)
    kind = "bytes" if obs_dtype == "uint8" else "normal"
    fbs = [synth.make_batch(50 + i, T, B, O, A, ragged=ragged, obs_kind=kind, frames=k) for i in range(2)]
    ef, pf, sf, of = _run_engine(k, obs_dtype, T, B, O, A, H, hp, params, fbs)
    ed, pd, sd, od = _run_engine(1, obs_dtype, T, B, O, A, H, hp, params, [synth.stack_frames(b, k) for b in fbs])
    assert ef.slab_bytes < ed.slab_bytes and ef.d["obs"].shape == (T + k, B, O // k)
    extra = 0 if obs_dtype == "uint8" and O <= 128 else 1  # the unstacking replaces the widening launch there
    assert ef.launches_per_step == ed.launches_per_step + extra, (ef.launches_per_step, ed.launches_per_step)
    assert torch.equal(pf, pd), float((pf - pd).abs().max())
    assert sf == sd
    for u, (a, b) in enumerate(zip(of, od)):
        for what, x, y in zip(("logits", "values", "vs", "pg_adv"), a, b):
            assert torch.equal(x, y), (u, what)
    assert torch.equal(ef.adam_m, ed.adam_m) and torch.equal(ef.adam_v, ed.adam_v)


def _dense_fed_frame_engine(*args, **kw):
    """A frame engine whose fill_host takes the dense batch the oracle runs on and stores its frames: obs[0]
    split into its k frames, then the newest frame of every later row.  Lossless for full-length batches (every
    row is a valid observation), which the caller checks."""
    from torched_impala_b200.engine import LearnerEngine

    class DenseFed(LearnerEngine):
        def fill_host(self, batch, slot=0):
            obs, k, F = batch["obs"], self.frames, self.F
            frames = np.concatenate([obs[0].reshape(-1, k, F).transpose(1, 0, 2), obs[1:, :, (k - 1) * F:]], axis=0)
            assert np.array_equal(synth.stack_frames({"obs": frames}, k)["obs"], obs)
            super().fill_host({**batch, "obs": np.ascontiguousarray(frames)}, slot)

    return DenseFed(*args, **kw)


def test_ram4_u8_frames_first_step_matches_oracle():
    """ram4 with byte frames against the float64 oracle, at the thresholds of test_gpu_obs_u8.py's oracle check.
    0/1 planes, as there: with 0..255 values at O512 the values are of order 1e3, and float32 rounding of
    them alone exceeds 1e-5 absolute on any path (the frame engine equals the dense engine bit for bit,
    test_frame_engine_equals_dense_engine)."""
    T, B, O, k, A, H = 20, 4096, 512, 4, 18, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(11, O, A, H)
    dense = synth.stack_frames(synth.make_batch(17, T, B, O, A, obs_kind="planes", frames=k), k)
    eng = _dense_fed_frame_engine(T, B, O, A, H, H, hp, use_graph=False, obs_dtype="uint8", frames=k)
    par = first_step_parity(eng, params, dense)
    assert eng.d["obs"].shape == (T + k, B, O // k)
    print("ram4 u8 frames", json.dumps(par))
    assert par["max_abs_vs"] < 1e-5, par
    assert par["max_abs_pg"] < 1e-5, par
    for key, v in par["scalars"].items():
        assert v["abs_err"] < 1e-5 * max(1.0, abs(v["ref"])), (key, v)
    check_engine_mlp(eng, params)
    if par["max_rel_grad"] >= 5e-5:
        check_grad_end_to_end(eng, params, dense, hp)
    assert par["max_abs_param_after_1_update"] < 5e-5, par
    assert par["frac_params_off"] < 1e-3, par


def _shard_results(frames, devices, T, B, O, A, H, hp, params, batch):
    """Each rank's engine DMAs its column range of one pinned host slab laid out for the full batch."""
    from torched_impala_b200.engine import LearnerEngine

    offs, total = _cabi.batch_layout(T, B, O, A, "uint8", frames)
    host = torch.zeros(total, dtype=torch.uint8).pin_memory()
    arr = host.numpy()
    dts = (np.uint8, np.float32, np.int32, np.float32, np.uint8, np.int32)
    for name, off, dt in zip(("obs", "beh_logits", "actions", "rewards", "done", "lens"), offs, dts):
        a = np.ascontiguousarray(batch[name]).astype(dt)
        arr[off:off + a.nbytes] = a.view(np.uint8).reshape(-1)
    out = []
    world = len(devices)
    for r, dev in enumerate(devices):
        eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=dev, use_graph=False,
                            obs_dtype="uint8", frames=frames)
        eng.load_state(params)
        eng.ingest_shard_from(host.data_ptr(), r * (B // world), B, 0)
        eng.synchronize()
        lo, hi = r * (B // world), (r + 1) * (B // world)
        for name in ("obs", "beh_logits", "actions", "rewards", "done"):
            assert np.array_equal(eng.d[name].cpu().numpy(), np.asarray(batch[name])[:, lo:hi]), (r, name)
        assert np.array_equal(eng.d["lens"].cpu().numpy(), batch["lens"][lo:hi])
        eng.step(0)
        eng.synchronize()
        out.append((eng.comm.clone().cpu(), eng.params.clone().cpu()))
    return out


@pytest.mark.parametrize("two_gpus", [False, True])
def test_frame_shard_ingest(ops, two_gpus):
    """Both halves of a frame host slab land as the column slices, and each rank's gradient and scalars equal
    the dense slab's; on one GPU, and with the ranks on two GPUs when there are two."""
    if two_gpus and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    T, B, O, k, A, H = 20, 512, 512, 4, 18, 256
    devices = ["cuda:0", "cuda:1" if two_gpus else "cuda:0"]
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(41, O, A, H)
    fb = synth.make_batch(43, T, B, O, A, ragged=True, obs_kind="bytes", frames=k)
    got = _shard_results(k, devices, T, B, O, A, H, hp, params, fb)
    want = _shard_results(1, devices, T, B, O, A, H, hp, params, synth.stack_frames(fb, k))
    for (cf, pf), (cd, pd) in zip(got, want):
        assert torch.equal(cf, cd) and torch.equal(pf, pd)


def _learner_check(*args):
    script = os.path.join(os.path.dirname(__file__), "frames_learner_process_check.py")
    res = subprocess.run([sys.executable, script, *map(str, args)], capture_output=True, text=True, timeout=500)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "FRAMES_LEARNER_OK" in res.stdout


@pytest.mark.parametrize("O,k,A,H,obs_dtype", [(512, 4, 18, 256, "uint8"), (24, 4, 4, 256, "float32")])
def test_frames_learner_process_ring(O, k, A, H, obs_dtype):
    """Forked Learner(frames=k) behind a frame RingQueue == the dense Learner on the same trajectories."""
    _learner_check(O, k, A, H, obs_dtype, 1)


def test_frames_learner_data_parallel_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    _learner_check(512, 4, 18, 256, "uint8", 2)
