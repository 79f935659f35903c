"""GPU: byte observations end to end, held to value identity with the float32 path.

Every result on uint8 observations must be torch.equal to the float32 path run on the same values converted
to float: the byte kernels drop only MMAs whose products are exactly zero (x_lo = 0) and keep the order of
the rest.  Checked for the K-streamed kernels directly (forward and backward, M not a multiple of 64, bytes
0..255 and 0/1 planes), for whole learner updates with graph replay (u8 slabs against f32 slabs), for the
widened O <= 128 path, for shard ingest, against the float64 oracle at MinAtar and for the forked Learner.
"""
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


def make_x(rng, M, O, kind):
    if kind == "planes":
        return (rng.random((M, O)) < 0.3).astype(np.uint8)
    return rng.integers(0, 256, (M, O), dtype=np.uint8)


@pytest.mark.parametrize("N2", [1, 6, 18, 32])
@pytest.mark.parametrize("H", [128, 256, 1024])
@pytest.mark.parametrize("O", [132, 400, 512, 1000, 1024])
def test_u8_kernels_equal_float_kernels(ops, O, H, N2):
    M = 1000 + O % 61  # not a multiple of 64
    p = synth.init_params(O + H + N2, O, N2, H)["policy"]
    params = ops.pack_params(p)
    for kind in ("bytes", "planes"):
        rng = np.random.default_rng(O * H + N2 + len(kind))
        x8 = torch.from_numpy(make_x(rng, M, O, kind)).cuda()
        xf = x8.float()
        dout = torch.from_numpy(rng.standard_normal((M, N2), dtype=np.float32) / M).cuda()
        got = ops.mlp_forward_u8(x8, params, O, H, N2)
        want = ops.mlp_forward(xf, params, O, H, N2)
        assert torch.equal(got, want), (kind, float((got - want).abs().max()))
        g8 = ops.mlp_backward_u8(x8, params, dout, O, H, N2)
        gf = ops.mlp_backward(xf, params, dout, O, H, N2)
        assert torch.equal(g8, gf), (kind, float((g8 - gf).abs().max()))
        assert not torch.isnan(g8).any()


def test_u8_widening_is_exact(ops):
    for n, off in ((1, 0), (4099, 0), (1 << 20, 0), (777, 1), (4096, 3)):
        x = torch.randint(0, 256, (n + off,), dtype=torch.uint8, device="cuda")[off:]
        assert torch.equal(ops.obs_u8_to_f32(x), x.float())


# name: (T, B, O, A, H, ragged, obs_kind, env)
ENGINE_CASES = {
    "ram": (20, 4096, 128, 18, 256, False, "bytes", {}),
    "ram4": (20, 4096, 512, 18, 256, False, "bytes", {}),
    "minatar": (20, 4096, 400, 6, 256, False, "planes", {}),
    "minatar_ragged": (20, 1024, 400, 6, 256, True, "planes", {}),
    "c4_shaped": (20, 1024, 24, 4, 256, True, "bytes", {}),
    "c5_shaped": (10, 1024, 64, 4, 512, True, "bytes", {}),
    "ram_fp32_kernels": (20, 512, 128, 18, 256, True, "bytes", {"IMPALA_MLP_TC": "0"}),
}


def _run_engine(obs_dtype, T, B, O, A, H, hp, params, batches):
    from torched_impala_b200.engine import LearnerEngine

    eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=True, obs_dtype=obs_dtype)
    eng.load_state(params)
    scal = []
    for u in range(4):
        b = batches[u % 2]
        eng.fill_host(b if obs_dtype == "uint8" else {**b, "obs": b["obs"].astype(np.float32)}, u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        scal.append(eng.read_scalars())
    eng.synchronize()
    return eng, eng.params.clone(), scal


@pytest.mark.parametrize("name", list(ENGINE_CASES))
def test_u8_engine_equals_f32_engine(ops, monkeypatch, name):
    T, B, O, A, H, ragged, kind, env = ENGINE_CASES[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(31, O, A, H)
    batches = [synth.make_batch(50 + i, T, B, O, A, ragged=ragged, obs_kind=kind) for i in range(2)]
    e8, p8, s8 = _run_engine("uint8", T, B, O, A, H, hp, params, batches)
    ef, pf, sf = _run_engine("float32", T, B, O, A, H, hp, params, batches)
    assert e8.slab_bytes < ef.slab_bytes and e8.d["obs"].dtype == torch.uint8
    assert e8.launches_per_step == ef.launches_per_step + (1 if O <= 128 else 0), (e8.launches_per_step,
                                                                                  ef.launches_per_step)
    assert torch.equal(p8, pf), float((p8 - pf).abs().max())
    assert s8 == sf
    assert torch.equal(e8.adam_m, ef.adam_m) and torch.equal(e8.adam_v, ef.adam_v)


def test_u8_first_step_matches_oracle_minatar_planes():
    """MinAtar (O400 A6) with 0/1 planes, ragged: thresholds of test_gpu_obs_wide.py."""
    from torched_impala_b200.engine import LearnerEngine

    T, B, O, A, H = 20, 1024, 400, 6, 256
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(11, O, A, H)
    batch = synth.make_batch(17, T, B, O, A, ragged=True, obs_kind="planes")
    eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=False, obs_dtype="uint8")
    par = first_step_parity(eng, params, batch)
    print("minatar planes u8", json.dumps(par))
    assert par["max_abs_vs"] < 1e-5, par
    assert par["max_abs_pg"] < 1e-5, par
    for k, v in par["scalars"].items():
        assert v["abs_err"] < 1e-5, (k, v)
    check_engine_mlp(eng, params)
    if par["max_rel_grad"] >= 5e-5:
        check_grad_end_to_end(eng, params, batch, hp)
    assert par["max_abs_param_after_1_update"] < 5e-5, par
    assert par["frac_params_off"] < 1e-3, par
    for k in ("norm_policy", "norm_value"):
        assert abs(par[k]["got"] - par[k]["ref"]) < 5e-5 * max(1.0, par[k]["ref"]), par


def _shard_results(obs_dtype, devices, T, B, O, A, H, hp, params, batch):
    """Each rank's engine DMAs its column range of one pinned host slab laid out for the full batch."""
    from torched_impala_b200.engine import LearnerEngine

    offs, total = _cabi.batch_layout(T, B, O, A, obs_dtype)
    host = torch.zeros(total, dtype=torch.uint8).pin_memory()
    arr = host.numpy()
    dts = (np.dtype(obs_dtype), np.float32, np.int32, np.float32, np.uint8, np.int32)
    for (name, v), off, dt in zip(((k, batch[k]) for k in ("obs", "beh_logits", "actions", "rewards", "done",
                                                           "lens")), offs, dts):
        a = np.ascontiguousarray(v).astype(dt)
        arr[off:off + a.nbytes] = a.view(np.uint8).reshape(-1)
    out = []
    world = len(devices)
    for r, dev in enumerate(devices):
        eng = LearnerEngine(T, B // world, O, A, H, H, hp, global_batch=B, device=dev, use_graph=False,
                            obs_dtype=obs_dtype)
        eng.load_state(params)
        eng.ingest_shard_from(host.data_ptr(), r * (B // world), B, 0)
        eng.step(0)
        eng.synchronize()
        out.append((eng.comm.clone().cpu(), eng.params.clone().cpu()))
    return out


@pytest.mark.parametrize("two_gpus", [False, True])
@pytest.mark.parametrize("O", [128, 400])
def test_u8_shard_ingest_equals_f32(ops, O, two_gpus):
    """Both ranks' column shards of one host slab (rank r's gradient and scalars in its `comm`): on one
    GPU, and with the ranks on two GPUs when there are two."""
    if two_gpus and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    T, B, A, H = 20, 512, 6, 256
    devices = ["cuda:0", "cuda:1" if two_gpus else "cuda:0"]
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    params = synth.init_params(41, O, A, H)
    batch = synth.make_batch(43, T, B, O, A, ragged=True, obs_kind="bytes")
    got = _shard_results("uint8", devices, T, B, O, A, H, hp, params, batch)
    want = _shard_results("float32", devices, T, B, O, A, H, hp, params, batch)
    for (c8, p8), (cf, pf) in zip(got, want):
        assert torch.equal(c8, cf) and torch.equal(p8, pf)


@pytest.mark.parametrize("O,A,H", [(400, 6, 256), (128, 18, 256)])
def test_u8_learner_process_ring(O, A, H):
    """Forked Learner(obs_dtype="uint8") behind a uint8 RingQueue == the float32 Learner on the same data."""
    script = os.path.join(os.path.dirname(__file__), "obs_u8_learner_process_check.py")
    res = subprocess.run([sys.executable, script, str(O), str(A), str(H)], capture_output=True, text=True,
                         timeout=400)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "OBS_U8_LEARNER_OK" in res.stdout
