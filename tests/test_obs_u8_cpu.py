"""CPU: byte observations (uint8 slabs and the K-streamed MLP kernels that read bytes).

Slab layout and shard-ingest ABI, the ring's pure-python layout mirror, the integer check of the
trajectory packers, the refused shapes of impala_mlp_{forward,backward}_u8, and the SASS of the byte
instantiations (16 HGMMA per chunk against the float kernels' 24, one warpgroup wait, no local memory)."""
import ctypes as C
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

from torched_impala_b200 import _cabi, synth
from torched_impala_b200.learner import pack_trajectory
from torched_impala_b200.ring import RingQueue, _layout

SHAPES = [(20, 4096, 128, 18), (20, 4096, 512, 18), (20, 4096, 400, 6), (1, 1, 1, 1), (7, 13, 33, 5),
          (100, 8192, 64, 4)]


def _layout_obs(T, B, O, A, code):
    offs, total = (C.c_int64 * 6)(), C.c_int64()
    rc = _cabi.lib().impala_batch_layout_obs(T, B, O, A, code, offs, C.byref(total))
    return rc, list(offs), total.value


@pytest.mark.parametrize("shape", SHAPES)
def test_layout_obs_f32_equals_batch_layout(shape):
    rc, offs, total = _layout_obs(*shape, _cabi.OBS_F32)
    assert rc == 0
    assert (offs, total) == tuple(_cabi.batch_layout(*shape))


@pytest.mark.parametrize("shape", SHAPES)
def test_layout_obs_u8_takes_one_byte_per_value(shape):
    T, B, O, A = shape
    rc, offs, total = _layout_obs(*shape, _cabi.OBS_U8)
    assert rc == 0 and offs[0] == 0
    assert offs[1] == (T + 1) * B * O + 255 & ~255  # obs: (T+1) B O bytes, then 256-byte alignment
    f_offs, f_total = _cabi.batch_layout(*shape)
    shift = f_offs[1] - offs[1]
    assert [o + shift for o in offs[1:]] == f_offs[1:] and total + shift == f_total  # the rest is unchanged


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_ring_layout_mirror_matches_c(shape, obs_dtype):
    assert _layout(*shape, obs_dtype) == tuple(_cabi.batch_layout(*shape, obs_dtype))


@pytest.mark.parametrize("code", [-1, 2, 7])
def test_bad_obs_dtype_is_refused(code):
    assert _layout_obs(4, 4, 4, 2, code)[0] == -1  # IMPALA_ERR_BAD_ARG
    buf = (C.c_uint8 * 4096)()
    assert _cabi.lib().impala_ingest_shard_obs(buf, buf, 4, 4, 4, 2, code, 0, 2, None) == -1
    with pytest.raises(ValueError):
        _layout(4, 4, 4, 2, "int8")


def _views(T, B, O, A, obs_dtype):
    offs, total = _layout(T, B, O, A, obs_dtype)
    buf = np.zeros(total, np.uint8)
    dts = [np.dtype(t) for t in (obs_dtype, np.float32, np.int32, np.float32, np.uint8, np.int32)]
    shapes = ((T + 1, B, O), (T, B, A), (T, B), (T, B), (T, B), (B,))
    names = ("obs", "beh_logits", "actions", "rewards", "done", "lens")
    return {n: buf[o:o + int(np.prod(s)) * dt.itemsize].view(dt).reshape(s)
            for n, o, s, dt in zip(names, offs, shapes, dts)}


def _trajs(T, B, O, A, kind="bytes"):
    batch = synth.make_batch(3, T, B, O, A, ragged=True, obs_kind=kind)
    return batch, synth.to_trajectories(batch)


@pytest.mark.parametrize("kind", ["bytes", "planes"])
def test_pack_trajectory_u8_is_byte_exact(kind):
    T, B, O, A = 6, 5, 12, 3
    batch, trs = _trajs(T, B, O, A, kind)
    v = _views(T, B, O, A, "uint8")
    for b, tr in enumerate(trs):
        pack_trajectory(v, b, tr, T)
    assert v["obs"].dtype == np.uint8 and np.array_equal(v["obs"], batch["obs"])
    assert np.array_equal(v["lens"], batch["lens"])


@pytest.mark.parametrize("bad", [0.5, -1.0, 256.0, float("nan")])
def test_pack_trajectory_u8_refuses_non_bytes(bad):
    T, B, O, A = 6, 2, 8, 3
    _, trs = _trajs(T, B, O, A)
    trs[0].obs[1] = trs[0].obs[1].clone()
    trs[0].obs[1][3] = bad
    with pytest.raises(ValueError, match="uint8"):
        pack_trajectory(_views(T, B, O, A, "uint8"), 0, trs[0], T)
    pack_trajectory(_views(T, B, O, A, "float32"), 0, trs[0], T)  # a float32 slab takes any value


def test_ring_put_u8_exact_and_refuses_non_bytes():
    T, B, O, A = 6, 4, 12, 3
    batch, trs = _trajs(T, B, O, A)
    q = RingQueue(T, B, O, A, slabs=2, obs_dtype="uint8")
    try:
        assert q.slab_bytes == _layout(T, B, O, A, "uint8")[1]
        for bad in (0.5, -1.0, 256.0):
            tr = _trajs(T, B, O, A)[1][0]
            tr.obs[0] = tr.obs[0].clone()
            tr.obs[0][0] = bad
            with pytest.raises(ValueError, match="uint8"):
                q.put(tr, timeout=1)
        assert int(q._control()["ticket"][0]) == 0  # refused before a column was taken
        for tr in trs:
            q.put(tr, timeout=1)
        k, _ = q.collect_batch(timeout=1)
        assert np.array_equal(q.views(k)["obs"], batch["obs"])
        with pytest.raises(ValueError, match="uint8"):
            q.put_block({**batch, "obs": batch["obs"].astype(np.float32)}, timeout=1)
    finally:
        q.close()


def test_learner_checks_ring_obs_dtype():
    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpPolicy, MlpValueFn
    from torched_impala_b200.utils import Counter as SharedCounter, default_hparams

    T, B, O, A = 5, 4, 8, 2
    hp = default_hparams(batch_size=B, max_timesteps=T, log_path=None)
    q = RingQueue(T, B, O, A, slabs=2, obs_dtype="uint8")
    try:
        with pytest.raises(ValueError, match="uint8"):
            Learner(1, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), q, SharedCounter(0))
        lrn = Learner(2, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), q, SharedCounter(0), obs_dtype="uint8")
        assert lrn._cfg()["obs_dtype"] == "uint8"
    finally:
        q.close()
    with pytest.raises(ValueError):
        Learner(3, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), None, SharedCounter(0), obs_dtype="float16")


def test_synth_integer_batches():
    n = synth.make_batch(4, 5, 6, 128, 3, ragged=True)
    for kind, hi in (("bytes", 255), ("planes", 1)):
        b = synth.make_batch(4, 5, 6, 128, 3, ragged=True, obs_kind=kind)
        assert b["obs"].dtype == np.uint8 and int(b["obs"].max()) == hi and int(b["obs"].min()) == 0
        for k in ("beh_logits", "actions", "rewards", "done", "lens"):
            assert np.array_equal(b[k], n[k])
        pad = np.arange(6)[:, None] > b["lens"][None, :]
        assert not b["obs"][pad].any()


@pytest.mark.parametrize("M,O,H,N2", [(81920, 512, 256, 18), (86016, 400, 256, 1), (5, 132, 128, 32),
                                      (1, 1024, 1024, 6)])
def test_u8_workspace_equals_f32(M, O, H, N2):
    """impala_mlp_backward_workspace sizes both: the byte backward wants exactly the float workspace."""
    lib = _cabi.lib()
    need = lib.impala_mlp_backward_workspace(M, O, H, N2)
    assert need > 0
    buf = (C.c_uint8 * 64)()  # never read: the size check comes before any launch
    assert lib.impala_mlp_backward_u8(buf, buf, buf, buf, buf, need - 1, M, O, H, N2, None) == -3
    assert lib.impala_mlp_backward(buf, buf, buf, buf, buf, need - 1, M, O, H, N2, None) == -3


# test_obs_wide_cpu.py's refused shapes, and the float-only shapes O <= 128
REFUSED = [(130, 256, 6, {}), (1028, 256, 6, {}), (512, 320, 6, {}), (512, 1152, 6, {}), (512, 256, 33, {}),
           (512, 256, 6, {"IMPALA_MLP_TC": "0"}), (512, 256, 6, {"IMPALA_MLP_TCW": "0"}),
           (128, 256, 18, {}), (24, 256, 4, {}), (64, 512, 4, {})]


@pytest.mark.parametrize("O,H,N2,env", REFUSED)
def test_u8_entry_points_refuse(monkeypatch, O, H, N2, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    lib = _cabi.lib()
    buf = (C.c_uint8 * 64)()  # never read: the shape check comes first
    assert lib.impala_mlp_forward_u8(buf, buf, buf, 1000, O, H, N2, None) == -2
    assert lib.impala_mlp_backward_u8(buf, buf, buf, buf, buf, 1 << 30, 1000, O, H, N2, None) == -2


def test_u8_entry_points_refuse_null():
    lib = _cabi.lib()
    assert lib.impala_mlp_forward_u8(None, None, None, 1000, 512, 256, 18, None) == -1
    assert lib.impala_obs_u8_to_f32(None, None, 10, None) == -1


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


# (mangled-name fragment of the byte instance, of the float instance)
OBS_KERNELS = [("mlp_fwd_obs_kernelILi1EhE", "mlp_fwd_obs_kernelILi1EfE"),
               ("mlp_fwd_obs_kernelILi4EhE", "mlp_fwd_obs_kernelILi4EfE"),
               ("mlp_fwd_obs_kernelILi32EhE", "mlp_fwd_obs_kernelILi32EfE"),
               ("mlp_bwd_obs_pre_kernelILi1EhE", "mlp_bwd_obs_pre_kernelILi1EfE"),
               ("mlp_bwd_obs_pre_kernelILi4EhE", "mlp_bwd_obs_pre_kernelILi4EfE"),
               ("mlp_bwd_obs_pre_kernelILi32EhE", "mlp_bwd_obs_pre_kernelILi32EfE"),
               ("mlp_bwd_obs_dw1_kernelIhE", "mlp_bwd_obs_dw1_kernelIfE")]


def _one(sass, frag):
    hits = [ops for name, ops in sass.items() if frag in name]
    assert len(hits) == 1, (frag, len(hits))
    return hits[0]


@pytest.mark.parametrize("u8,f32", OBS_KERNELS)
def test_u8_obs_kernels_issue_two_thirds_of_the_mmas(sass_by_kernel, u8, f32):
    ops_u8, ops_f32 = _one(sass_by_kernel, u8), _one(sass_by_kernel, f32)
    waits = lambda ops: sum(n for k, n in ops.items() if k.startswith("WARPGROUP.DEPBAR"))  # noqa: E731
    assert ops_u8["HGMMA"] == 16 and waits(ops_u8) == 1, (u8, ops_u8["HGMMA"], waits(ops_u8))
    assert ops_f32["HGMMA"] == 24 and waits(ops_f32) == 1, (f32, ops_f32["HGMMA"], waits(ops_f32))
    assert ops_u8["LDL"] == 0 and ops_u8["STL"] == 0


def test_widening_kernel_is_built(sass_by_kernel):
    assert any("obs_u8_to_f32_kernel" in name for name in sass_by_kernel)


def test_ops_wrappers_take_uint8_only():
    from torched_impala_b200 import ops

    with pytest.raises(_cabi.ImpalaCudaError):  # CPU tensors: refused before any launch
        ops.mlp_forward_u8(torch.zeros(4, 132, dtype=torch.uint8), torch.zeros(4), 132, 128, 1)
