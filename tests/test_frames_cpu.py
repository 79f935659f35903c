"""CPU: frame-stacked observations stored once per frame.

Slab layout and shard-ingest ABI of impala_batch_layout_frames against the ring's pure-python mirror, the
argument checks of the three new entry points, the trajectory packer's frame split and overlap check (through
RingQueue.put), the Learner's frames checks, synth's frame batches, and ptxas's resource report of the
unstacking kernel."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from torched_impala_b200 import _cabi, synth
from torched_impala_b200.learner import pack_trajectory
from torched_impala_b200.ring import RingQueue, _layout

# (T, B, F, frames, A)
SHAPES = [(20, 4096, 128, 4, 18), (20, 4096, 128, 8, 18), (1, 1, 1, 1, 1), (1, 1, 1, 3, 1), (7, 13, 6, 4, 5),
          (20, 1024, 3, 8, 4), (100, 8192, 16, 4, 4)]


def _layout_frames(T, B, F, k, A, code):
    offs, total = (C.c_int64 * 6)(), C.c_int64()
    rc = _cabi.lib().impala_batch_layout_frames(T, B, F, k, A, code, offs, C.byref(total))
    return rc, list(offs), total.value


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_frames_layout_equals_ring_mirror(shape, obs_dtype):
    T, B, F, k, A = shape
    rc, offs, total = _layout_frames(T, B, F, k, A, _cabi.OBS_DTYPES[obs_dtype])
    assert rc == 0
    assert (offs, total) == _layout(T, B, k * F, A, obs_dtype, k)
    assert (offs, total) == tuple(_cabi.batch_layout(T, B, k * F, A, obs_dtype, k))
    assert offs[1] == (T + k) * B * F * np.dtype(obs_dtype).itemsize + 255 & ~255


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_one_frame_is_the_obs_layout(shape, obs_dtype):
    T, B, F, _, A = shape
    code = _cabi.OBS_DTYPES[obs_dtype]
    offs, total = (C.c_int64 * 6)(), C.c_int64()
    assert _cabi.lib().impala_batch_layout_obs(T, B, F, A, code, offs, C.byref(total)) == 0
    assert _layout_frames(T, B, F, 1, A, code) == (0, list(offs), total.value)


# the slab sizes that motivate frame slabs: (T, B, O, frames, A, obs_dtype, dense bytes, frame bytes)
TABLE = [(20, 4096, 512, 4, 18, "uint8", 50_692_096, 19_234_816),
         (20, 4096, 512, 4, 18, "float32", 182_812_672, 56_983_552),
         (20, 4096, 1024, 8, 18, "uint8", 94_732_288, 21_331_968)]


@pytest.mark.parametrize("T,B,O,k,A,obs_dtype,dense,frames", TABLE)
def test_slab_bytes_of_the_named_configs(T, B, O, k, A, obs_dtype, dense, frames):
    assert _cabi.batch_layout(T, B, O, A, obs_dtype)[1] == dense
    assert _cabi.batch_layout(T, B, O, A, obs_dtype, k)[1] == frames


@pytest.mark.parametrize("args", [(0, 4, 4, 2, 2, 0), (4, 0, 4, 2, 2, 0), (4, 4, 0, 2, 2, 0), (4, 4, 4, 0, 2, 0),
                                  (4, 4, 4, -1, 2, 0), (4, 4, 4, 2, 0, 0), (4, 4, 4, 2, 2, 2), (4, 4, 4, 2, 2, -1)])
def test_bad_layout_and_shard_args_are_refused(args):
    T, B, F, k, A, code = args
    assert _layout_frames(T, B, F, k, A, code)[0] == -1  # IMPALA_ERR_BAD_ARG
    buf = (C.c_uint8 * 4096)()
    assert _cabi.lib().impala_ingest_shard_frames(buf, buf, T, B, F, k, A, code, 0, 1, None) == -1


@pytest.mark.parametrize("b0,B_local", [(-1, 2), (0, 0), (3, 2), (0, 5)])
def test_bad_shard_ranges_are_refused(b0, B_local):
    buf = (C.c_uint8 * 4096)()
    assert _cabi.lib().impala_ingest_shard_frames(buf, buf, 4, 4, 4, 2, 2, 0, b0, B_local, None) == -1
    assert _cabi.lib().impala_ingest_shard_frames(None, buf, 4, 4, 4, 2, 2, 0, 0, 2, None) == -1


U8, F32 = _cabi.OBS_U8, _cabi.OBS_F32


@pytest.mark.parametrize("pair", [(F32, U8), (2, F32), (U8, 2), (-1, -1)])
def test_unstack_refuses_other_dtype_pairs(pair):
    buf = (C.c_uint8 * 64)()  # never read: the argument checks come before any launch
    assert _cabi.lib().impala_obs_unstack(buf, pair[0], buf, pair[1], 2, 2, 2, 2, None) == -1


@pytest.mark.parametrize("R,B,F,k", [(0, 2, 2, 2), (2, 0, 2, 2), (2, 2, 0, 2), (2, 2, 2, 0), (-1, 2, 2, 2)])
def test_unstack_refuses_bad_sizes(R, B, F, k):
    buf = (C.c_uint8 * 64)()
    for pair in ((U8, U8), (U8, F32), (F32, F32)):
        assert _cabi.lib().impala_obs_unstack(buf, pair[0], buf, pair[1], R, B, F, k, None) == -1


def test_unstack_refuses_null():
    buf = (C.c_uint8 * 64)()
    assert _cabi.lib().impala_obs_unstack(None, U8, buf, U8, 2, 2, 2, 2, None) == -1
    assert _cabi.lib().impala_obs_unstack(buf, U8, None, U8, 2, 2, 2, 2, None) == -1


def _views(T, B, O, A, obs_dtype, k):
    offs, total = _layout(T, B, O, A, obs_dtype, k)
    buf = np.zeros(total, np.uint8)
    dts = [np.dtype(t) for t in (obs_dtype, np.float32, np.int32, np.float32, np.uint8, np.int32)]
    shapes = ((T + k, B, O // k), (T, B, A), (T, B), (T, B), (T, B), (B,))
    names = ("obs", "beh_logits", "actions", "rewards", "done", "lens")
    return {n: buf[o:o + int(np.prod(s)) * dt.itemsize].view(dt).reshape(s)
            for n, o, s, dt in zip(names, offs, shapes, dts)}


@pytest.mark.parametrize("k,F,kind", [(4, 32, "bytes"), (2, 3, "normal"), (8, 1, "planes"), (3, 6, "normal")])
def test_packed_frames_unstack_to_the_trajectory(k, F, kind):
    T, B, A = 9, 7, 3
    fb = synth.make_batch(5, T, B, k * F, A, ragged=True, obs_kind=kind, frames=k)
    dense = synth.stack_frames(fb, k)
    trs = synth.to_trajectories(dense)
    obs_dtype = "float32" if kind == "normal" else "uint8"
    v = _views(T, B, k * F, A, obs_dtype, k)
    v["obs"][:] = 1  # the packer must overwrite every frame of the column, the padding included
    for b, tr in enumerate(trs):
        pack_trajectory(v, b, tr, T)
    assert v["obs"].tobytes() == fb["obs"].astype(obs_dtype).tobytes()
    got = synth.stack_frames({"obs": v["obs"]}, k)["obs"]  # numpy unstacking of the packed slab
    for b, L in enumerate(fb["lens"].tolist()):
        want = np.stack([t.numpy() for t in trs[b].obs]).astype(obs_dtype)
        assert got[:L + 1, b].tobytes() == want.tobytes()
        assert not v["obs"][L + k:, b].any()
    for name in ("beh_logits", "actions", "rewards", "done", "lens"):
        assert np.array_equal(v[name], fb[name])


def test_synth_frame_batches():
    T, B, O, A, k = 6, 9, 24, 3, 4
    d = synth.make_batch(4, T, B, O, A, ragged=True)
    fb = synth.make_batch(4, T, B, O, A, ragged=True, frames=k)
    assert fb["obs"].shape == (T + k, B, O // k) and fb["obs"].dtype == np.float32
    for name in ("beh_logits", "actions", "rewards", "done", "lens"):
        assert np.array_equal(fb[name], d[name])
    assert fb["obs"][np.arange(T + k)[:, None] < fb["lens"][None, :] + k].all()  # N(0, 1): no zero draws
    assert not fb["obs"][np.arange(T + k)[:, None] >= fb["lens"][None, :] + k].any()
    s = synth.stack_frames(fb, k)["obs"]
    assert s.shape == (T + 1, B, O)
    assert np.array_equal(s[3, 2], np.concatenate([fb["obs"][3 + j, 2] for j in range(k)]))
    assert synth.make_batch(4, T, B, O, A, frames=k, obs_kind="bytes")["obs"].dtype == np.uint8


def test_broken_overlap_raises_and_publishes_an_empty_column():
    T, B, F, k, A = 6, 4, 5, 3, 2
    fb = synth.make_batch(8, T, B, k * F, A, ragged=True, obs_kind="bytes", frames=k)
    trs = synth.to_trajectories(synth.stack_frames(fb, k))
    step = min(2, len(trs[1].obs) - 1)
    trs[1].obs[step] = trs[1].obs[step].clone()
    trs[1].obs[step][0] += 1  # its oldest frame no longer equals the second frame of the step before
    q = RingQueue(T, B, k * F, A, slabs=2, obs_dtype="uint8", frames=k)
    try:
        q.put(trs[0], timeout=1)
        with pytest.raises(ValueError, match=f"trajectory .*observation {step} "):
            q.put(trs[1], timeout=1)
        for tr in trs[2:]:
            q.put(tr, timeout=1)
        kk, _ = q.collect_batch(timeout=1)  # every column filled: the learner does not stall
        v = q.views(kk)
        assert v["lens"][1] == 0 and not v["obs"][:, 1].any() and not v["rewards"][:, 1].any()
        for b in (0, 2, 3):
            L = int(fb["lens"][b])
            assert np.array_equal(v["obs"][:, b], fb["obs"][:, b]) and v["lens"][b] == L
    finally:
        q.close()


def test_ring_put_block_takes_frame_blocks():
    T, B, O, A, k = 5, 8, 12, 3, 4
    fb = synth.make_batch(2, T, 4, O, A, ragged=True, frames=k)
    q = RingQueue(T, B, O, A, slabs=2, frames=k)
    try:
        assert q.views(0)["obs"].shape == (T + k, B, O // k)
        with pytest.raises(ValueError, match="ring takes"):
            q.put_block(synth.stack_frames(fb, k), timeout=1)
        q.put_block(fb, timeout=1)
        q.put_block(fb, timeout=1)
        kk, _ = q.collect_batch(timeout=1)
        assert np.array_equal(q.views(kk)["obs"][:, 4:], fb["obs"])
    finally:
        q.close()


def test_learner_checks_frames():
    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpPolicy, MlpValueFn
    from torched_impala_b200.utils import Counter as SharedCounter, default_hparams

    T, B, O, A = 5, 4, 8, 2
    hp = default_hparams(batch_size=B, max_timesteps=T, log_path=None)
    q = RingQueue(T, B, O, A, slabs=2, frames=4)
    try:
        with pytest.raises(ValueError, match="frames"):
            Learner(1, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), q, SharedCounter(0))
        with pytest.raises(ValueError, match="frames"):
            Learner(2, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), q, SharedCounter(0), frames=2)
        lrn = Learner(3, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), q, SharedCounter(0), frames=4)
        assert lrn._cfg()["frames"] == 4
    finally:
        q.close()
    with pytest.raises(ValueError, match="frames"):
        Learner(4, hp, MlpPolicy(O, A, 8), MlpValueFn(O, 8), None, SharedCounter(0), frames=3)
    with pytest.raises(ValueError):
        RingQueue(T, B, O, A, slabs=2, frames=3)


def test_unstack_kernel_has_no_spills_or_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.fail("nvcc not found")
    src = os.path.join(os.path.dirname(_cabi.__file__), "csrc", "obs_frames.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", src, "-o", str(tmp_path / "obs_frames.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    blocks = re.split(r"Compiling entry function", res.stderr)[1:]
    unstack = [b for b in blocks if "obs_unstack_kernel" in b.splitlines()[0]]
    assert len(unstack) == 6, len(unstack)  # 3 dtype pairs x (16-byte vectors, elements)
    for b in unstack:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b, b
        assert not re.search(r"\d+ bytes lmem", b) or re.search(r"\b0 bytes lmem", b), b
