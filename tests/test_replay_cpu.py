"""CPU: experience replay without a device - argument checks, the sampling plan, the numpy composition the GPU
tests compare against, the C entry point's argument checks and the compose kernel's ptxas report."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle.replay import compose_batch
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.replay import ReplaySampler, check_replay_args
from torched_impala_b200.ring import RingQueue


def test_replay_args():
    assert check_replay_args(8, 0, 0) == 8
    assert check_replay_args(8, 3, 5) == 3
    assert check_replay_args(8, 1, 7) == 1
    for R, Br in ((0, 4), (2, 0), (-1, 4), (2, -1), (2, 8), (2, 9)):
        with pytest.raises(ValueError, match="replay"):
            check_replay_args(8, R, Br)
    for args in ((0, 4, 4), (2, 0, 4), (2, 4, 0)):
        with pytest.raises(ValueError):
            ReplaySampler(0, *args)


def test_learner_checks_replay():
    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpPolicy, MlpValueFn
    from torched_impala_b200.utils import Counter as SharedCounter, default_hparams

    T, B, O, A = 5, 8, 6, 2
    hp = default_hparams(batch_size=B, max_timesteps=T, log_path=None)
    nets = lambda: (MlpPolicy(O, A, 8), MlpValueFn(O, 8))  # noqa: E731
    for kw in (dict(replay_slabs=2), dict(replay_columns=2), dict(replay_slabs=2, replay_columns=B)):
        with pytest.raises(ValueError, match="replay"):
            Learner(1, hp, *nets(), None, SharedCounter(0), **kw)
    with pytest.raises(ValueError, match="one device"):
        Learner(2, hp, *nets(), None, SharedCounter(0), replay_slabs=2, replay_columns=4, devices=["cuda:0", "cuda:1"])
    wide, fresh = RingQueue(T, B, O, A, slabs=2), RingQueue(T, B - 3, O, A, slabs=2)
    try:
        with pytest.raises(ValueError, match=r"5 trajectories.*built for 8"):
            Learner(3, hp, *nets(), wide, SharedCounter(0), replay_slabs=2, replay_columns=3)
        lrn = Learner(4, hp, *nets(), fresh, SharedCounter(0), replay_slabs=2, replay_columns=3)
        cfg = lrn._cfg()
        assert (cfg["replay_slabs"], cfg["replay_columns"], cfg["B"], lrn.B_fresh) == (2, 3, B, 5)
        off = Learner(5, hp, *nets(), wide, SharedCounter(0))
        assert (off._cfg()["replay_slabs"], off._cfg()["replay_columns"], off.B_fresh) == (0, 0, B)
    finally:
        wide.close()
        fresh.close()


@pytest.mark.parametrize("R,Bf,Br", [(1, 3, 2), (2, 4, 4), (5, 2, 7)])
def test_plans_stay_inside_the_pool(R, Bf, Br):
    s = ReplaySampler(3, R, Bf, Br)
    slots = R + 2
    first = s.plan(1)
    assert first.dtype == np.int32 and first.shape == (Bf + Br, 2)
    assert (first[Bf:, 0] == -1).all() and (first[Bf:, 1] == 0).all()
    for n in range(1, 40):
        plan = s.plan(n)
        assert np.array_equal(plan[:Bf], np.stack([np.full(Bf, n % slots), np.arange(Bf)], 1))  # identity: fresh
        if n == 1:
            continue
        u, c = s.sources(n)
        assert u.shape == c.shape == (Br,)
        assert u.min() >= max(1, n - R) and u.max() <= n - 1
        assert c.min() >= 0 and c.max() < Bf
        assert np.array_equal(plan[Bf:, 0], u % slots) and np.array_equal(plan[Bf:, 1], c)
        # never the slot of update n (its own fresh batch) nor the one being filled for update n + 1
        assert not np.isin(plan[Bf:, 0], [n % slots, (n + 1) % slots]).any()
        # a slot names one update of the pool: no two pool updates share a slot
        assert len({int(x) % slots for x in range(max(1, n - R), n)}) == min(R, n - 1)


def test_same_seed_same_plans_and_any_order():
    a, b, other = ReplaySampler(7, 3, 5, 6), ReplaySampler(7, 3, 5, 6), ReplaySampler(8, 3, 5, 6)
    plans = [a.plan(n) for n in range(1, 12)]
    for n in reversed(range(1, 12)):  # a pure function of (seed, n)
        assert np.array_equal(b.plan(n), plans[n - 1])
    assert any(not np.array_equal(other.plan(n), plans[n - 1]) for n in range(2, 12))
    assert not np.array_equal(plans[5][5:, 1], plans[6][5:, 1])  # consecutive updates draw differently
    with pytest.raises(ValueError):
        a.plan(0)


def test_every_source_of_a_small_pool_is_drawn():
    R, Bf, Br = 3, 4, 5
    s = ReplaySampler(0, R, Bf, Br)
    seen = np.zeros((R, Bf), np.int64)  # (age - 1, column)
    for n in range(R + 1, R + 401):
        u, c = s.sources(n)
        np.add.at(seen, (n - 1 - u, c), 1)
    assert seen.sum() == 400 * Br
    assert seen.min() > 0.6 * seen.mean() and seen.max() < 1.4 * seen.mean(), seen  # uniform: about 167 each


def _tiny(seed, T, Bf, O, A, **kw):
    return synth.make_batch(seed, T, Bf, O, A, ragged=True, **kw)


def test_compose_batch_on_a_hand_made_history():
    T, Bf, O, A = 4, 3, 2, 2
    hist = {0: _tiny(1, T, Bf, O, A), 2: _tiny(2, T, Bf, O, A)}
    plan = np.array([[2, 0], [2, 1], [2, 2], [0, 1], [-1, 0], [0, 1], [2, 0]], np.int32)
    out = compose_batch(hist, plan)
    assert out["obs"].shape == (T + 1, 7, O) and out["lens"].shape == (7,) and out["done"].dtype == np.uint8
    for name in ("obs", "beh_logits", "actions", "rewards", "done"):
        assert np.array_equal(out[name][:, :3], hist[2][name])                 # the identity part
        assert np.array_equal(out[name][:, 3], hist[0][name][:, 1])
        assert np.array_equal(out[name][:, 5], hist[0][name][:, 1])            # a repeated source
        assert np.array_equal(out[name][:, 6], hist[2][name][:, 0])
        assert not out[name][:, 4].any()                                       # the empty column
        assert out[name].dtype == hist[0][name].dtype
    assert out["lens"].tolist() == [*hist[2]["lens"], hist[0]["lens"][1], 0, hist[0]["lens"][1], hist[2]["lens"][0]]


def test_compose_batch_frames_and_bytes():
    T, Bf, O, A, k = 5, 2, 8, 3, 4
    hist = {1: _tiny(3, T, Bf, O, A, obs_kind="bytes", frames=k)}
    out = compose_batch(hist, [[1, 1], [1, 0], [-1, 0]])
    assert out["obs"].shape == (T + k, 3, O // k) and out["obs"].dtype == np.uint8
    assert np.array_equal(out["obs"][:, 0], hist[1]["obs"][:, 1]) and not out["obs"][:, 2].any()


def _compose_rc(dst, store, nbytes, plan, T, B, Bf, F, k, A, code):
    return _cabi.lib().impala_batch_compose(dst, store, nbytes, plan, T, B, Bf, F, k, A, code, None)


def test_compose_refuses_bad_arguments():
    buf = (C.c_uint8 * 64)()  # never read: the argument checks come before any launch
    big = 1 << 20
    good = (4, 6, 3, 5, 2, 2, _cabi.OBS_U8)
    for i in range(4):
        ptrs = [buf, buf, big, buf]
        ptrs[i] = None if i != 2 else 16  # a NULL pointer; a store slab smaller than the fresh layout
        assert _compose_rc(*ptrs, *good) == -1, i
    for T, B, Bf, F, k, A, code in ((4, 6, 0, 5, 2, 2, 1), (4, 6, -1, 5, 2, 2, 1), (4, 6, 6, 5, 2, 2, 1),
                                    (4, 6, 7, 5, 2, 2, 1), (4, 6, 3, 5, 2, 2, 2), (4, 6, 3, 5, 2, 2, -1),
                                    (0, 6, 3, 5, 2, 2, 0), (4, 6, 3, 0, 2, 2, 0), (4, 6, 3, 5, 0, 2, 0),
                                    (4, 6, 3, 5, 2, 0, 0)):
        assert _compose_rc(buf, buf, big, buf, T, B, Bf, F, k, A, code) == -1, (T, B, Bf, F, k, A, code)


def test_compose_kernel_has_no_spills_or_local_memory(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.fail("nvcc not found")
    src = os.path.join(os.path.dirname(_cabi.__file__), "csrc", "batch_compose.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", src, "-o", str(tmp_path / "batch_compose.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    blocks = [b for b in re.split(r"Compiling entry function", res.stderr)[1:] if "batch_compose_kernel" in b]
    assert len(blocks) == 1, len(blocks)  # one kernel serves the three vector widths and the six tensors
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blocks[0], blocks[0]
    assert not re.search(r"\d+ bytes lmem", blocks[0]) or re.search(r"\b0 bytes lmem", blocks[0]), blocks[0]
