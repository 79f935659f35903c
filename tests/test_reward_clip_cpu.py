"""CPU: reward clipping - the float64 transforms, the oracle on clipped rewards, argument checks before any
CUDA work, the C ABI declaration and export, and the local-memory traffic of the clip kernels' SASS."""
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

import reward_clip_oracle as rorc
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.utils import default_hparams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = [-np.inf, -7.0, -1.0, -0.5, 0.0, 0.5, 1.0, 7.0, np.inf, np.nan]


def test_abs_one_transform():
    got = rorc.clip_rewards(R, "abs_one")
    want = torch.clamp(torch.tensor(R, dtype=torch.float64), -1.0, 1.0).numpy()
    assert np.array_equal(got, want, equal_nan=True)
    assert np.array_equal(got, [-1, -1, -1, -0.5, 0, 0.5, 1, 1, 1, np.nan], equal_nan=True)


def test_soft_asymmetric_transform():
    got = rorc.clip_rewards(R, "soft_asymmetric")
    assert np.isnan(got[-1])
    assert got[0] == -1.5 and got[8] == 5.0  # +-inf saturates
    for r, g in zip(R[1:8], got[1:8]):
        want = (5.0 if r >= 0 else 1.5) * np.tanh(r / 5.0)
        assert abs(g - want) <= 1e-15 * max(1.0, abs(want)), (r, g, want)
    assert got[4] == 0.0 and np.all(np.diff(got[:9]) >= 0)


def test_unknown_mode_refused_by_oracle():
    with pytest.raises(ValueError):
        rorc.clip_rewards([0.0], "sign")


@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("reward_clip", rorc.MODES)
def test_oracle_equals_plain_oracle_on_preclipped_rewards(reward_clip, mode):
    T, B, A = 15, 11, 5
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    b = synth.make_batch(4, T, B, 3, A, ragged=True)
    rng = np.random.default_rng(9)
    rewards = (10.0 * rng.uniform(-1, 1, (T, B))).astype(np.float32)
    logits = (b["beh_logits"] + 0.3 * rng.standard_normal((T, B, A))).astype(np.float32)
    v = rng.standard_normal((T + 1, B))
    got = rorc.vtrace_loss(v, logits, b["beh_logits"], b["actions"], rewards, b["done"], b["lens"], hp, B,
                           reward_clip, mode)
    rc = rorc.clip_rewards(rewards, reward_clip)
    vs, pg, _ = orc.vtrace(v, logits, b["beh_logits"], b["actions"], rc, b["done"], b["lens"], hp.gamma,
                           hp.rho_bar, hp.c_bar, mode)
    want = orc.losses(v, vs, logits, b["actions"], pg, b["lens"], hp.v_loss_c, hp.policy_loss_c, hp.entropy_c, B)
    assert np.array_equal(got["vs"], vs) and np.array_equal(got["pg_adv"], pg)
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "dv", "dlogits"):
        assert np.array_equal(got[k], want[k]), k
    valid = np.arange(T)[:, None] < b["lens"][None, :]
    raw = float(rewards.astype(np.float64)[valid].sum() / B)
    assert got["batch_mean_reward"] == raw
    assert raw != float(rc[valid].sum() / B)  # the rewards reach past the clip range


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


@pytest.mark.parametrize("bad", ["clip", "ABS_ONE", "", 1, True])
def test_engine_refuses_bad_reward_clip_before_cuda(monkeypatch, bad):
    from torched_impala_b200.engine import LearnerEngine

    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    with pytest.raises(ValueError, match="abs_one"):
        LearnerEngine(5, 8, 4, 2, 8, 8, hp, reward_clip=bad)
    with pytest.raises(AssertionError):  # a good value goes on to the device checks
        LearnerEngine(5, 8, 4, 2, 8, 8, hp, reward_clip="soft_asymmetric")


class _Net(torch.nn.Module):
    def __init__(self, O, H, N2):
        super().__init__()
        self.model = torch.nn.Sequential(torch.nn.Linear(O, H), torch.nn.Dropout(0.0), torch.nn.ReLU(),
                                         torch.nn.Linear(H, N2))


def test_learner_refuses_bad_reward_clip_and_carries_good_one(monkeypatch):
    import multiprocessing as mp

    from torched_impala_b200.learner import Learner

    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    with pytest.raises(ValueError, match="soft_asymmetric"):
        Learner(0, hp, _Net(4, 8, 2), _Net(4, 8, 1), mp.Queue(), None, reward_clip="tanh")
    for rc in (None, "abs_one", "soft_asymmetric"):
        ln = Learner(0, hp, _Net(4, 8, 2), _Net(4, 8, 1), mp.Queue(), None, reward_clip=rc)
        assert ln._cfg()["reward_clip"] == rc


def test_header_and_signature():
    hdr = open(os.path.join(ROOT, "include", "impala_b200.h")).read()
    assert re.search(r"\bint impala_vtrace_loss_rclip\(", hdr)
    assert "#define IMPALA_REWARD_CLIP_ABS_ONE 1" in hdr and "#define IMPALA_REWARD_CLIP_SOFT_ASYMMETRIC 2" in hdr
    assert _cabi.REWARD_CLIPS == {"abs_one": 1, "soft_asymmetric": 2}
    # impala_vtrace_loss's arguments before the stream, then diag, popart, reward_clip and the stream
    plain, rclip = _cabi.SIGNATURES["impala_vtrace_loss"][1], _cabi.SIGNATURES["impala_vtrace_loss_rclip"][1]
    assert rclip[:len(plain) - 1] == plain[:-1] and len(rclip) == len(plain) + 3


def test_library_exports_entry_point():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([nm, "-D", "--defined-only", _cabi.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    assert re.search(r"\bT impala_vtrace_loss_rclip$", out, re.M)


def _targs(name):
    m = re.search(r"vtrace_lane_kernelI((?:L[ib]\d+E)+)E", name)
    return tuple(int(x) for x in re.findall(r"L[ib](\d+)E", m.group(1)))


@pytest.fixture(scope="module")
def vtrace_sass():
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
            cur = _targs(m.group(1)) if "vtrace_lane_kernel" in m.group(1) else None
            if cur is not None:
                kernels[cur] = Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and cur is not None:
            kernels[cur][m.group(1)] += 1
    return kernels


def test_clip_instantiations_cover_every_loss_launch_shape(vtrace_sass):
    # template arguments: AP, S, MAXT, MINB, WITH_LOSS, VEC, DIAG, POPART, RCLIP
    loss = {k[:-1] for k in vtrace_sass if k[4] == 1 and k[-1] == 0}
    clip = {k[:-1] for k in vtrace_sass if k[-1] == 1}
    assert loss and clip == loss
    assert len(clip) == 54  # (AP 2, 4 at S 1, 2, 5; AP 8, 16, 32) x VEC x {plain, diag, popart}


def test_clip_instantiations_spill_only_where_their_twins_do(vtrace_sass):
    local = ("LDL", "STL")
    for k, ops in vtrace_sass.items():
        if k[-1] != 1:
            continue
        twin = vtrace_sass[k[:-1] + (0,)]
        if not any(twin[m] for m in local):
            assert not any(ops[m] for m in local), (k, {m: ops[m] for m in local})
