"""GPU: reward clipping inside the V-trace kernel (impala_vtrace_loss_rclip).

abs_one clipping is exact in float32, so the clip kernels fed raw rewards must reproduce, bit for bit, the
plain / diag / PopArt kernels fed host-clipped rewards, except batch_mean_reward, which stays the raw mean.
soft_asymmetric is checked against the float64 oracle (tests/reward_clip_oracle.py).  Then the engine (CUDA
graph, replay, uint8 frames), a forked Learner behind a RingQueue and (>= 2 devices) data-parallel training."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import reward_clip_oracle as rorc
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.engine import LearnerEngine
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu

OUT_KEYS = ("vs", "pg_adv", "dlogits", "dv")


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _case(T, B, A, seed, lo=-10.0, hi=10.0):
    """A ragged batch with empty columns (lens 0) and rewards spread over [lo, hi] at every step."""
    b = synth.make_batch(seed, T, B, 3, A, ragged=True)
    rng = np.random.default_rng(seed + 1)
    lens = b["lens"].copy()
    lens[::9] = 0
    rewards = rng.uniform(lo, hi, (T, B)).astype(np.float32)
    logits = (b["beh_logits"] + 0.5 * rng.standard_normal((T, B, A))).astype(np.float32)
    v = rng.standard_normal((T + 1, B), dtype=np.float32)
    return dict(logits=logits, beh=b["beh_logits"], actions=b["actions"], rewards=rewards, done=b["done"],
                lens=lens, v=v)


def _soft_rewards(rng, T, B):
    """Raw rewards whose soft_asymmetric images are about N(0, 1) (the scale of the other parity tests' rewards, so
    vs and pg_adv stay within the magnitudes the 1e-5 absolute contract is stated for), drawn through both branches
    of the transform up to its saturation (y near -1.5), plus 3 % of large rewards, |r| in [10, 40]."""
    y = np.clip(rng.standard_normal((T, B)), -1.49, 4.99)
    with np.errstate(invalid="ignore"):  # np.where evaluates both branches
        r = np.where(y < 0, 5.0 * np.arctanh(y / 1.5), 5.0 * np.arctanh(y / 5.0))
    u, mag = rng.random((T, B)), rng.uniform(10.0, 40.0, (T, B))
    r = np.where(u < 0.01, mag, np.where(u < 0.03, -mag, r))
    return r.astype(np.float32)


def _against_oracle(got, c, rewards, hp, B, reward_clip, mode="reference"):
    """Per element 1e-5 absolute (DESIGN.md §2) on vs (valid rows), pg_adv, dlogits and dv; the four scalars
    within the contract's 1e-5, relative beyond magnitude 1 at these small batches (as tests/test_gpu_parity.py)."""
    T = rewards.shape[0]
    want = rorc.vtrace_loss(c["v"], c["logits"], c["beh"], c["actions"], rewards, c["done"], c["lens"], hp, B,
                            reward_clip, mode)
    valid_v = np.arange(T + 1)[:, None] <= c["lens"][None, :]
    err = np.abs(np.where(valid_v, got["vs"].cpu().numpy(), 0.0) - want["vs"]).max()
    assert err < 1e-5, ("vs", err, np.abs(want["vs"]).max())
    for k in ("pg_adv", "dlogits", "dv"):
        err = np.abs(got[k].cpu().numpy() - want[k]).max()
        assert err < 1e-5, (k, err, np.abs(want[k]).max())
    s = got["scalars"].cpu().tolist()
    for i, k in enumerate(("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward")):
        if np.isfinite(want[k]):
            assert abs(s[i] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, s[i], want[k])
        else:  # the raw mean of rewards with +-inf in them
            assert s[i] == want[k] or (np.isnan(s[i]) and np.isnan(want[k])), (k, s[i], want[k])


def _args(c, rewards):
    return (dev(c["logits"]), dev(c["beh"]), dev(c["actions"]), dev(rewards), dev(c["done"]), dev(c["lens"]),
            dev(c["v"]))


VARIANTS = ("plain", "diag", "popart")


def _twin(ops, variant, args, hp, inv_batch, mode, popart):
    if variant == "plain":
        return ops.vtrace_loss(*args, hp, inv_batch, mode=mode)
    if variant == "diag":
        return ops.vtrace_loss_diag(*args, hp, inv_batch, mode=mode)
    return ops.vtrace_loss_popart(*args, hp, inv_batch, popart, mode=mode)


def _clip(ops, variant, args, hp, inv_batch, mode, popart, reward_clip="abs_one"):
    return ops.vtrace_loss_rclip(*args, hp, inv_batch, reward_clip, mode=mode, diagnostics=variant == "diag",
                                 popart=popart if variant == "popart" else None)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("T", [20, 100])
@pytest.mark.parametrize("A", [2, 4, 6, 18, 32])  # register (AP 2, 4), spilling (AP 8, S 2), streaming paths
def test_abs_one_equals_host_clipped(ops, A, T, mode, variant):
    B = 77
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9, gamma=0.97)
    c = _case(T, B, A, 100 * A + T)
    popart = ops.popart_stats(0.7, 6.0)
    clipped = np.clip(c["rewards"], -1.0, 1.0)
    got = _clip(ops, variant, _args(c, c["rewards"]), hp, 1.0 / B, mode, popart)
    want = _twin(ops, variant, _args(c, clipped), hp, 1.0 / B, mode, popart)
    raw = _twin(ops, variant, _args(c, c["rewards"]), hp, 1.0 / B, mode, popart)
    for k in OUT_KEYS:
        assert torch.equal(got[k], want[k]), k
    assert torch.equal(got["scalars"][:3], want["scalars"][:3])
    if variant != "plain":
        assert torch.equal(got["diag"], want["diag"])
    g3, r3 = float(got["scalars"][3]), float(raw["scalars"][3])
    assert abs(g3 - r3) <= 1e-12 * abs(r3), (g3, r3)
    assert g3 != float(want["scalars"][3])  # the raw mean, not the clipped one


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("A", [4, 18])
def test_identity_region(ops, A, variant):
    """Rewards inside [-1, 1]: abs_one changes nothing, so every output equals the kernel without clipping."""
    T, B = 20, 64
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9)
    c = _case(T, B, A, 7 + A, -1.0, 1.0)
    c["rewards"][0, :4] = [-1.0, 1.0, 0.0, -0.0]
    popart = ops.popart_stats(-0.3, 2.0)
    got = _clip(ops, variant, _args(c, c["rewards"]), hp, 1.0 / B, "reference", popart)
    want = _twin(ops, variant, _args(c, c["rewards"]), hp, 1.0 / B, "reference", popart)
    for k in OUT_KEYS:
        assert torch.equal(got[k], want[k]), k
    valid = np.arange(T)[:, None] < c["lens"][None, :]
    s_got, s_want = got["scalars"].cpu().numpy(), want["scalars"].cpu().numpy()
    assert np.array_equal(s_got[:3], s_want[:3])
    assert abs(s_got[3] - s_want[3]) <= 1e-12 * max(1e-300, abs(s_want[3])) and valid.any()


@pytest.mark.parametrize("mode", ["reference", "paper"])
@pytest.mark.parametrize("T", [20, 100])
@pytest.mark.parametrize("A", [2, 4, 6, 18, 32])
def test_soft_asymmetric_against_oracle(ops, A, T, mode):
    B = 77
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9, gamma=0.97)
    c = _case(T, B, A, 300 + A + T)
    r = _soft_rewards(np.random.default_rng(301 + A + T), T, B)
    got = ops.vtrace_loss_rclip(*_args(c, r), hp, 1.0 / B, "soft_asymmetric", mode=mode)
    _against_oracle(got, c, r, hp, B, "soft_asymmetric", mode)


@pytest.mark.parametrize("reward_clip", rorc.MODES)
@pytest.mark.parametrize("A", [4, 6, 32])
def test_nan_and_infinity(ops, A, reward_clip):
    T, B = 20, 64
    hp = default_hparams(batch_size=B, rho_bar=1.0, c_bar=0.9)
    c = _case(T, B, A, 50 + A)
    c["lens"][:] = T
    r = _soft_rewards(np.random.default_rng(51 + A), T, B)
    r[3, 5], r[7, 6] = np.inf, -np.inf
    fin = ops.vtrace_loss_rclip(*_args(c, r), hp, 1.0 / B, reward_clip)
    for k in OUT_KEYS:
        assert torch.isfinite(fin[k]).all(), k
    # the kernel's saturation values (+-1; 5 and -1.5) against the oracle's, through vs and pg_adv
    _against_oracle(fin, c, r, hp, B, reward_clip)
    r[9, 10] = np.nan
    bad = ops.vtrace_loss_rclip(*_args(c, r), hp, 1.0 / B, reward_clip)
    vs = bad["vs"].cpu().numpy()
    assert np.isnan(vs[9, 10]) and np.isfinite(np.delete(vs, 10, axis=1)).all()
    assert torch.isnan(bad["scalars"][:2]).all()  # the value and policy losses


def test_refused_arguments(ops):
    T, B, A = 5, 8, 4
    hp = default_hparams(batch_size=B)
    c = _case(T, B, A, 1)
    a = _args(c, c["rewards"])
    lib = _cabi.lib()
    ws = torch.zeros(int(lib.impala_vtrace_loss_diag_workspace(T, B, A)), dtype=torch.uint8, device="cuda")
    outs = [torch.empty(n, dtype=torch.float32, device="cuda") for n in ((T + 1) * B, T * B, T * B * A, (T + 1) * B)]
    sc = torch.empty(12, dtype=torch.float64, device="cuda")  # 4 scalars, then the 8 diag sums
    st = ops.popart_stats()

    def call(diag, popart, code):
        p = lambda t: t.data_ptr()  # noqa: E731
        return lib.impala_vtrace_loss_rclip(*[p(t) for t in a], *[p(t) for t in outs], p(sc), p(ws), ws.numel(), T, B,
                                            A, 0.99, 1.0, 1.0, 0.5, 1.0, 0.01, 1.0 / B, 0, diag, popart, code, None)

    for code in (0, 3, -1):
        assert call(None, None, code) == -1
    assert call(None, st.data_ptr(), 1) == -1  # popart without diag
    assert call(None, None, 1) == 0 and call(sc.data_ptr() + 32, st.data_ptr(), 2) == 0
    torch.cuda.synchronize()


ENGINE = {"c4": (20, 1024, 24, 4, 256), "ram4": (20, 256, 512, 18, 256)}
ENGINE_CASES = {  # shape, engine arguments
    "c4": ("c4", {}),
    "c4-diag-popart": ("c4", dict(diagnostics=True, popart=True, popart_beta=0.1)),
    "c4-paper": ("c4", dict(mode="paper")),
    "ram4-replay-u8-frames4": ("ram4", dict(replay_slabs=2, replay_columns=64, obs_dtype="uint8", frames=4)),
}


@pytest.mark.parametrize("case", list(ENGINE_CASES))
def test_engine_equals_plain_engine_on_clipped_slabs(case):
    shape, kw = ENGINE_CASES[case]
    T, B, O, A, H = ENGINE[shape]
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9, max_updates=8)
    clip, plain = LearnerEngine(T, B, O, A, H, H, hp, reward_clip="abs_one", **kw), LearnerEngine(T, B, O, A, H, H,
                                                                                                  hp, **kw)
    assert clip.use_graph and plain.use_graph
    params = synth.init_params(3, O, A, H)
    for e in (clip, plain):
        e.load_state(params)
    Bf = B - kw.get("replay_columns", 0)
    kind = "bytes" if kw.get("obs_dtype") == "uint8" else "normal"
    for u in range(5):
        bt = synth.make_batch(60 + u, T, Bf, O, A, ragged=(u % 2 == 1), obs_kind=kind, frames=kw.get("frames", 1))
        bt["rewards"] = bt["rewards"] * np.float32(4.0)
        bc = dict(bt, rewards=np.clip(bt["rewards"], -1.0, 1.0))
        for e, b_ in ((clip, bt), (plain, bc)):
            e.fill_host(b_, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
        sc, sp = clip.read_scalars(), plain.read_scalars()
        for k in ("value_fn_loss", "policy_loss", "policy_entropy"):
            assert sc[k] == sp[k], (u, k)
        if not kw.get("replay_columns"):
            valid = np.arange(T)[:, None] < bt["lens"][None, :]
            raw = bt["rewards"].astype(np.float64)[valid].sum() / B
            assert abs(sc["batch_mean_reward"] - raw) <= 1e-12 * abs(raw), (u, sc["batch_mean_reward"], raw)
    for e in (clip, plain):
        e.synchronize()
    assert clip.launches_per_step == plain.launches_per_step
    for name in ("params", "adam_m", "adam_v", "adam_step", "popart_buf"):
        assert torch.equal(getattr(clip, name), getattr(plain, name)), name


def test_engine_without_clip_launches_the_untransformed_kernel():
    T, B, O, A, H = 20, 64, 8, 4, 64
    hp = default_hparams(batch_size=B, max_timesteps=T)
    a, b = LearnerEngine(T, B, O, A, H, H, hp), LearnerEngine(T, B, O, A, H, H, hp, reward_clip=None)
    params = synth.init_params(3, O, A, H)
    for e in (a, b):
        e.load_state(params)
    for u in range(3):
        bt = synth.make_batch(5 + u, T, B, O, A, ragged=True)
        bt["rewards"] = bt["rewards"] * np.float32(4.0)
        for e in (a, b):
            e.fill_host(bt, u % 2)
            e.ingest(u % 2)
            e.step(u % 2)
        assert a.read_scalars() == b.read_scalars()
    assert torch.equal(a.params, b.params) and b.reward_clip_code == 0


def test_forked_learner(tmp_path):
    script = os.path.join(os.path.dirname(__file__), "reward_clip_learner_process_check.py")
    outs = {}
    for mode in ("clip", "plain"):
        out = tmp_path / f"weights_{mode}.npz"
        res = subprocess.run([sys.executable, script, str(tmp_path / f"logs_{mode}"), mode, str(out)],
                             capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
        assert "REWARD_CLIP_LEARNER_OK" in res.stdout
        outs[mode] = np.load(out)
    on, off = outs["clip"], outs["plain"]
    weights = [k for k in on.files if "/" in k]
    assert weights and set(on.files) == set(off.files)
    for k in weights:
        assert np.array_equal(on[k], off[k]), k
    # the logged batch_mean_reward is the raw one under clipping, the clipped one for the plain run on clipped data
    assert np.allclose(on["logged_reward"], on["raw_reward"], rtol=1e-6, atol=1e-6)
    assert np.allclose(off["logged_reward"], off["clipped_reward"], rtol=1e-6, atol=1e-6)
    assert not np.allclose(on["raw_reward"], on["clipped_reward"])


@pytest.mark.parametrize("allreduce", ["peer", "nccl"])
def test_two_gpus(allreduce):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs (data-parallel path)")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    script = os.path.join(os.path.dirname(__file__), "multi_gpu_reward_clip_check.py")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script],
                         capture_output=True, text=True, timeout=240, env=dict(os.environ, IMPALA_ALLREDUCE=allreduce))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "MULTI_GPU_REWARD_CLIP_OK" in res.stdout
