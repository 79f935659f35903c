"""CPU: diagonal Gaussian policies - the float64 oracle against torch autograd on torch.distributions.Normal, the
slab layouts, argument checks before any CUDA work, the C ABI and the local-memory traffic of the Gaussian
kernels' SASS."""
import ctypes as C
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

import gaussian_oracle as gorc
import reward_clip_oracle as rorc
from torched_impala_b200 import _cabi
from torched_impala_b200.utils import default_hparams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _torch_update(x, hp, batch_size, mode, reward_clip, popart):
    """The reference learner's loss (learner.py:104-162), one trajectory at a time, with a Normal policy and
    autograd for d total / d [m | s] and d total / d v (PopArt: v normalized, targets in reward units)."""
    T, B, A2 = x["cur"].shape
    A = A2 // 2
    mu_p, sig = (0.0, 1.0) if popart is None else popart
    z = torch.tensor(x["cur"], dtype=F64, requires_grad=True)
    n = torch.tensor(x["v"], dtype=F64, requires_grad=True)
    beh = torch.tensor(x["beh"], dtype=F64)
    act = torch.tensor(x["actions"], dtype=F64)
    rw = x["rewards"] if reward_clip is None else rorc.clip_rewards(x["rewards"], reward_clip)
    total = torch.zeros((), dtype=F64)
    sums = dict(value_fn_loss=0.0, policy_loss=0.0, policy_entropy=0.0)
    vs_all, pg_all = np.zeros((T + 1, B)), np.zeros((T, B))
    lp_all, ent_all, kl_all = np.zeros((T, B)), np.zeros((T, B)), np.zeros((T, B))
    for b in range(B):
        L = int(x["lens"][b])
        pi = torch.distributions.Normal(z[:L, b, :A], torch.exp(z[:L, b, A:]))
        mu = torch.distributions.Normal(beh[:L, b, :A], torch.exp(beh[:L, b, A:]))
        lp = pi.log_prob(act[:L, b]).sum(-1)
        lpb = mu.log_prob(act[:L, b]).sum(-1)
        ent = pi.entropy().sum(-1)
        kl = torch.distributions.kl_divergence(mu, pi).sum(-1)
        v = sig * n[:L + 1, b] + mu_p
        r = torch.tensor(rw[:L, b], dtype=F64)
        # learner.py:109: gamma * ~done is a float32 tensor
        disc = (hp.gamma * torch.tensor(1 - x["done"][:L, b].astype(np.int64), dtype=torch.float32)).to(F64)
        with torch.no_grad():
            ratio = torch.exp(lp - lpb)
            rho, c = torch.clamp(ratio, max=hp.rho_bar), torch.clamp(ratio, max=hp.c_bar)
            vt = torch.zeros(L + 1, dtype=F64)
            if mode == "reference":
                delta = rho * (r + hp.gamma * v[1:] - v[:1])
                for i in range(L - 1, -1, -1):
                    vt[i] = delta[i] + disc[i] * c[i] * (vt[i + 1] - v[i + 1])
            else:
                delta = rho * (r + disc * v[1:] - v[:-1])
                for i in range(L - 1, -1, -1):
                    vt[i] = delta[i] + disc[i] * c[i] * vt[i + 1]
            vt = vt + v
            pg = rho * (r + disc * vt[1:] - v[:-1]) / sig
        vl = 0.5 * torch.sum(((v - vt) / sig) ** 2)
        pl = torch.sum(-lp * pg)
        pe = torch.sum(ent)
        total = total + (hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * pe) / batch_size
        for k, t in (("value_fn_loss", vl), ("policy_loss", pl), ("policy_entropy", pe)):
            sums[k] += t.item() / batch_size
        vs_all[:L + 1, b], pg_all[:L, b] = vt.numpy(), pg.numpy()
        lp_all[:L, b], ent_all[:L, b], kl_all[:L, b] = lp.detach().numpy(), ent.detach().numpy(), kl.detach().numpy()
    total.backward()
    return dict(sums, vs=vs_all, pg_adv=pg_all, dparams=z.grad.numpy(), dv=n.grad.numpy(), log_pi=lp_all,
                entropy=ent_all, kl=kl_all, total_loss=total.item())


@pytest.mark.parametrize("popart", [None, (0.4, 2.5)])
@pytest.mark.parametrize("reward_clip", [None, "abs_one", "soft_asymmetric"])
@pytest.mark.parametrize("mode", ["reference", "paper"])
def test_oracle_matches_autograd_on_normal(mode, reward_clip, popart):
    T, B, A = 9, 7, 3
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    x = gorc.make_inputs(5, T, B, A)
    x["rewards"] = (x["rewards"] * 3.0).astype(np.float32)  # past the clip ranges
    got = gorc.vtrace_loss(x["v"], x["cur"], x["beh"], x["actions"], x["rewards"], x["done"], x["lens"], hp, B,
                           mode, reward_clip, popart)
    want = _torch_update(x, hp, B, mode, reward_clip, popart)
    valid = np.arange(T)[:, None] < x["lens"][None, :]
    for k in ("log_pi", "entropy", "kl"):
        np.testing.assert_allclose(np.where(valid, got[k], 0.0), want[k], rtol=0, atol=1e-12, err_msg=k)
    for k in ("vs", "pg_adv", "dparams", "dv"):
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-12, err_msg=k)
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "total_loss"):
        assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), (k, got[k], want[k])
    raw = float(np.where(valid, x["rewards"].astype(np.float64), 0.0).sum() / B)
    assert got["batch_mean_reward"] == raw
    assert got["diag"][0] == valid.sum() and abs(got["diag"][4] - want["kl"].sum()) <= 1e-12 * max(1, got["diag"][4])


@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
@pytest.mark.parametrize("frames", [1, 4])
def test_layout_act(obs_dtype, frames):
    lib = _cabi.lib()
    T, B, F, A = 20, 96, 7, 6
    code = _cabi.obs_dtype_code(obs_dtype)

    def lay(fn, *args):
        offs, tot = (C.c_int64 * 6)(), C.c_int64()
        assert fn(*args, offs, C.byref(tot)) == 0
        return list(offs), tot.value

    cat = lay(lib.impala_batch_layout_act, T, B, F, frames, A, code, _cabi.ACT_CATEGORICAL)
    assert cat == lay(lib.impala_batch_layout_frames, T, B, F, frames, A, code)
    offs, tot = lay(lib.impala_batch_layout_act, T, B, F, frames, A, code, _cabi.ACT_GAUSSIAN)
    ob = 1 if obs_dtype == "uint8" else 4
    sizes = [(T + frames) * B * F * ob, T * B * 2 * A * 4, T * B * A * 4, T * B * 4, T * B, B * 4]
    off = 0
    for i, n in enumerate(sizes):
        assert offs[i] == off and off % 256 == 0
        off = (off + n + 255) // 256 * 256
    assert tot == off
    assert (offs, tot) == _cabi.batch_layout(T, B, F * frames, A, obs_dtype, frames, "gaussian")
    bad = (C.c_int64 * 6)()
    assert lib.impala_batch_layout_act(T, B, F, frames, A, code, 2, bad, C.byref(C.c_int64())) == -1


def _no_cuda(*a, **k):
    raise AssertionError("CUDA was touched before the arguments were checked")


@pytest.mark.parametrize("bad", [dict(action_dist="normal"), dict(action_dist=None), dict(action_dist="gaussian", A=17),
                                 dict(action_dist="gaussian", A=32)])
def test_engine_refuses_bad_action_dist_before_cuda(monkeypatch, bad):
    from torched_impala_b200.engine import LearnerEngine

    monkeypatch.setattr(torch.cuda, "is_available", _no_cuda)
    monkeypatch.setattr(_cabi, "lib", _no_cuda)
    hp = default_hparams(batch_size=8, max_timesteps=5)
    A = bad.get("A", 2)
    with pytest.raises(ValueError):
        LearnerEngine(5, 8, 4, A, 8, 8, hp, action_dist=bad["action_dist"])
    for A in (1, 16):  # good values go on to the device checks
        with pytest.raises(AssertionError):
            LearnerEngine(5, 8, 4, A, 8, 8, hp, action_dist="gaussian")


def test_header_and_signature():
    hdr = open(os.path.join(ROOT, "include", "impala_b200.h")).read()
    for fn in ("impala_vtrace_loss_gauss", "impala_batch_layout_act", "impala_ingest_shard_act",
               "impala_batch_compose_act"):
        assert re.search(rf"\bint {fn}\(", hdr), fn
    assert "#define IMPALA_ACT_CATEGORICAL 0" in hdr and "#define IMPALA_ACT_GAUSSIAN 1" in hdr
    assert _cabi.ACT_DISTS == {"categorical": 0, "gaussian": 1}
    assert _cabi.SIGNATURES["impala_vtrace_loss_gauss"] == _cabi.SIGNATURES["impala_vtrace_loss_rclip"]


def test_library_exports_entry_points():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([nm, "-D", "--defined-only", _cabi.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    for fn in ("impala_vtrace_loss_gauss", "impala_batch_layout_act", "impala_ingest_shard_act",
               "impala_batch_compose_act"):
        assert re.search(rf"\bT {fn}$", out, re.M), fn


@pytest.fixture(scope="module")
def gauss_sass():
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
            t = re.search(r"vtrace_gauss_kernelI((?:L[ib]\d+E)+)E", m.group(1))
            cur = tuple(int(v) for v in re.findall(r"L[ib](\d+)E", t.group(1))) if t else None
            if cur is not None:
                kernels[cur] = Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and cur is not None:
            kernels[cur][m.group(1)] += 1
    return kernels


def test_gauss_instantiations(gauss_sass):
    # template arguments: AP, S, MAXT, MINB, VEC, DIAG, POPART, RCLIP
    assert len(gauss_sass) == 48  # AP 2, 4, 8, 16 x VEC x {plain, diag, popart} x reward clip
    assert {k[:2] for k in gauss_sass} == {(2, 2), (4, 2), (8, 1), (16, 1)}


@pytest.mark.parametrize("A", [1, 2, 6, 8, 16])
def test_gauss_kernels_at_launcher_shapes_do_not_spill(gauss_sass, A):
    ap = next(p for p in (2, 4, 8, 16) if A <= p)
    vec = int(A == ap)
    picked = {k: ops for k, ops in gauss_sass.items() if k[0] == ap and k[4] == vec}
    assert len(picked) == 6
    for k, ops in picked.items():
        assert not (ops["LDL"] or ops["STL"]), (k, ops["LDL"], ops["STL"])
