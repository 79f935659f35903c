"""CPU: the shared-torso actor-critic (one hidden layer feeding the policy and the value head).

The float64 oracle (tests/shared_torso_oracle.py) against torch autograd on a float64 shared-torso module, for
categorical and Gaussian policies, with and without PopArt and reward clipping; the C ABI declarations, exports
and ctypes signatures; the refusals of LearnerEngine and Learner before any CUDA work; the state-dict views of
the one parameter block; and the split-head kernel twins in the built library's SASS."""
from collections import Counter
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import shared_torso_oracle as sorc
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, models, synth
from torched_impala_b200.engine import LearnerEngine, check_shared_torso
from torched_impala_b200.utils import default_hparams

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "impala_b200.h")
ENTRIES = ("impala_mlp_forward_shared", "impala_mlp_backward_shared")


# ------------------------------------------------------------------------------------ oracle vs autograd
class SharedNet(torch.nn.Module):
    def __init__(self, net):
        super().__init__()
        self.w1, self.b1, self.w2, self.b2 = (torch.nn.Parameter(torch.tensor(p, dtype=torch.float64)) for p in net)

    def forward(self, x):
        return torch.relu(x @ self.w1.T + self.b1) @ self.w2.T + self.b2


def _autograd_step(net, batch, r, hp, B, gaussian, popart):
    """The loss of the shared network in torch (vs and pg_adv are constants, as under no_grad at learner.py:120),
    its gradient, then clip_grad_norm_ over the whole network and torch.optim.Adam at 0.95 lr."""
    m = SharedNet(net)
    obs = torch.tensor(batch["obs"], dtype=torch.float64)
    out = m(obs)
    T = out.shape[0] - 1
    lens = torch.tensor(batch["lens"]).long()
    valid = (torch.arange(T)[:, None] < lens[None, :]).double()
    valid_v = (torch.arange(T + 1)[:, None] <= lens[None, :]).double()
    mu, sigma = popart if popart else (0.0, 1.0)
    v = out[..., -1] * sigma + mu
    vs = torch.tensor(r["vs"])
    pg = torch.tensor(r["pg_adv"])  # normalized under PopArt already
    z = out[:-1, :, :-1]
    if gaussian:
        A = z.shape[-1] // 2
        dist = torch.distributions.Normal(z[..., :A], torch.exp(z[..., A:]))
        lp = dist.log_prob(torch.tensor(batch["actions"], dtype=torch.float64)).sum(-1)
        ent = dist.entropy().sum(-1)
    else:
        lsm = torch.log_softmax(z, -1)
        lp = lsm.gather(-1, torch.tensor(batch["actions"]).long()[..., None])[..., 0]
        ent = -(lsm.exp() * lsm).sum(-1)
    vl = 0.5 * (((v - vs) / sigma) ** 2 * valid_v).sum()
    pl = (-lp * pg * valid).sum()
    pe = (ent * valid).sum()
    total = (hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * pe) / B
    total.backward()
    grads = [p.grad.detach().clone().numpy() for p in m.parameters()]
    norm = float(torch.nn.utils.clip_grad_norm_(list(m.parameters()), hp.max_norm))
    opt = torch.optim.Adam(m.parameters(), lr=0.95 * hp.lr, betas=(0.9, 0.999), eps=1e-8)
    opt.step()
    return float(total.detach()), grads, norm, [p.detach().numpy() for p in m.parameters()]


@pytest.mark.parametrize("reward_clip", [None, "soft_asymmetric"])
@pytest.mark.parametrize("popart", [False, True])
@pytest.mark.parametrize("gaussian", [False, True])
def test_oracle_matches_autograd(gaussian, popart, reward_clip):
    T, B, O, A, H = 6, 5, 7, 3, 16
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    N = 2 * A if gaussian else A
    params = synth.init_params(3, O, N, H)
    batch = (synth.make_gaussian_batch(5, T, B, O, A, ragged=True, params=params) if gaussian
             else synth.make_batch(5, T, B, O, A, ragged=True))
    mu, nu = (0.4, 2.0) if popart else (0.0, 1.0)
    lrn = sorc.SharedLearner(params, hp, gaussian=gaussian, reward_clip=reward_clip, popart=popart, mu=mu, nu=nu)
    net0 = [p.copy() for p in lrn.net]
    r = lrn.forward_backward(batch)
    total, grads, norm, after = _autograd_step(net0, batch, r, hp, B, gaussian, (mu, lrn.sigma) if popart else None)
    assert abs(r["total_loss"] - total) < 1e-12 * max(1.0, abs(total))
    for g, w in zip(r["grad"], grads):
        assert np.abs(g - w).max() < 1e-12 * max(1.0, np.abs(w).max())
    # the policy outputs' rows >= T B have no gradient, the value column gets one on every row
    assert np.abs(r["grad"][3][-1] - r["dv"].sum()) < 1e-12 * max(1.0, abs(r["dv"].sum()))
    n = lrn.apply(r["grad"])
    assert abs(n["norm_policy"] - norm) < 1e-12 * norm and n["norm_value"] == 0.0
    for p, w in zip(lrn.net, after):
        assert np.abs(p - w).max() < 1e-12


def test_popart_rescale_touches_only_the_value_head():
    T, B, O, A, H = 5, 4, 6, 2, 8
    hp = default_hparams(batch_size=B, max_timesteps=T)
    lrn = sorc.SharedLearner(synth.init_params(2, O, A, H), hp, popart=True, beta=0.5)
    before = [p.copy() for p in lrn.net]
    out = orc.mlp_forward(synth.make_batch(1, T, B, O, A)["obs"].astype(np.float64), *lrn.net)[0]
    folded = out[..., -1] * lrn.sigma + lrn.mu
    lrn.popart_step(10.0, 30.0, 200.0)
    assert all(np.array_equal(a, b) for a, b in zip(before[:2], lrn.net[:2]))
    assert np.array_equal(before[2][:-1], lrn.net[2][:-1]) and np.array_equal(before[3][:-1], lrn.net[3][:-1])
    out1 = orc.mlp_forward(synth.make_batch(1, T, B, O, A)["obs"].astype(np.float64), *lrn.net)[0]
    assert np.abs(out1[..., -1] * lrn.sigma + lrn.mu - folded).max() < 1e-9  # output-preserving


# ---------------------------------------------------------------------------------------------- C ABI
def _decl_params(name):
    text = open(HEADER).read()
    m = re.search(rf"\b{name}\(([^)]*)\)\s*;", text)
    assert m, f"{name} is not declared in include/impala_b200.h"
    return [p.strip() for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", ENTRIES)
def test_header_export_and_signature(name):
    params = _decl_params(name)
    res, args = _cabi.SIGNATURES[name]
    assert res is C.c_int and len(args) == len(params), (name, len(args), len(params))
    for p, a in zip(params, args):
        want = C.c_void_p if "*" in p else C.c_int64 if p.startswith("int64_t") else C.c_int
        assert a is want, (name, p, a)
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    assert hasattr(C.CDLL(_cabi.LIB_PATH), name)


# ------------------------------------------------------------------------------------------ refusals
def test_check_shared_torso():
    assert check_shared_torso(False, 64, 128, 40) is False  # off: nothing is checked
    assert check_shared_torso(True, 256, 256, 31) is True
    with pytest.raises(ValueError, match="H_pi"):
        check_shared_torso(True, 128, 256, 4)
    with pytest.raises(ValueError, match="31 policy outputs"):
        check_shared_torso(True, 128, 128, 32)


@pytest.mark.parametrize("kw", [dict(A=4, H_pi=128, H_v=256), dict(A=32, H_pi=128, H_v=128),
                                dict(A=16, H_pi=128, H_v=128, action_dist="gaussian")])
def test_engine_refuses_before_cuda(kw, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)  # reached only if the check did not fire
    a = dict(kw)
    with pytest.raises(ValueError):
        LearnerEngine(20, 8, 24, a.pop("A"), a.pop("H_pi"), a.pop("H_v"), default_hparams(batch_size=8),
                      shared_torso=True, **a)


def test_learner_refuses_in_the_launching_process():
    from torched_impala_b200.learner import Learner

    hp = default_hparams(batch_size=8, max_timesteps=20)
    with pytest.raises(ValueError, match="H_pi"):
        Learner(0, hp, models.MlpPolicy(24, 4, 128), models.MlpValueFn(24, 64), None, None, shared_torso=True)
    with pytest.raises(ValueError, match="31 policy outputs"):
        Learner(0, hp, models.MlpPolicy(24, 32, 64), models.MlpValueFn(24, 64), None, None, shared_torso=True)


# ------------------------------------------------------------------------------------- state views
def _host_engine(O, N, H):
    """The parameter bookkeeping of a shared-torso engine, without its device buffers."""
    eng = LearnerEngine.__new__(LearnerEngine)
    eng.shared_torso, eng.O, eng.N_pi, eng.H_pi, eng.H_v = True, O, N, H, H
    eng.pi_off, eng.n_pi = _cabi.param_layout(O, H, N + 1)
    eng.n_total = eng.n_pi
    return eng


def test_views_of_the_block_round_trip():
    O, N, H = 24, 5, 64
    eng = _host_engine(O, N, H)
    rng = np.random.default_rng(0)
    net = [rng.standard_normal(s) for s in ((H, O), (H,), (N + 1, H), (N + 1,))]
    v = sorc.views(net)
    flat = np.zeros(eng.n_total)
    for grp, key, off, shp in eng._segments():  # what load_state writes (the value torso is skipped there)
        if grp == "value_fn" and key in orc.PKEYS[:2]:
            continue
        flat[off:off + int(np.prod(shp))] = np.asarray(v[grp][key]).reshape(-1)
    back = {"policy": {}, "value_fn": {}}
    for grp, key, off, shp in eng._segments():  # what state() reads
        back[grp][key] = flat[off:off + int(np.prod(shp))].reshape(shp)
    for g in back:
        for k in orc.PKEYS:
            assert np.array_equal(back[g][k], v[g][k]), (g, k)
    w = sorc.join(back["policy"], back["value_fn"])
    assert all(np.array_equal(a, b) for a, b in zip(w, net))
    # the block's layout: W2 rows [policy | value] and b2 entries, contiguous
    assert eng.pi_off[2] + N * H == dict((k, o) for g, k, o, _ in eng._segments() if g == "value_fn")[orc.PKEYS[2]]


def test_shared_checkpoint_loads_into_the_reference_modules(tmp_path):
    O, A, H = 8, 3, 32
    net = sorc.join(synth.init_params(1, O, A, H)["policy"], synth.init_params(1, O, A, H)["value_fn"])
    v = sorc.views(net, 0.5, 2.0)
    ckpt = {"policy_state_dict": {k: torch.tensor(t) for k, t in v["policy"].items()},
            "value_fn_state_dict": {k: torch.tensor(t) for k, t in v["value_fn"].items()}, "shared_torso": True}
    torch.save(ckpt, tmp_path / "c.pt")
    got = torch.load(tmp_path / "c.pt")
    pol, vf = models.MlpPolicy(O, A, H).double().eval(), models.MlpValueFn(O, H).double().eval()
    pol.load_state_dict(got["policy_state_dict"])
    vf.load_state_dict(got["value_fn_state_dict"])
    x = torch.randn(5, O, dtype=torch.float64)
    want = orc.mlp_forward(x.numpy(), *net)[0]
    with torch.no_grad():
        assert np.abs(pol(x).numpy() - want[:, :A]).max() < 1e-12
        assert np.abs(vf(x).numpy()[:, 0] - (want[:, A] * 2.0 + 0.5)).max() < 1e-12


# ------------------------------------------------------------------------------------------- SASS
MLP_KERNELS = ("mlp_fwd_tc", "mlp_bwd_tc", "mlp_bwd_tcw", "mlp_fwd_obs", "mlp_bwd_obs_pre", "mlp_fwd", "mlp_bwd")


@pytest.fixture(scope="module")
def sass():
    """{kernel key: (SASS mnemonic counts, resource usage)} of the MLP kernels; key = the demangled name and
    template arguments, e.g. "mlp_fwd_tc_split_kernel<4, 1>" (a split-head twin) and "mlp_fwd_tc_kernel<4, 1>" (its
    dense twin)."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not shutil.which("c++filt"):
        pytest.skip("cuobjdump / c++filt not available")
    if not os.path.exists(_cabi.LIB_PATH):
        pytest.fail(f"{_cabi.LIB_PATH} has not been built")
    out = subprocess.run([exe, "-sass", _cabi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    ops, cur = {}, None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            ops[cur] = Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+(?:\.[A-Za-z0-9_]+)*)", ln)
        if m and cur:
            parts = m.group(1).split(".")
            for i in range(1, len(parts) + 1):  # every dot prefix: HGMMA, HGMMA.64x64x8, ...
                ops[cur][".".join(parts[:i])] += 1
    res = subprocess.run([exe, "-res-usage", _cabi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", res))
    names = list(ops)
    dm = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    found = {}
    for n, d in zip(names, dm.splitlines()):
        m = re.search(r"(?:::|\s)((\w+?)(?:_split)?_kernel(?:<[^()]*>)?)\(", d)
        if m and m.group(2) in MLP_KERNELS:
            found[m.group(1)] = (ops[n], usage.get(n, ""))
    return found


def _is_twin(key):
    """Tensor-core and K-streamed twins are kernels of their own names; the FP32 twins are SPLIT = true."""
    return "_split_kernel" in key or (key.startswith(("mlp_fwd_kernel", "mlp_bwd_kernel")) and key.endswith(", true>"))


def _fp32(key):
    return key.startswith(("mlp_fwd_kernel", "mlp_bwd_kernel"))


def _dense(twin):
    if _fp32(twin):
        return twin[:-len(", true>")] + ", false>"
    d = twin.replace("_split_kernel", "_kernel")
    return d + "<4>" if d == "mlp_bwd_tc_kernel" else d  # the narrow backward's twin has NP = 4 fixed


def test_split_twins_match_their_dense_twins(sass):
    twins = [k for k in sass if _is_twin(k)]
    tc = [k for k in twins if not _fp32(k)]
    # forward: 3 NP x 3 K-atom counts; backward: 1 narrow + 6 wide; obs: 2 NP x 2 element types, each direction
    assert len(tc) == 24, sorted(tc)
    assert len(twins) > len(tc)  # the FP32 twins
    for k in twins:
        targs = re.findall(r"\d+", k.split("<", 1)[1]) if "<" in k else ["4"]
        assert targs[2 if _fp32(k) else 0] != "1", k  # one output: no twin
        assert _dense(k) in sass, k
        (o, _), (c, _) = sass[k], sass[_dense(k)]
        for op in ("HGMMA", "WARPGROUP.DEPBAR", "WARPGROUP.ARRIVE"):
            assert o[op] == c[op], (k, op, o[op], c[op])
        if k.startswith(("mlp_fwd_tc_split_kernel<4, 1>", "mlp_bwd_tc_split_kernel")):  # narrow: m64n64 MMAs
            assert o["HGMMA.64x64x8"] > 0, k


def test_split_twins_do_not_spill(sass):
    """No tensor-core twin has a stack frame; an FP32 twin has exactly its dense twin's (the butterfly array of the
    instantiations that do not keep it in registers, which is not a spill)."""
    def frame(u):
        return re.search(r"STACK:(\d+)", u).group(1), re.search(r"LOCAL:(\d+)", u).group(1)

    for k, (_, u) in sass.items():
        if _is_twin(k):
            if _fp32(k):
                assert frame(u) == frame(sass[_dense(k)][1]), (k, u)
            else:
                assert frame(u) == ("0", "0"), (k, u)
