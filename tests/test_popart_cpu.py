"""CPU: PopArt - the float64 oracle against an independent torch-autograd restatement, its properties (output
preservation, scale invariance, folding), argument checks, the Learner config and the C ABI declarations."""
import os
import re

import numpy as np
import pytest
import torch

import popart_oracle as porc
from conftest import PKEYS
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.optim import check_popart_args
from torched_impala_b200.utils import default_hparams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch_update(params, batch, hp, mu, nu, beta, optimizer):
    """One PopArt update restated with torch autograd in float64: nn.Linear heads, the normalized loss,
    clip_grad_norm_, torch.optim.Adam / RMSprop, then the statistics and the rescale."""
    torch.manual_seed(0)
    pi = [torch.tensor(np.asarray(params["policy"][k], np.float64), requires_grad=True) for k in PKEYS]
    vf = [torch.tensor(np.asarray(params["value_fn"][k], np.float64), requires_grad=True) for k in PKEYS]
    head = torch.nn.Linear(vf[2].shape[1], 1).double()
    with torch.no_grad():
        head.weight.copy_(vf[2]), head.bias.copy_(vf[3])
    obs = torch.tensor(np.asarray(batch["obs"], np.float64))
    T = obs.shape[0] - 1
    B = obs.shape[1]
    sigma = porc.sigma_of(mu, nu)
    n = head(torch.relu(obs @ vf[0].T + vf[1]))[..., 0]
    logits = torch.relu(obs[:-1] @ pi[0].T + pi[1]) @ pi[2].T + pi[3]
    v = sigma * n + mu
    vs, pg, _ = porc.orc.vtrace(v.detach().numpy(), logits.detach().numpy(), batch["beh_logits"], batch["actions"],
                                batch["rewards"], batch["done"], batch["lens"], hp.gamma, hp.rho_bar, hp.c_bar)
    vs_t, pg_t = torch.tensor(vs), torch.tensor(pg / sigma)
    lens = torch.tensor(batch["lens"])
    valid_v = torch.arange(T + 1)[:, None] <= lens[None, :]
    valid = torch.arange(T)[:, None] < lens[None, :]
    vl = 0.5 * (torch.where(valid_v, (v - vs_t) / sigma, 0.0) ** 2).sum()
    lsm = torch.log_softmax(logits, -1)
    nll = -lsm.gather(-1, torch.tensor(batch["actions"], dtype=torch.int64)[..., None])[..., 0]
    pl = torch.where(valid, nll * pg_t, 0.0).sum()
    ent = torch.where(valid, -(lsm.exp() * lsm).sum(-1), 0.0).sum()
    total = (hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * ent) / B
    ps = pi + [vf[0], vf[1], head.weight, head.bias]
    total.backward()
    torch.nn.utils.clip_grad_norm_(pi, hp.max_norm)
    torch.nn.utils.clip_grad_norm_(ps[4:], hp.max_norm)
    if optimizer == "adam":
        opt = torch.optim.Adam(ps, lr=hp.lr)
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.95)
    else:
        opt = torch.optim.RMSprop(ps, lr=hp.lr, alpha=0.99, eps=0.01)
        sched = None
    opt.step()
    if sched is not None:
        sched.step()
    m = valid.numpy()
    n_, s1, s2 = float(m.sum()), float(vs[:T][m].sum()), float((vs[:T][m] ** 2).sum())
    mu1, nu1, sg1 = porc.stats_update(mu, nu, n_, s1, s2, beta)
    with torch.no_grad():
        head.weight.mul_(sigma / sg1)
        head.bias.copy_((sigma * head.bias + mu - mu1) / sg1)
    return [p.detach().numpy() for p in ps], (mu1, nu1, sg1)


@pytest.mark.parametrize("optimizer", ["adam", "rmsprop"])
@pytest.mark.parametrize("mu,nu", [(0.0, 1.0), (1.5, 6.0), (-20.0, 500.0)])
def test_oracle_matches_torch_autograd(optimizer, mu, nu):
    T, B, O, A, H = 12, 9, 5, 3, 16
    hp = default_hparams(batch_size=B, max_timesteps=T, rho_bar=1.0, c_bar=0.9)
    params = synth.init_params(11, O, A, H)
    batch = synth.make_batch(12, T, B, O, A, ragged=True)
    kw = dict(optimizer_kwargs=dict(alpha=0.99, eps=0.01)) if optimizer == "rmsprop" else {}
    if optimizer == "rmsprop":
        kw["lr_lambda"] = lambda e: 1.0
    ref = porc.BatchedLearner(params, hp, optimizer, beta=0.3, mu=mu, nu=nu, **kw)
    ref.update(batch)
    want, stats = _torch_update(params, batch, hp, mu, nu, 0.3, optimizer)
    for got, w in zip(ref.pi + ref.vf, want):
        assert np.allclose(got, np.asarray(w).reshape(got.shape), rtol=0, atol=1e-12)
    assert np.allclose((ref.mu, ref.nu, ref.sigma), stats, rtol=1e-12, atol=0)


def test_output_preservation_and_fold_round_trip():
    rng = np.random.default_rng(3)
    vf = [rng.standard_normal((8, 4)), rng.standard_normal(8), rng.standard_normal((1, 8)), rng.standard_normal(1)]
    hid = np.maximum(rng.standard_normal((50, 4)) @ vf[0].T + vf[1], 0)
    mu, sigma = 2.0, 3.0
    before = sigma * (hid @ vf[2].T + vf[3]) + mu
    learner = porc.BatchedLearner.__new__(porc.BatchedLearner)
    learner.vf, learner.mu, learner.nu, learner.sigma, learner.beta = [x.copy() for x in vf], mu, mu * mu + 9.0, sigma, 0.4
    learner.popart_step(100.0, 100.0 * 7.0, 100.0 * 80.0)
    after = learner.sigma * (hid @ learner.vf[2].T + learner.vf[3]) + learner.mu
    assert learner.sigma != sigma and np.allclose(after, before, rtol=1e-13, atol=1e-12)
    back = porc.unfold(porc.fold(vf, mu, sigma), mu, sigma)
    for a, b in zip(back, vf):
        assert np.allclose(a, b, rtol=1e-15, atol=1e-15)


def test_oracle_scale_invariance():
    T, B, O, A, H = 10, 6, 4, 3, 8
    hp = default_hparams(batch_size=B, max_timesteps=T)
    params = synth.init_params(2, O, A, H)
    batch = synth.make_batch(5, T, B, O, A, ragged=True)
    a = porc.BatchedLearner(params, hp, beta=0.2)
    b = porc.BatchedLearner(params, hp, beta=0.2, mu=0.0, nu=1024.0 ** 2)
    big = dict(batch, rewards=batch["rewards"] * 1024.0)
    for _ in range(3):
        a.update(batch), b.update(big)
    for x, y in zip(a.pi + a.vf, b.pi + b.vf):
        assert np.allclose(x, y, rtol=1e-12, atol=1e-14)
    assert np.isclose(b.sigma, 1024.0 * a.sigma, rtol=1e-12)


@pytest.mark.parametrize("bad", [0.0, -0.1, 1.5, float("nan"), float("inf"), "x"])
def test_bad_beta_refused(bad):
    with pytest.raises(ValueError):
        check_popart_args(True, bad)


def test_switch_must_be_bool():
    with pytest.raises(ValueError):
        check_popart_args("yes", 3e-4)
    assert check_popart_args(False, 1.0) == 1.0


def test_learner_cfg_carries_popart():
    import multiprocessing as mp

    from torched_impala_b200.learner import Learner

    class Net(torch.nn.Module):
        def __init__(self, O, H, N2):
            super().__init__()
            self.model = torch.nn.Sequential(torch.nn.Linear(O, H), torch.nn.Dropout(0.0), torch.nn.ReLU(),
                                             torch.nn.Linear(H, N2))

    hp = default_hparams(batch_size=8, max_timesteps=5)
    ln = Learner(0, hp, Net(4, 8, 2), Net(4, 8, 1), mp.Queue(), None, popart=True, popart_beta=0.01)
    c = ln._cfg()
    assert c["popart"] is True and c["popart_beta"] == 0.01
    with pytest.raises(ValueError):
        Learner(0, hp, Net(4, 8, 2), Net(4, 8, 1), mp.Queue(), None, popart=True, popart_beta=2.0)


def test_header_and_signatures():
    hdr = open(os.path.join(ROOT, "include", "impala_b200.h")).read()
    for name in ("impala_vtrace_loss_popart", "impala_clip_optim_popart", "impala_gather_clip_optim_popart"):
        assert re.search(rf"\bint {name}\(", hdr), name
        assert name in _cabi.SIGNATURES
    assert len(_cabi.SIGNATURES["impala_vtrace_loss_popart"][1]) == len(_cabi.SIGNATURES["impala_vtrace_loss_diag"][1]) + 1
    assert len(_cabi.SIGNATURES["impala_clip_optim_popart"][1]) == len(_cabi.SIGNATURES["impala_clip_optim"][1]) + 6
    assert (len(_cabi.SIGNATURES["impala_gather_clip_optim_popart"][1])
            == len(_cabi.SIGNATURES["impala_gather_clip_optim"][1]) + 6)
    assert "#define IMPALA_POPART_STATS 5" in hdr and _cabi.POPART_STATS == 5


def test_init_state_carries_statistics(tmp_path):
    from torched_impala_b200 import dp

    st = {"policy": {"a": np.ones(2)}, "value_fn": {"b": np.zeros(3)}}
    dp.write_init_state(str(tmp_path / "s.npz"), st, None, {"mu": 1.5, "nu": 4.0})
    got, table = dp.read_init_state(str(tmp_path / "s.npz"))
    assert table is None and float(got["popart"]["mu"]) == 1.5 and float(got["popart"]["nu"]) == 4.0
