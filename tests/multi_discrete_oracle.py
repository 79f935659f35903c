"""TEST INFRASTRUCTURE - float64 numpy statement of impala_vtrace_loss_md (multi-discrete policies).

K independent softmax heads over the N = sum n_k policy outputs, head k owning z[s_k : s_k + n_k]; the action is one
index a_k per head, actions (T, B, K).  With p the softmax within a head:
    log pi(a)  = sum_k log p_k(a_k)                 (the same for mu with the behaviour logits)
    H          = sum_k H_k,  H_k = -sum_{j in k} p_j log p_j
    KL(mu||pi) = sum_k KL_k
    dz_j       = inv_batch [policy_loss_c pg_adv (p_j - [j = s_k + a_k]) + entropy_c p_j (log p_j + H_k)], j in head k
The ratio pi(a) / mu(a) enters tests/gaussian_oracle.py's vtrace_from_ratio (both modes, the reference's quirks);
the losses, the reward transform (tests/reward_clip_oracle.py) and PopArt's (mu, sigma) are those of the Gaussian
oracle.  K = 1 is the categorical policy of oracle/impala_oracle.py.
"""
from __future__ import annotations

import numpy as np

import reward_clip_oracle as rorc
from gaussian_oracle import vtrace_from_ratio
from oracle import impala_oracle as orc

F64 = np.float64


def starts(heads):
    return np.concatenate([[0], np.cumsum(heads)[:-1]]).astype(int)


def head_log_softmax(z, heads):
    """log p per output (..., N): the log-softmax within each head."""
    z = np.asarray(z, F64)
    return np.concatenate([orc.log_softmax(z[..., s:s + n]) for s, n in zip(starts(heads), heads)], -1)


def log_prob(z, actions, heads):
    lz = head_log_softmax(z, heads)
    a = np.asarray(actions).astype(np.int64) + starts(heads)
    return np.take_along_axis(lz, a, -1).sum(-1)


def head_entropy(z, heads):
    """(..., K) per-head entropies."""
    lz = head_log_softmax(z, heads)
    return np.stack([-(np.exp(lz[..., s:s + n]) * lz[..., s:s + n]).sum(-1) for s, n in zip(starts(heads), heads)], -1)


def kl(z_beh, z_cur, heads):
    """KL(mu || pi) per step, summed over the heads."""
    lb, lc = head_log_softmax(z_beh, heads), head_log_softmax(z_cur, heads)
    return (np.exp(lb) * (lb - lc)).sum(-1)


def vtrace_loss(v, cur, beh, actions, rewards, done, lens, hp, batch_size, heads, mode="reference", reward_clip=None,
                popart=None):
    """Every output of impala_vtrace_loss_md in float64 (names as tests/gaussian_oracle.py's vtrace_loss, dlogits
    in place of dparams)."""
    heads = tuple(heads)
    T, B = np.asarray(rewards).shape
    lens = np.asarray(lens)
    mu_p, sigma = (0.0, 1.0) if popart is None else (float(popart[0]), float(popart[1]))
    v = sigma * np.asarray(v, F64) + mu_p
    r = np.asarray(rewards, F64) if reward_clip is None else rorc.clip_rewards(rewards, reward_clip)
    valid = np.arange(T)[:, None] < lens[None, :]
    valid_v = np.arange(T + 1)[:, None] <= lens[None, :]
    lp, lpb = log_prob(cur, actions, heads), log_prob(beh, actions, heads)
    ratio = np.exp(lp - lpb)
    vs, pg_r, rho = vtrace_from_ratio(v, ratio, r, done, lens, hp.gamma, hp.rho_bar, hp.c_bar, mode)
    pg = pg_r / sigma
    err = np.where(valid_v, v - vs, 0.0) / sigma
    hk = head_entropy(cur, heads)
    ent = hk.sum(-1)
    inv_b = 1.0 / batch_size
    vl = 0.5 * (err ** 2).sum() * inv_b
    pl = np.where(valid, -lp * pg, 0.0).sum() * inv_b
    pe = np.where(valid, ent, 0.0).sum() * inv_b
    with np.errstate(invalid="ignore"):
        rw = np.where(valid, np.asarray(rewards, F64), 0.0).sum() * inv_b
    dv = hp.v_loss_c * err * inv_b
    lz = head_log_softmax(cur, heads)
    p = np.exp(lz)
    onehot = np.zeros_like(p)
    a = np.asarray(actions).astype(np.int64) + starts(heads)
    np.put_along_axis(onehot, a, 1.0, -1)
    h_of = np.repeat(hk, heads, -1)  # H_k at every output of head k
    dl = inv_b * (hp.policy_loss_c * pg[..., None] * (p - onehot) + hp.entropy_c * p * (lz + h_of))
    dlogits = np.where(valid[..., None], dl, 0.0)
    klt = kl(beh, cur, heads)
    vs_t = vs[:T]
    diag = np.array([valid.sum(), np.where(valid, lp - lpb, 0.0).sum(), (valid & (ratio > hp.rho_bar)).sum(),
                     (valid & (ratio > hp.c_bar)).sum(), np.where(valid, klt, 0.0).sum(),
                     np.where(valid, vs_t, 0.0).sum(), np.where(valid, vs_t ** 2, 0.0).sum(),
                     np.where(valid, vs_t - v[:T], 0.0).sum()], F64)
    return dict(vs=vs, pg_adv=pg, rho=rho, ratio=ratio, value_fn_loss=vl, policy_loss=pl, policy_entropy=pe,
                batch_mean_reward=rw, scalars=np.array([vl, pl, pe, rw]), dv=dv, dlogits=dlogits, log_pi=lp,
                entropy=ent, kl=klt, diag=diag,
                total_loss=hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * pe)


def make_inputs(seed, T, B, heads, ragged=True, spread=(0.1, 0.3)):
    """Current logits ~ 2 N(0, 1); behaviour logits perturbed by 0.1-0.3 from them; one action per head sampled from
    the behaviour policy; float32 / int32 like the slabs.  Ragged: lens in [0, T], some columns empty, some full."""
    heads = tuple(heads)
    rng = np.random.default_rng(seed)
    N, K = sum(heads), len(heads)
    cur = (2.0 * rng.standard_normal((T, B, N))).astype(np.float32)
    beh = (cur + rng.uniform(*spread, (T, B, N)) * rng.choice([-1.0, 1.0], (T, B, N))).astype(np.float32)
    act = np.zeros((T, B, K), np.int32)
    lb = head_log_softmax(beh, heads)
    for k, (s, n) in enumerate(zip(starts(heads), heads)):
        cdf = np.cumsum(np.exp(lb[..., s:s + n]), -1)
        act[..., k] = np.minimum((rng.uniform(size=(T, B, 1)) > cdf).sum(-1), n - 1)
    lens = rng.integers(0, T + 1, B).astype(np.int32) if ragged else np.full(B, T, np.int32)
    if ragged and B >= 3:
        lens[0], lens[1] = 0, T
    rewards = rng.standard_normal((T, B)).astype(np.float32)
    done = (rng.uniform(size=(T, B)) < 0.05).astype(np.uint8)
    pad = np.arange(T)[:, None] >= lens[None, :]
    beh[pad], act[pad], rewards[pad], done[pad] = 0.0, 0, 0.0, 0
    v = rng.standard_normal((T + 1, B)).astype(np.float32)
    return dict(cur=cur, beh=beh, actions=act, rewards=rewards, done=done, lens=lens, v=v)


class MdLearner(orc.BatchedLearner):
    """The oracle learner with the multi-discrete policy terms."""

    def __init__(self, params, hp, heads):
        super().__init__(params, hp)
        self.heads = tuple(heads)

    def forward_backward(self, batch, mode="reference", batch_size=None):
        hp = self.hp
        B_glob = hp.batch_size if batch_size is None else batch_size
        obs = np.asarray(batch["obs"], np.float64)
        Tp1, B, O = obs.shape
        T = Tp1 - 1
        v2, v_pre = orc.mlp_forward(obs, *self.vf)
        z, pi_pre = orc.mlp_forward(obs[:-1], *self.pi)
        out = vtrace_loss(v2[..., 0], z, batch["beh_logits"], batch["actions"], batch["rewards"], batch["done"],
                          batch["lens"], hp, B_glob, self.heads, mode)
        out["g_policy"] = list(orc.mlp_backward(obs[:-1].reshape(T * B, O), pi_pre.reshape(T * B, -1), self.pi[2],
                                                out["dlogits"].reshape(T * B, -1)))
        out["g_value"] = list(orc.mlp_backward(obs.reshape(Tp1 * B, O), v_pre.reshape(Tp1 * B, -1), self.vf[2],
                                               out["dv"].reshape(Tp1 * B, 1)))
        return out
