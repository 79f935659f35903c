"""TEST INFRASTRUCTURE - float64 numpy statement of impala_vtrace_loss_gauss (diagonal Gaussian policies).

The policy outputs z = [m | s] (T, B, 2A): means m_k and log standard deviations s_k, sigma_k = e^{s_k}.  The
behaviour record is the actor's [m | s], the action the unsquashed sample a (T, B, A).
    log pi(a) = sum_k [-((a_k - m_k) / sigma_k)^2 / 2 - s_k - log(2 pi) / 2]    (torch Normal.log_prob summed)
    H         = sum_k [s_k + (1 + log(2 pi)) / 2]
    KL(mu||pi)= sum_k [s_k - sb_k + (sigma_b,k^2 + (mb_k - m_k)^2) / (2 sigma_k^2) - 1/2]
The ratio pi(a) / mu(a) enters the V-trace recurrence of oracle/impala_oracle.py (both modes, the reference's
quirks included); the losses keep the reference's structure (learner.py:149-162): value 0.5 sum (v - vs)^2,
policy sum -log pi(a) pg_adv, entropy sum H, each sum_b .. / batch_size.  Options on top, as the kernel has them:
the reward transform of tests/reward_clip_oracle.py and PopArt statistics (mu, sigma) of tests/popart_oracle.py.
"""
from __future__ import annotations

import numpy as np

import reward_clip_oracle as rorc
from oracle import impala_oracle as orc

F64 = np.float64
HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)


def split(z):
    z = np.asarray(z, F64)
    A = z.shape[-1] // 2
    return z[..., :A], z[..., A:]


def log_prob(z, a):
    m, s = split(z)
    u = (np.asarray(a, F64) - m) * np.exp(-s)
    return (-0.5 * u * u - s - HALF_LOG_2PI).sum(-1)


def entropy(z):
    _, s = split(z)
    return (s + 0.5 + HALF_LOG_2PI).sum(-1)


def kl(z_beh, z_cur):
    """KL(mu || pi) per step, mu = the behaviour Gaussian, pi = the current one."""
    mb, sb = split(z_beh)
    m, s = split(z_cur)
    return (s - sb + (np.exp(2.0 * sb) + (mb - m) ** 2) / (2.0 * np.exp(2.0 * s)) - 0.5).sum(-1)


def vtrace_from_ratio(v, ratio, rewards, done, lens, gamma, rho_bar, c_bar, mode="reference"):
    """oracle/impala_oracle.py's vtrace (learner.py:116-135) with the importance ratio given."""
    v = np.asarray(v, F64)
    T, B = ratio.shape
    valid = np.arange(T)[:, None] < lens[None, :]
    rho = np.where(valid, np.minimum(ratio, rho_bar), 0.0)
    c = np.where(valid, np.minimum(ratio, c_bar), 0.0)
    disc = (np.float32(gamma) * (~done.astype(bool)).astype(np.float32)).astype(F64)
    disc = np.where(valid, disc, 0.0)
    r = np.asarray(rewards, F64)
    acc = np.zeros((T + 1, B), F64)
    if mode == "reference":
        delta = rho * (r + gamma * v[1:] - v[:1])
        for i in range(T - 1, -1, -1):
            acc[i] = delta[i] + disc[i] * c[i] * (acc[i + 1] - v[i + 1])
    elif mode == "paper":
        delta = rho * (r + disc * v[1:] - v[:-1])
        for i in range(T - 1, -1, -1):
            acc[i] = delta[i] + disc[i] * c[i] * acc[i + 1]
    else:
        raise ValueError(mode)
    vs = acc + v
    pg_adv = rho * (r + disc * vs[1:] - v[:-1])
    vs = np.where(np.arange(T + 1)[:, None] <= lens[None, :], vs, 0.0)
    return vs, pg_adv, rho


def vtrace_loss(v, cur, beh, actions, rewards, done, lens, hp, batch_size, mode="reference", reward_clip=None,
                popart=None):
    """Every output of impala_vtrace_loss_gauss in float64.

    v (T+1, B): the value output (normalized under popart = (mu, sigma), reward units otherwise); cur / beh
    (T, B, 2A); actions (T, B, A).  Returns vs, pg_adv, rho, the four scalars, dv, dparams (T, B, 2A), the per-step
    log_pi, entropy and kl, and diag: the eight off-policy sums of impala_vtrace_loss_diag."""
    T, B = np.asarray(rewards).shape
    lens = np.asarray(lens)
    mu_p, sigma = (0.0, 1.0) if popart is None else (float(popart[0]), float(popart[1]))
    v = sigma * np.asarray(v, F64) + mu_p  # reward units
    r = np.asarray(rewards, F64) if reward_clip is None else rorc.clip_rewards(rewards, reward_clip)
    valid = np.arange(T)[:, None] < lens[None, :]
    valid_v = np.arange(T + 1)[:, None] <= lens[None, :]
    lp, lpb = log_prob(cur, actions), log_prob(beh, actions)
    ratio = np.exp(lp - lpb)
    vs, pg_r, rho = vtrace_from_ratio(v, ratio, r, done, lens, hp.gamma, hp.rho_bar, hp.c_bar, mode)
    pg = pg_r / sigma
    err = np.where(valid_v, v - vs, 0.0) / sigma  # normalized error: the value loss and dv
    ent = entropy(cur)
    inv_b = 1.0 / batch_size
    vl = 0.5 * (err ** 2).sum() * inv_b
    pl = np.where(valid, -lp * pg, 0.0).sum() * inv_b
    pe = np.where(valid, ent, 0.0).sum() * inv_b
    with np.errstate(invalid="ignore"):
        rw = np.where(valid, np.asarray(rewards, F64), 0.0).sum() * inv_b  # the raw rewards
    dv = hp.v_loss_c * err * inv_b
    m, s = split(cur)
    a = np.asarray(actions, F64)
    iv = np.exp(-2.0 * s)
    cp = hp.policy_loss_c * pg[..., None]
    dm = -cp * (a - m) * iv * inv_b
    ds = (cp * (1.0 - (a - m) ** 2 * iv) - hp.entropy_c) * inv_b
    dparams = np.where(valid[..., None], np.concatenate([dm, ds], -1), 0.0)
    klt = kl(beh, cur)
    vs_t = vs[:T]
    diag = np.array([valid.sum(), np.where(valid, lp - lpb, 0.0).sum(), (valid & (ratio > hp.rho_bar)).sum(),
                     (valid & (ratio > hp.c_bar)).sum(), np.where(valid, klt, 0.0).sum(),
                     np.where(valid, vs_t, 0.0).sum(), np.where(valid, vs_t ** 2, 0.0).sum(),
                     np.where(valid, vs_t - v[:T], 0.0).sum()], F64)
    return dict(vs=vs, pg_adv=pg, rho=rho, ratio=ratio, value_fn_loss=vl, policy_loss=pl, policy_entropy=pe,
                batch_mean_reward=rw, scalars=np.array([vl, pl, pe, rw]), dv=dv, dparams=dparams, log_pi=lp,
                entropy=ent, kl=klt, diag=diag,
                total_loss=hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * pe)


def make_inputs(seed, T, B, A, ragged=True, spread=(0.1, 0.3)):
    """Current outputs m ~ N(0, 1), s ~ U(-1.5, 0.5); behaviour outputs perturbed by 0.1-0.3 from them; actions
    sampled from the behaviour Gaussian; float32 like the slabs.  Ragged: lens in [0, T] with some columns empty
    and some full."""
    rng = np.random.default_rng(seed)
    m = rng.standard_normal((T, B, A))
    s = rng.uniform(-1.5, 0.5, (T, B, A))
    d = rng.uniform(*spread, (T, B, 2 * A)) * rng.choice([-1.0, 1.0], (T, B, 2 * A))
    cur = np.concatenate([m, s], -1).astype(np.float32)
    beh = (cur + d).astype(np.float32)
    mb, sb = split(beh)
    act = (mb + np.exp(sb) * rng.standard_normal((T, B, A))).astype(np.float32)
    lens = rng.integers(0, T + 1, B).astype(np.int32) if ragged else np.full(B, T, np.int32)
    if ragged and B >= 3:
        lens[0], lens[1] = 0, T
    rewards = rng.standard_normal((T, B)).astype(np.float32)
    done = (rng.uniform(size=(T, B)) < 0.05).astype(np.uint8)
    t = np.arange(T)[:, None]
    pad = t >= lens[None, :]
    beh[pad], act[pad], rewards[pad], done[pad] = 0.0, 0.0, 0.0, 0  # slab padding; cur is a network output
    v = rng.standard_normal((T + 1, B)).astype(np.float32)
    return dict(cur=cur, beh=beh, actions=act, rewards=rewards, done=done, lens=lens, v=v)


class GaussLearner(orc.BatchedLearner):
    """The oracle learner with the Gaussian policy terms (tests/gaussian_oracle.py)."""

    def forward_backward(self, batch, mode="reference", batch_size=None):
        hp = self.hp
        B_glob = hp.batch_size if batch_size is None else batch_size
        obs = np.asarray(batch["obs"], np.float64)
        Tp1, B, O = obs.shape
        T = Tp1 - 1
        v2, v_pre = orc.mlp_forward(obs, *self.vf)
        z, pi_pre = orc.mlp_forward(obs[:-1], *self.pi)
        out = vtrace_loss(v2[..., 0], z, batch["beh_logits"], batch["actions"], batch["rewards"], batch["done"],
                               batch["lens"], hp, B_glob, mode)
        out["g_policy"] = list(orc.mlp_backward(obs[:-1].reshape(T * B, O), pi_pre.reshape(T * B, -1), self.pi[2],
                                                out["dparams"].reshape(T * B, -1)))
        out["g_value"] = list(orc.mlp_backward(obs.reshape(Tp1 * B, O), v_pre.reshape(Tp1 * B, -1), self.vf[2],
                                               out["dv"].reshape(Tp1 * B, 1)))
        return out
