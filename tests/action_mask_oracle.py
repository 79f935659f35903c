"""TEST INFRASTRUCTURE - float64 numpy statement of impala_vtrace_loss_mask (invalid-action masking).

A categorical policy is one head of N outputs; a multi-discrete one K heads (tests/multi_discrete_oracle.py).  legal
(T, B, N) bool says which outputs are legal; a head with no legal entry is all-legal.  pi and mu are the softmaxes
within each head renormalised over its legal entries, every illegal entry is -inf in log p and 0 in p, and
    log pi(a), the ratio, V-trace, vs, pg_adv and the losses as the multi-discrete oracle,
    H_k = -sum_{j in k legal} p_j log p_j,  KL(mu||pi) = sum over the legal entries,
    dz_j = the multi-discrete formula at legal j, exactly 0 at illegal j.
The logit values at illegal entries never enter: they are replaced by -inf before anything else.
"""
from __future__ import annotations

import numpy as np

import multi_discrete_oracle as morc
import reward_clip_oracle as rorc
from gaussian_oracle import vtrace_from_ratio
from oracle import impala_oracle as orc
from torched_impala_b200 import synth

F64 = np.float64
starts = morc.starts


def normalise(legal, heads):
    """legal with every head that has no legal entry made all-legal."""
    legal = np.array(legal, bool)
    for s, n in zip(starts(heads), heads):
        h = legal[..., s:s + n]
        h |= ~h.any(-1, keepdims=True)
    return legal


def head_log_softmax(z, legal, heads):
    """log p per output (..., N) within each head over its legal entries; -inf at the illegal ones."""
    z = np.where(legal, np.asarray(z, F64), -np.inf)
    out = []
    for s, n in zip(starts(heads), heads):
        h = z[..., s:s + n]
        m = h.max(-1, keepdims=True)
        out.append(h - m - np.log(np.exp(h - m).sum(-1, keepdims=True)))
    return np.concatenate(out, -1)


def vtrace_loss(v, cur, beh, actions, legal, rewards, done, lens, hp, batch_size, heads, mode="reference",
                reward_clip=None, popart=None):
    """Every output of impala_vtrace_loss_mask in float64; actions (T, B, K) indices (without the legal word)."""
    heads = tuple(heads)
    T, B = np.asarray(rewards).shape
    lens = np.asarray(lens)
    legal = normalise(legal, heads)
    mu_p, sigma = (0.0, 1.0) if popart is None else (float(popart[0]), float(popart[1]))
    v = sigma * np.asarray(v, F64) + mu_p
    r = np.asarray(rewards, F64) if reward_clip is None else rorc.clip_rewards(rewards, reward_clip)
    valid = np.arange(T)[:, None] < lens[None, :]
    valid_v = np.arange(T + 1)[:, None] <= lens[None, :]
    a = np.asarray(actions).astype(np.int64) + starts(heads)
    lz, lzb = head_log_softmax(cur, legal, heads), head_log_softmax(beh, legal, heads)
    lp = np.take_along_axis(lz, a, -1).sum(-1)
    lpb = np.take_along_axis(lzb, a, -1).sum(-1)
    ratio = np.exp(lp - lpb)
    vs, pg_r, rho = vtrace_from_ratio(v, ratio, r, done, lens, hp.gamma, hp.rho_bar, hp.c_bar, mode)
    pg = pg_r / sigma
    err = np.where(valid_v, v - vs, 0.0) / sigma
    p, pb = np.exp(lz), np.exp(lzb)
    plogp = np.where(legal, p * np.where(legal, lz, 0.0), 0.0)
    hk = np.stack([-plogp[..., s:s + n].sum(-1) for s, n in zip(starts(heads), heads)], -1)
    ent = hk.sum(-1)
    inv_b = 1.0 / batch_size
    vl = 0.5 * (err ** 2).sum() * inv_b
    pl = np.where(valid, -lp * pg, 0.0).sum() * inv_b
    pe = np.where(valid, ent, 0.0).sum() * inv_b
    with np.errstate(invalid="ignore"):
        rw = np.where(valid, np.asarray(rewards, F64), 0.0).sum() * inv_b
    dv = hp.v_loss_c * err * inv_b
    onehot = np.zeros_like(p)
    np.put_along_axis(onehot, a, 1.0, -1)
    h_of = np.repeat(hk, heads, -1)
    with np.errstate(invalid="ignore"):
        dl = inv_b * (hp.policy_loss_c * pg[..., None] * (p - onehot) + hp.entropy_c * p * (np.where(legal, lz, 0.0)
                                                                                              + h_of))
    dlogits = np.where(valid[..., None] & legal, dl, 0.0)
    klt = np.where(legal, pb * (np.where(legal, lzb, 0.0) - np.where(legal, lz, 0.0)), 0.0).sum(-1)
    vs_t = vs[:T]
    diag = np.array([valid.sum(), np.where(valid, lp - lpb, 0.0).sum(), (valid & (ratio > hp.rho_bar)).sum(),
                     (valid & (ratio > hp.c_bar)).sum(), np.where(valid, klt, 0.0).sum(),
                     np.where(valid, vs_t, 0.0).sum(), np.where(valid, vs_t ** 2, 0.0).sum(),
                     np.where(valid, vs_t - v[:T], 0.0).sum()], F64)
    return dict(vs=vs, pg_adv=pg, rho=rho, ratio=ratio, value_fn_loss=vl, policy_loss=pl, policy_entropy=pe,
                batch_mean_reward=rw, scalars=np.array([vl, pl, pe, rw]), dv=dv, dlogits=dlogits, log_pi=lp,
                entropy=ent, kl=klt, diag=diag,
                total_loss=hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * pe)


def make_inputs(seed, T, B, heads, density=0.5, ragged=True, spread=(0.1, 0.3), garbage=True, single=0.1):
    """morc.make_inputs' inputs with legal masks (synth.draw_legal with `density` and a fraction `single` of
    single-legal steps; density 1.0 = every entry legal), the actions
    drawn from the masked behaviour policy and, with `garbage`, +-1e30 / -inf / NaN in the illegal behaviour and
    current logits.  `actions` is (T, B, K + 1) int32 ending in the legal word (padded steps: 0), `idx` the indices."""
    heads = tuple(heads)
    c = morc.make_inputs(seed, T, B, heads, ragged=ragged, spread=spread)
    rng = np.random.default_rng(seed + 104729)
    legal = (np.ones((T, B, sum(heads)), bool) if density >= 1.0 else
             synth.draw_legal(rng, T, B, heads, density, single))
    lb = head_log_softmax(c["beh"], legal, heads)
    idx = np.zeros((T, B, len(heads)), np.int32)
    for k, (s, n) in enumerate(zip(starts(heads), heads)):
        cdf = np.cumsum(np.exp(lb[..., s:s + n]), -1)
        a = np.minimum((1.0 - rng.uniform(size=(T, B, 1)) > cdf).sum(-1), n - 1)
        while True:
            off = ~np.take_along_axis(legal[..., s:s + n], a[..., None], -1)[..., 0]
            if not off.any():
                break
            a = np.where(off, a - 1, a)
        idx[..., k] = a
    pad = np.arange(T)[:, None] >= c["lens"][None, :]
    idx[pad], legal[pad] = 0, False
    if garbage and density < 1.0:
        g = np.array([1e30, -1e30, -np.inf, np.nan], np.float32)
        ill = ~normalise(legal, heads)
        c["cur"] = np.where(ill, g[rng.integers(0, 4, ill.shape)], c["cur"]).astype(np.float32)
        c["beh"] = np.where(ill, g[rng.integers(0, 4, ill.shape)], c["beh"]).astype(np.float32)
    c["idx"], c["legal"] = idx, legal
    c["actions"] = np.concatenate([idx, synth.legal_words(legal)[..., None]], -1).astype(np.int32)
    return c


class MaskLearner(orc.BatchedLearner):
    """The oracle learner with masked policy terms; batch["actions"] ends in the legal word, batch["legal"] holds
    the masks."""

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
        out = vtrace_loss(v2[..., 0], z, batch["beh_logits"], np.asarray(batch["actions"])[..., :-1], batch["legal"],
                          batch["rewards"], batch["done"], batch["lens"], hp, B_glob, self.heads, mode)
        out["g_policy"] = list(orc.mlp_backward(obs[:-1].reshape(T * B, O), pi_pre.reshape(T * B, -1), self.pi[2],
                                                out["dlogits"].reshape(T * B, -1)))
        out["g_value"] = list(orc.mlp_backward(obs.reshape(Tp1 * B, O), v_pre.reshape(Tp1 * B, -1), self.vf[2],
                                               out["dv"].reshape(Tp1 * B, 1)))
        return out
