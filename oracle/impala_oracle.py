"""TEST INFRASTRUCTURE - float64 numpy restatement of the learner update, (T, B) batched.

Every function states the reference lines it restates.  The reference works on
one variable-length trajectory at a time; here the same arithmetic is applied to
all B columns of a zero-padded time-major batch with `lens[b]` valid steps, so
per-element outputs (v_s, pg advantage, dL/dlogits, dL/dv, gradients) can be
compared with the CUDA path.  Quirks of the reference are reproduced on purpose
(SURVEY.md section 0.2):

  * `learner.py:126`  delta uses `v[:1]` (V(x_0) for every step) and the python
    double `gamma`, not `disc`;
  * `learner.py:130`  the accumulator recurrence subtracts `v[i+1]` a second time;
  * `learner.py:109`  `disc = gamma * ~done` is a float32 tensor (python float x bool).
"""
from __future__ import annotations

import numpy as np

F64 = np.float64


# --------------------------------------------------------------------------- MLPs
def mlp_forward(x, w1, b1, w2, b2):
    """models.py:12-25 / :40-52 in eval mode: Linear -> (Dropout = identity) -> ReLU -> Linear.

    x (..., O) -> returns (out (..., N2), pre-activation (..., H)).
    """
    pre = x @ w1.T + b1
    hid = np.maximum(pre, 0.0)
    return hid @ w2.T + b2, pre


def mlp_backward(x, pre, w2, dout):
    """Autograd of the above w.r.t. the four parameter tensors (learner.py:174-175).

    x (M, O), pre (M, H), dout (M, N2).  Observations need no gradient.
    """
    hid = np.maximum(pre, 0.0)
    dw2 = dout.T @ hid
    db2 = dout.sum(0)
    dpre = (dout @ w2) * (pre > 0.0)
    dw1 = dpre.T @ x
    db1 = dpre.sum(0)
    return dw1, db1, dw2, db2


# ----------------------------------------------------------------------- log-probs
def log_softmax(z):
    m = z.max(-1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(-1, keepdims=True))


def taken_log_probs(logits, actions):
    """learner.py:298-303 action_log_probs: log_softmax(logits)[a]."""
    lsm = log_softmax(logits)
    return np.take_along_axis(lsm, actions[..., None].astype(np.int64), -1)[..., 0]


# -------------------------------------------------------------------------- V-trace
def vtrace(v, cur_logits, beh_logits, actions, rewards, done, lens, gamma, rho_bar, c_bar,
           mode="reference"):
    """learner.py:116-135 for every column b at once.

    v (T+1, B); logits (T, B, A); actions/rewards/done (T, B); lens (B,).
    Returns vs (T+1, B) [the reference's `vt` after :131], pg_adv (T, B), rho (T, B).
    Padded positions (t >= lens[b] for step tensors, i > lens[b] for vs) are 0.
    mode="paper" is the Espeholt et al. recurrence (not parity-checked against anything).
    """
    v = np.asarray(v, F64)
    T, B = rewards.shape
    t_idx = np.arange(T)[:, None]
    valid = t_idx < lens[None, :]
    lp_cur = taken_log_probs(np.asarray(cur_logits, F64), actions)         # :116
    lp_beh = taken_log_probs(np.asarray(beh_logits, F64), actions)         # :117
    is_ratio = np.exp(lp_cur - lp_beh)                                     # :121-123
    rho = np.where(valid, np.minimum(is_ratio, rho_bar), 0.0)              # :124
    c = np.where(valid, np.minimum(is_ratio, c_bar), 0.0)                  # :125
    # :109  float32 tensor (python float * bool tensor -> default dtype), then promoted
    disc = (np.float32(gamma) * (~done.astype(bool)).astype(np.float32)).astype(F64)
    disc = np.where(valid, disc, 0.0)
    r = np.asarray(rewards, F64)
    acc = np.zeros((T + 1, B), F64)                                        # :127
    if mode == "reference":
        delta = rho * (r + gamma * v[1:] - v[:1])                          # :126 (v[:1] quirk)
        for i in range(T - 1, -1, -1):                                     # :129-130
            acc[i] = delta[i] + disc[i] * c[i] * (acc[i + 1] - v[i + 1])
    elif mode == "paper":
        delta = rho * (r + disc * v[1:] - v[:-1])
        for i in range(T - 1, -1, -1):
            acc[i] = delta[i] + disc[i] * c[i] * acc[i + 1]
    else:
        raise ValueError(mode)
    vs = acc + v                                                           # :131
    pg_adv = rho * (r + disc * vs[1:] - v[:-1])                            # :135
    vs = np.where(np.arange(T + 1)[:, None] <= lens[None, :], vs, 0.0)
    return vs, pg_adv, rho


# --------------------------------------------------------------------------- losses
def losses(v, vs, cur_logits, actions, pg_adv, lens, hp_v_loss_c, hp_policy_loss_c,
           hp_entropy_c, batch_size):
    """learner.py:149-162 + helper functions :306-321, summed over time, mean over batch.

    Returns dict(value_fn_loss, policy_loss, policy_entropy, total_loss) - the four
    numbers the reference logs at :223-240 - and the closed-form gradients of
    total_loss w.r.t. v and the current logits (what autograd produces at :175).
    """
    T, B, A = cur_logits.shape
    z = np.asarray(cur_logits, F64)
    valid = np.arange(T)[:, None] < lens[None, :]
    valid_v = np.arange(T + 1)[:, None] <= lens[None, :]
    lsm = log_softmax(z)
    p = np.exp(lsm)
    adv = np.where(valid_v, v - vs, 0.0)
    vl_b = 0.5 * (adv ** 2).sum(0)                                         # :306-307 via :149
    nll = -np.take_along_axis(lsm, actions[..., None].astype(np.int64), -1)[..., 0]
    pl_b = np.where(valid, nll * pg_adv, 0.0).sum(0)                       # :317-321 via :150-152
    ent_t = -(p * lsm).sum(-1)
    h_b = np.where(valid, ent_t, 0.0).sum(0)                               # :310-314, negated at :153
    value_fn_loss = vl_b.sum() / batch_size                                # :160
    policy_loss = pl_b.sum() / batch_size                                  # :161
    policy_entropy = h_b.sum() / batch_size                                # :162
    total = (hp_v_loss_c * vl_b + hp_policy_loss_c * pl_b - hp_entropy_c * h_b).sum() / batch_size  # :154-159
    # autograd closed form (vs, pg_adv are no_grad, learner.py:120)
    dv = hp_v_loss_c * adv / batch_size
    onehot = np.zeros_like(z)
    np.put_along_axis(onehot, actions[..., None].astype(np.int64), 1.0, -1)
    dz = (hp_policy_loss_c * pg_adv[..., None] * (p - onehot)
          + hp_entropy_c * p * (lsm + ent_t[..., None])) / batch_size
    dz = np.where(valid[..., None], dz, 0.0)
    return dict(value_fn_loss=value_fn_loss, policy_loss=policy_loss,
                policy_entropy=policy_entropy, total_loss=total, dv=dv, dlogits=dz)


# --------------------------------------------------------------------- clip + Adam
def clip_coef(grads, max_norm):
    """torch.nn.utils.clip_grad_norm_ as called at learner.py:176-181 (L2, eps 1e-6, clamp 1).

    A NaN norm gives a NaN coefficient, as torch.clamp propagates it (Python's min(1.0, nan) is 1.0)."""
    total = np.sqrt(sum(float((g.astype(F64) ** 2).sum()) for g in grads))
    return (total if np.isnan(total) else min(1.0, max_norm / (total + 1e-6))), total


class Adam:
    """torch.optim.Adam defaults as constructed at learner.py:39-42.

    betas (0.9, 0.999), eps 1e-8, no weight decay; LambdaLR(lambda e: 0.95) makes the
    effective learning rate the constant 0.95 * hp.lr from the very first step.
    """

    def __init__(self, params, lr):
        self.lr = 0.95 * lr
        self.m = [np.zeros_like(p) for p in params]
        self.v = [np.zeros_like(p) for p in params]
        self.t = 0

    def step(self, params, grads):
        self.t += 1
        b1, b2, eps = 0.9, 0.999, 1e-8
        bc1 = 1.0 - b1 ** self.t
        bc2 = 1.0 - b2 ** self.t
        for p, g, m, v in zip(params, grads, self.m, self.v):
            m *= b1
            m += (1.0 - b1) * g
            v *= b2
            v += (1.0 - b2) * g * g
            p -= (self.lr / bc1) * m / (np.sqrt(v) / np.sqrt(bc2) + eps)


PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")


class BatchedLearner:
    """One full reference update (learner.py:75-183) on a dense padded batch."""

    def __init__(self, params, hp):
        self.hp = hp
        self.pi = [np.array(params["policy"][k], F64) for k in PKEYS]
        self.vf = [np.array(params["value_fn"][k], F64) for k in PKEYS]
        self.opt = Adam(self.pi + self.vf, hp.lr)

    def forward_backward(self, batch, mode="reference", batch_size=None):
        hp = self.hp
        B_glob = hp.batch_size if batch_size is None else batch_size
        obs = np.asarray(batch["obs"], F64)
        Tp1, B, O = obs.shape
        T = Tp1 - 1
        lens = batch["lens"]
        v2, v_pre = mlp_forward(obs, *self.vf)                             # :112
        v = v2[..., 0]
        logits, pi_pre = mlp_forward(obs[:-1], *self.pi)                   # :113
        vs, pg_adv, rho = vtrace(v, logits, batch["beh_logits"], batch["actions"],
                                 batch["rewards"], batch["done"], lens, hp.gamma, hp.rho_bar,
                                 hp.c_bar, mode)
        out = losses(v, vs, logits, batch["actions"], pg_adv, lens, hp.v_loss_c,
                     hp.policy_loss_c, hp.entropy_c, B_glob)
        A = logits.shape[-1]
        g_pi = mlp_backward(obs[:-1].reshape(T * B, O), pi_pre.reshape(T * B, -1), self.pi[2],
                            out["dlogits"].reshape(T * B, A))
        g_vf = mlp_backward(obs.reshape(Tp1 * B, O), v_pre.reshape(Tp1 * B, -1), self.vf[2],
                            out["dv"].reshape(Tp1 * B, 1))
        valid = np.arange(T)[:, None] < lens[None, :]
        reward = float(np.where(valid, batch["rewards"].astype(F64), 0.0).sum() / B_glob)  # :108
        out.update(v=v, logits=logits, vs=vs, pg_adv=pg_adv, rho=rho, g_policy=list(g_pi),
                   g_value=list(g_vf), batch_mean_reward=reward)
        return out

    def apply(self, g_policy, g_value):
        """learner.py:176-183: per-group clip, one Adam over both groups."""
        c_pi, n_pi = clip_coef(g_policy, self.hp.max_norm)
        c_vf, n_vf = clip_coef(g_value, self.hp.max_norm)
        grads = [g * c_pi for g in g_policy] + [g * c_vf for g in g_value]
        self.opt.step(self.pi + self.vf, grads)
        return dict(norm_policy=n_pi, norm_value=n_vf)

    def update(self, batch, mode="reference"):
        out = self.forward_backward(batch, mode)
        out.update(self.apply(out["g_policy"], out["g_value"]))
        return out

    def state(self):
        return {"policy": dict(zip(PKEYS, (p.copy() for p in self.pi))),
                "value_fn": dict(zip(PKEYS, (p.copy() for p in self.vf)))}
