"""TEST INFRASTRUCTURE - float64 restatement of one learner update of a shared-torso actor-critic.

One network W1 (H, O), b1, W2 (N + 1, H), b2 (N + 1) on all (T+1) B observation rows:
  1. out = mlp(obs) on the (T+1) B rows;
  2. the policy outputs are columns [0, N) of the first T B rows, the values column N of all rows;
  3. V-trace and the losses of the selected kind (categorical or Gaussian, PopArt, reward clipping) give dlogits
     (T, B, N) and dv (T+1, B); the network's output gradient is dz = [dlogits padded with a zero time step | dv];
  4. ONE clip norm over the whole network (clip_grad_norm_ of its four tensors);
  5. the update rule (Adam at 0.95 lr, as oracle/impala_oracle.py), then the PopArt statistics and the rescale of
     the value head (row N of W2, b2[N]).

Parameters are held as the engine holds them: the value head normalized under PopArt.  views() gives the
reference-format policy / value_fn state dicts the engine's state() returns (value head folded under PopArt).
"""
from __future__ import annotations

import numpy as np

import gaussian_oracle as gorc
import popart_oracle as porc
import reward_clip_oracle as rorc
from oracle import impala_oracle as orc

F64 = np.float64
PKEYS = orc.PKEYS


def join(policy: dict, value_fn: dict) -> list:
    """[W1, b1, W2, b2] of the shared network from a policy state dict (torso and policy head) and a value_fn
    state dict (value head; its first layer is ignored, as LearnerEngine.load_state does)."""
    p = [np.asarray(policy[k], F64) for k in PKEYS]
    v = [np.asarray(value_fn[k], F64) for k in PKEYS]
    return [p[0].copy(), p[1].copy(), np.concatenate([p[2], v[2]], 0), np.concatenate([p[3], v[3]], 0)]


def views(net: list, mu: float = 0.0, sigma: float = 1.0) -> dict:
    """Reference-format state dicts of the shared network: the policy view (W1, b1, W2[:N], b2[:N]) and the
    value view (W1, b1, W2[N:], b2[N:]), the value head folded into reward units by (mu, sigma)."""
    w1, b1, w2, b2 = net
    return {"policy": dict(zip(PKEYS, (w1.copy(), b1.copy(), w2[:-1].copy(), b2[:-1].copy()))),
            "value_fn": dict(zip(PKEYS, (w1.copy(), b1.copy(), w2[-1:] * sigma, b2[-1:] * sigma + mu)))}


def heads_loss(out, batch, hp, batch_size, mode="reference", gaussian=False, reward_clip=None, popart=None):
    """V-trace and the losses on the split outputs out (T+1, B, N+1).  popart = (mu, sigma) or None.  Returns the
    oracle dict of the selected kind with `dlogits` (T, B, N), `dv` (T+1, B) and, under PopArt, the statistics'
    inputs n, s1, s2."""
    v, z = out[..., -1], out[:-1, :, :-1]
    b = batch
    if gaussian:
        r = gorc.vtrace_loss(v, z, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], hp, batch_size,
                             mode, reward_clip, popart)
        r["dlogits"] = r["dparams"]
        r.update(n=float(r["diag"][0]), s1=float(r["diag"][5]), s2=float(r["diag"][6]))
        return r
    if popart is not None:
        rb = b if reward_clip is None else dict(b, rewards=rorc.clip_rewards(b["rewards"], reward_clip))
        r = porc.vtrace_popart(v, popart[0], popart[1], z, rb, hp, batch_size, mode)
        T = z.shape[0]
        valid = np.arange(T)[:, None] < b["lens"][None, :]
        r["batch_mean_reward"] = float(np.where(valid, np.asarray(b["rewards"], F64), 0.0).sum() / batch_size)
        return r
    if reward_clip is not None:
        return rorc.vtrace_loss(v, z, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], hp,
                                batch_size, reward_clip, mode)
    vs, pg, rho = orc.vtrace(v, z, b["beh_logits"], b["actions"], b["rewards"], b["done"], b["lens"], hp.gamma,
                             hp.rho_bar, hp.c_bar, mode)
    r = orc.losses(v, vs, z, b["actions"], pg, b["lens"], hp.v_loss_c, hp.policy_loss_c, hp.entropy_c, batch_size)
    T = z.shape[0]
    valid = np.arange(T)[:, None] < b["lens"][None, :]
    r.update(vs=vs, pg_adv=pg, rho=rho,
             batch_mean_reward=float(np.where(valid, np.asarray(b["rewards"], F64), 0.0).sum() / batch_size))
    return r


class SharedLearner:
    """One shared network trained by the learner update above.  params = {"policy", "value_fn"} state dicts (the
    value head normalized under PopArt, as LearnerEngine holds it after load_state at mu 0, nu 1)."""

    def __init__(self, params, hp, gaussian=False, reward_clip=None, popart=False, beta=3e-4, mu=0.0, nu=1.0):
        self.hp, self.gaussian, self.reward_clip, self.popart = hp, gaussian, reward_clip, popart
        self.net = join(params["policy"], params["value_fn"])
        self.opt = orc.Adam(self.net, hp.lr)
        self.beta, self.mu, self.nu = float(beta), float(mu), float(nu)
        self.sigma = porc.sigma_of(self.mu, self.nu)

    def forward_backward(self, batch, mode="reference", batch_size=None):
        hp = self.hp
        B_glob = hp.batch_size if batch_size is None else batch_size
        obs = np.asarray(batch["obs"], F64)
        Tp1, B, O = obs.shape
        out, pre = orc.mlp_forward(obs, *self.net)
        r = heads_loss(out, batch, hp, B_glob, mode, self.gaussian, self.reward_clip,
                       (self.mu, self.sigma) if self.popart else None)
        dz = np.concatenate([np.concatenate([r["dlogits"], np.zeros((1,) + r["dlogits"].shape[1:])], 0),
                             np.asarray(r["dv"], F64)[..., None]], -1)
        r["grad"] = list(orc.mlp_backward(obs.reshape(Tp1 * B, O), pre.reshape(Tp1 * B, -1), self.net[2],
                                          dz.reshape(Tp1 * B, -1)))
        r["out"] = out
        return r

    def apply(self, grad):
        """One clip norm over the whole network, then the update rule."""
        c, norm = orc.clip_coef(grad, self.hp.max_norm)
        self.opt.step(self.net, [g * c for g in grad])
        return dict(norm_policy=norm, norm_value=0.0)

    def popart_step(self, n, s1, s2):
        mu1, nu1, sg1 = porc.stats_update(self.mu, self.nu, n, s1, s2, self.beta)
        self.net[2][-1] *= self.sigma / sg1
        self.net[3][-1] = (self.sigma * self.net[3][-1] + self.mu - mu1) / sg1
        self.mu, self.nu, self.sigma = mu1, nu1, sg1

    def update(self, batch, mode="reference"):
        r = self.forward_backward(batch, mode)
        r.update(self.apply(r["grad"]))
        if self.popart:
            self.popart_step(r["n"], r["s1"], r["s2"])
        return r

    def views(self):
        return views(self.net, self.mu, self.sigma) if self.popart else views(self.net)
