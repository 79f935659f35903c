"""TEST INFRASTRUCTURE - float64 restatement of the learner update with PopArt value normalization
(van Hasselt et al. 2016, single task), on top of tests/optim_oracle.py.

The value net outputs the normalized value n; the value in reward units is v = sigma n + mu.  Update k:
  1. V-trace and the losses on v (vs in reward units); value loss 0.5 sum ((v - vs) / sigma)^2, policy
     gradient and policy loss on pg_adv / sigma;
  2. clip + optimizer step on that gradient;
  3. mu' = (1 - beta) mu + beta S1 / n, nu' = (1 - beta) nu + beta S2 / n over the valid steps t < lens[b],
     sigma' = clamp(sqrt(max(nu' - mu'^2, 0)), 1e-4, 1e6) (n = 0: unchanged);
  4. W2 <- W2 sigma / sigma', b2 <- (sigma b2 + mu - mu') / sigma'.
"""
from __future__ import annotations

import numpy as np

import optim_oracle
from oracle import impala_oracle as orc

F64 = np.float64


def sigma_of(mu, nu):
    return min(max(np.sqrt(max(nu - mu * mu, 0.0)), 1e-4), 1e6)


def fold(vf, mu, sigma):
    """Normalized value head -> reward units (W2 sigma, b2 sigma + mu); vf = [W1, b1, W2, b2]."""
    return [vf[0], vf[1], vf[2] * sigma, vf[3] * sigma + mu]


def unfold(vf, mu, sigma):
    return [vf[0], vf[1], vf[2] / sigma, (vf[3] - mu) / sigma]


def vtrace_popart(n, mu, sigma, logits, batch, hp, batch_size, mode="reference"):
    """Outputs of impala_vtrace_loss_popart on the normalized values n (T+1, B)."""
    v = sigma * np.asarray(n, F64) + mu
    vs, pg, rho = orc.vtrace(v, logits, batch["beh_logits"], batch["actions"], batch["rewards"], batch["done"],
                             batch["lens"], hp.gamma, hp.rho_bar, hp.c_bar, mode)
    out = orc.losses(v / sigma, vs / sigma, logits, batch["actions"], pg / sigma, batch["lens"], hp.v_loss_c,
                     hp.policy_loss_c, hp.entropy_c, batch_size)
    T = pg.shape[0]
    valid = np.arange(T)[:, None] < batch["lens"][None, :]
    out.update(v=v, vs=vs, pg_adv=pg / sigma, rho=rho, n=float(valid.sum()), s1=float(vs[:T][valid].sum()),
               s2=float((vs[:T][valid] ** 2).sum()))
    return out


def stats_update(mu, nu, n, s1, s2, beta):
    if n <= 0:
        return mu, nu, sigma_of(mu, nu)
    mu1 = (1.0 - beta) * mu + beta * s1 / n
    nu1 = (1.0 - beta) * nu + beta * s2 / n
    return mu1, nu1, sigma_of(mu1, nu1)


class BatchedLearner(optim_oracle.BatchedLearner):
    """optim_oracle.BatchedLearner with PopArt; `params` holds the NORMALIZED value function."""

    def __init__(self, params, hp, optimizer="adam", optimizer_kwargs=None, lr_lambda=None, beta=3e-4, mu=0.0,
                 nu=1.0):
        super().__init__(params, hp, optimizer, optimizer_kwargs, lr_lambda)
        self.beta, self.mu, self.nu = float(beta), float(mu), float(nu)
        self.sigma = sigma_of(self.mu, self.nu)

    def forward_backward(self, batch, mode="reference", batch_size=None):
        hp = self.hp
        B_glob = hp.batch_size if batch_size is None else batch_size
        obs = np.asarray(batch["obs"], F64)
        Tp1, B, O = obs.shape
        T = Tp1 - 1
        n2, v_pre = orc.mlp_forward(obs, *self.vf)
        logits, pi_pre = orc.mlp_forward(obs[:-1], *self.pi)
        out = vtrace_popart(n2[..., 0], self.mu, self.sigma, logits, batch, hp, B_glob, mode)
        A = logits.shape[-1]
        out["g_policy"] = list(orc.mlp_backward(obs[:-1].reshape(T * B, O), pi_pre.reshape(T * B, -1), self.pi[2],
                                                out["dlogits"].reshape(T * B, A)))
        out["g_value"] = list(orc.mlp_backward(obs.reshape(Tp1 * B, O), v_pre.reshape(Tp1 * B, -1), self.vf[2],
                                               out["dv"].reshape(Tp1 * B, 1)))
        out["logits"] = logits
        return out

    def popart_step(self, n, s1, s2):
        mu1, nu1, sg1 = stats_update(self.mu, self.nu, n, s1, s2, self.beta)
        self.vf[2] *= self.sigma / sg1
        self.vf[3][...] = (self.sigma * self.vf[3] + self.mu - mu1) / sg1
        self.mu, self.nu, self.sigma = mu1, nu1, sg1

    def update(self, batch, mode="reference"):
        out = self.forward_backward(batch, mode)
        out.update(self.apply(out["g_policy"], out["g_value"]))
        self.popart_step(out["n"], out["s1"], out["s2"])
        return out
