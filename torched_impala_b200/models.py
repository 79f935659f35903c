"""Host-side (CPU, float64) MLP modules with the reference's state_dict layout.

The learner never runs these on the update path - it only reads their parameters
(`model.0.weight (H,O)`, `model.0.bias`, `model.3.weight (out,H)`, `model.3.bias`;
reference models.py:13-18,41-46) and writes new values back in place so that actor
processes, which do run them on CPU, see the update.  They are defined here so the
package is usable without the reference checkout; the reference's own `MlpPolicy` /
`MlpValueFn` objects work identically with `Learner`.
"""
from __future__ import annotations

import torch
import torch.nn as nn


def _two_layer(obs_dim: int, hidden_dim: int, out_dim: int) -> nn.Sequential:
    # indices 0 and 3 carry the parameters; 1 is the reference's Dropout(p=0.8), 2 the ReLU
    return nn.Sequential(nn.Linear(obs_dim, hidden_dim), nn.Dropout(p=0.8), nn.ReLU(),
                         nn.Linear(hidden_dim, out_dim)).to(torch.float64)


def _masked(z, action_mask):
    """z with -inf at the illegal entries of action_mask (true = legal)."""
    m = torch.as_tensor(action_mask).to(torch.bool)
    if m.shape != z.shape[-1:]:
        raise ValueError(f"action_mask of shape {tuple(m.shape)} for {z.shape[-1]} policy outputs")
    return z.masked_fill(~m, -torch.inf)


class MlpPolicy(nn.Module):
    def __init__(self, obs_dim: int, action_dim: int, hidden_dim: int):
        super().__init__()
        self.model = _two_layer(obs_dim, hidden_dim, action_dim)

    def forward(self, x):
        return self.model(x)

    def select_action(self, obs, deterministic: bool = False, action_mask=None):
        """Actor-side sampling (reference models.py:27-34): returns (action, logits).  action_mask (A,) bool or 0 / 1,
        true meaning legal (Learner(action_mask=True)): the sample (or argmax) is taken over the legal actions only;
        the logits returned are the raw ones - the learner applies the mask it is given with the step."""
        logits = self.forward(obs)
        z = logits if action_mask is None else _masked(logits.detach(), action_mask)
        if deterministic:
            return torch.argmax(z), logits
        return torch.multinomial(torch.softmax(z, dim=-1), num_samples=1), logits


class GaussianMlpPolicy(nn.Module):
    """Diagonal Gaussian policy with a state-dependent log-std (Learner(action_dist="gaussian")): the same
    two-layer MLP with 2 action_dim outputs [mean_0..A-1 | log_std_0..A-1], so the state_dict keys are MlpPolicy's."""

    def __init__(self, obs_dim: int, action_dim: int, hidden_dim: int):
        super().__init__()
        self.action_dim = action_dim
        self.model = _two_layer(obs_dim, hidden_dim, 2 * action_dim)

    def forward(self, x):
        return self.model(x)

    def select_action(self, obs, deterministic: bool = False):
        """Returns (action (A,) float64, params (2A,)): the unsquashed sample mean + exp(log_std) eps (the mean when
        deterministic).  The learner needs the sample itself; clip it to the action space only for env.step."""
        params = self.forward(obs)
        mean, log_std = params[..., :self.action_dim], params[..., self.action_dim:]
        if deterministic:
            return mean.detach().clone(), params
        with torch.no_grad():
            return mean + torch.exp(log_std) * torch.randn_like(mean), params


class MultiDiscreteMlpPolicy(nn.Module):
    """Factorised categorical policy over a MultiDiscrete([n_0, .., n_K-1]) space (Learner(action_dist=
    "multi_discrete", action_heads=...) or LearnerEngine): the same two-layer MLP with N = sum n_k outputs, head k owning
    [s_k, s_k + n_k), so the state_dict keys are MlpPolicy's."""

    def __init__(self, obs_dim: int, action_heads, hidden_dim: int):
        super().__init__()
        self.action_heads = tuple(int(n) for n in action_heads)
        self.model = _two_layer(obs_dim, hidden_dim, sum(self.action_heads))

    def forward(self, x):
        return self.model(x)

    def select_action(self, obs, deterministic: bool = False, action_mask=None):
        """Returns (actions (K,) int64, logits (N,)): one index per head, sampled from the softmax of its slice (the
        per-head argmax when deterministic).  action_mask (N,), true meaning legal: each head samples over its legal
        entries only; the logits returned are the raw ones."""
        logits = self.forward(obs)
        out = []
        with torch.no_grad():
            zm = logits if action_mask is None else _masked(logits, action_mask)
            for z in torch.split(zm, self.action_heads, dim=-1):
                out.append(z.argmax(-1) if deterministic else
                           torch.multinomial(torch.softmax(z, dim=-1).reshape(-1, z.shape[-1]), 1).reshape(z.shape[:-1]))
        return torch.stack(out, -1).to(torch.int64), logits


class MlpValueFn(nn.Module):
    def __init__(self, obs_dim: int, hidden_dim: int):
        super().__init__()
        self.model = _two_layer(obs_dim, hidden_dim, 1)

    def forward(self, observation):
        return self.model(observation)
