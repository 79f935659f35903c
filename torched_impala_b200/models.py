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


class MlpPolicy(nn.Module):
    def __init__(self, obs_dim: int, action_dim: int, hidden_dim: int):
        super().__init__()
        self.model = _two_layer(obs_dim, hidden_dim, action_dim)

    def forward(self, x):
        return self.model(x)

    def select_action(self, obs, deterministic: bool = False):
        """Actor-side sampling (reference models.py:27-34): returns (action, logits)."""
        logits = self.forward(obs)
        if deterministic:
            return torch.argmax(logits), logits
        return torch.multinomial(torch.softmax(logits, dim=-1), num_samples=1), logits


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


class MlpValueFn(nn.Module):
    def __init__(self, obs_dim: int, hidden_dim: int):
        super().__init__()
        self.model = _two_layer(obs_dim, hidden_dim, 1)

    def forward(self, observation):
        return self.model(observation)
