"""TEST INFRASTRUCTURE - float64 numpy statement of the reward transforms of impala_vtrace_loss_rclip.

The transforms are DeepMind's IMPALA `reward_clipping` modes:
    abs_one          clip(r, -1, 1)
    soft_asymmetric  where(r < 0, 0.3 tanh(r / 5), tanh(r / 5)) * 5
NaN stays NaN (as torch.clamp keeps it); +-inf saturates.  The V-trace targets and losses are the unchanged
oracle's on the transformed rewards; batch_mean_reward is the mean of the RAW rewards over the valid steps.
"""
from __future__ import annotations

import numpy as np

from oracle import impala_oracle as orc

F64 = np.float64
MODES = ("abs_one", "soft_asymmetric")


def clip_rewards(r, mode):
    """The transform f(r) in float64, elementwise."""
    r = np.asarray(r, F64)
    if mode == "abs_one":
        out = np.where(r > 1.0, 1.0, r)
        return np.where(out < -1.0, -1.0, out)
    if mode == "soft_asymmetric":
        t = np.tanh(r / 5.0)
        return np.where(r < 0.0, 0.3 * t, t) * 5.0
    raise ValueError(f"reward_clip must be one of {MODES}, got {mode!r}")


def vtrace_loss(v, cur_logits, beh_logits, actions, rewards, done, lens, hp, batch_size, reward_clip,
                mode="reference"):
    """vs, pg_adv and the losses of oracle/impala_oracle.py on f(rewards), plus batch_mean_reward of the raw
    rewards (sum over t < lens[b], divided by batch_size)."""
    rc = clip_rewards(rewards, reward_clip)
    vs, pg, rho = orc.vtrace(v, cur_logits, beh_logits, actions, rc, done, lens, hp.gamma, hp.rho_bar, hp.c_bar,
                             mode)
    out = orc.losses(np.asarray(v, F64), vs, cur_logits, actions, pg, lens, hp.v_loss_c, hp.policy_loss_c,
                     hp.entropy_c, batch_size)
    T = np.asarray(rewards).shape[0]
    valid = np.arange(T)[:, None] < np.asarray(lens)[None, :]
    with np.errstate(invalid="ignore"):  # +inf and -inf among the raw rewards: NaN, as the kernel's sum
        raw_sum = np.where(valid, np.asarray(rewards, F64), 0.0).sum()
    out.update(vs=vs, pg_adv=pg, rho=rho, batch_mean_reward=float(raw_sum / batch_size))
    return out
