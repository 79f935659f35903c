"""TEST INFRASTRUCTURE - float64 numpy statement of the off-policy diagnostics of impala_vtrace_loss_diag.

The reference logs none of these, so there is no golden pin: tests/test_diagnostics_cpu.py checks this
statement against an independent per-trajectory torch.distributions restatement, and the GPU tests
check the kernel against this statement.

A valid step is t < lens[b] (the mask of the losses).  Per valid step, with pi = softmax(cur_logits)
and mu = softmax(beh_logits):
    log_ratio_t = log pi(a_t) - log mu(a_t),  ratio_t = exp(log_ratio_t)
    KL_t        = sum_k mu_k (log mu_k - log pi_k)          KL(mu || pi)
    err_t       = vs_t - v_t
"""
from __future__ import annotations

import numpy as np

F64 = np.float64
SUM_NAMES = ("n", "log_ratio", "n_rho_clipped", "n_c_clipped", "kl", "vs", "vs_sq", "err")


def _log_softmax(z):
    m = z.max(-1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(-1, keepdims=True))


def diagnostics(v, vs, cur_logits, beh_logits, actions, lens, rho_bar, c_bar):
    """The eight float64 sums over the valid steps, in the order of impala_vtrace_loss_diag's `diag`.

    v, vs (T+1, B); logits (T, B, A); actions (T, B); lens (B,)."""
    cur = np.asarray(cur_logits, F64)
    T = cur.shape[0]
    L = np.clip(np.asarray(lens, np.int64), 0, T)
    valid = np.arange(T)[:, None] < L[None, :]
    lp, lq = _log_softmax(cur), _log_softmax(np.asarray(beh_logits, F64))
    a = np.asarray(actions, np.int64)[..., None]
    log_ratio = (np.take_along_axis(lp, a, -1) - np.take_along_axis(lq, a, -1))[..., 0]
    ratio = np.exp(log_ratio)
    kl = (np.exp(lq) * (lq - lp)).sum(-1)
    vs_t = np.asarray(vs, F64)[:T]
    err = vs_t - np.asarray(v, F64)[:T]
    terms = (np.ones_like(ratio), log_ratio, (ratio > rho_bar).astype(F64), (ratio > c_bar).astype(F64), kl,
             vs_t, vs_t * vs_t, err)
    return np.array([np.where(valid, x, 0.0).sum() for x in terms], F64)


def derived(sums, value_fn_loss, batch_size):
    """The logged values from the (all-rank) sums.  sum err^2 = 2 batch_size value_fn_loss (the baseline
    loss 0.5 sum_{t <= lens} (v - vs)^2 / batch_size has a zero t = lens term)."""
    n, s_lr, n_rho, n_c, s_kl, s_vs, s_vs2, s_err = (float(x) for x in sums)
    nan = float("nan")
    if n <= 0:
        return dict(valid_steps=n, log_ratio_mean=nan, rho_clip_fraction=nan, c_clip_fraction=nan,
                    kl_behaviour_current=nan, value_explained_variance=nan)
    var_vs = s_vs2 / n - (s_vs / n) ** 2
    var_err = 2.0 * batch_size * value_fn_loss / n - (s_err / n) ** 2
    ev = 1.0 - var_err / var_vs if n >= 2 and var_vs > 0.0 else nan
    return dict(valid_steps=n, log_ratio_mean=s_lr / n, rho_clip_fraction=n_rho / n, c_clip_fraction=n_c / n,
                kl_behaviour_current=s_kl / n, value_explained_variance=ev)
