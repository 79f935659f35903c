"""Optimizer choice and learning-rate schedule of the learner, checked and tabulated on the host.

The update runs inside the step's captured CUDA graph (and, with N > 1 GPUs, inside the consumer of the
peer-memory exchange), so a per-update learning rate cannot be a launch argument: the engine keeps a float32
table in device memory and impala_clip_optim reads entry min(n - 1, len - 1) for update n, n the step counter
the kernel keeps.  That is torch's LambdaLR: update n uses hp.lr * lr_lambda(n - 1).

Nothing here touches a device, so the checks can be tested anywhere.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from . import _cabi

# torch.optim.RMSprop's keyword names and defaults (centered and weight_decay only at their defaults)
RMSPROP_DEFAULTS = {"alpha": 0.99, "eps": 1e-8, "momentum": 0.0}
_RMSPROP_OFF = {"centered": False, "weight_decay": 0.0}  # accepted at torch's default only
# the reference's Adam and LambdaLR (learner.py:39-42)
ADAM_BETAS, ADAM_EPS, REFERENCE_LR_FACTOR = (0.9, 0.999), 1e-8, 0.95


@dataclass(frozen=True, eq=False)
class OptimConfig:
    """rule: "adam" | "rmsprop"; h0, h1, eps: the kernel's hyperparameters (Adam: beta1, beta2; RMSprop:
    alpha, momentum); lr_table: float32 rates of updates 1, 2, ... (the last one repeats), None for the
    reference's Adam at a constant 0.95 * hp.lr passed as a launch argument (impala_clip_adam)."""
    rule: str
    h0: float
    h1: float
    eps: float
    lr_table: np.ndarray | None
    lr_scalar: float  # the launch argument when lr_table is None

    @property
    def rule_code(self) -> int:
        return _cabi.OPT_RULES[self.rule]

    @property
    def is_default(self) -> bool:
        return self.lr_table is None

    def lr_of(self, n: int) -> float:
        """The learning rate update n (1-based) uses, as the kernel reads it (float32)."""
        if n < 1:
            raise ValueError(f"updates are numbered from 1, got {n}")
        if self.lr_table is None:
            return float(np.float32(self.lr_scalar))
        return float(self.lr_table[min(n, len(self.lr_table)) - 1])


def _finite_number(name: str, value) -> float:
    try:
        x = float(value)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a number, got {value!r}") from None
    if not math.isfinite(x):
        raise ValueError(f"{name} must be finite, got {value!r}")
    return x


def _check_table(table, source: str) -> np.ndarray:
    t64 = np.asarray(table, dtype=np.float64).reshape(-1)
    if t64.size < 1:
        raise ValueError(f"{source}: the learning-rate table is empty")
    bad = np.flatnonzero(~np.isfinite(t64) | (t64 < 0))
    if bad.size:
        e = int(bad[0])
        raise ValueError(f"{source}: the learning rate of epoch e={e} is {t64[e]!r}; it must be finite and >= 0")
    with np.errstate(over="ignore"):
        t32 = t64.astype(np.float32)
    bad = np.flatnonzero(~np.isfinite(t32))
    if bad.size:
        e = int(bad[0])
        raise ValueError(f"{source}: the learning rate of epoch e={e} ({t64[e]!r}) overflows float32")
    return t32


def tabulate_lr(lr: float, lr_lambda, n: int) -> np.ndarray:
    """float32(lr * lr_lambda(e)) for e in [0, n), computed in float64; a non-finite or negative value raises
    ValueError naming e."""
    if not callable(lr_lambda):
        raise ValueError(f"lr_lambda must be callable (as for torch.optim.lr_scheduler.LambdaLR), got {lr_lambda!r}")
    out = np.empty(max(1, int(n)), np.float64)
    for e in range(out.size):
        try:
            f = float(lr_lambda(e))
        except (TypeError, ValueError) as exc:
            raise ValueError(f"lr_lambda({e}) did not return a number: {exc}") from None
        out[e] = float(lr) * f
        if not (math.isfinite(out[e]) and out[e] >= 0.0):
            raise ValueError(f"lr_lambda: the learning rate of epoch e={e} is lr * {f!r} = {out[e]!r}; "
                             "it must be finite and >= 0")
    return _check_table(out, "lr_lambda")


def optim_config(hp, optimizer: str = "adam", optimizer_kwargs: dict | None = None, lr_lambda=None,
                 lr_table=None) -> OptimConfig:
    """Check the optimizer arguments of LearnerEngine / Learner and build the learning-rate table.

    optimizer "adam" takes no keyword arguments (betas and eps are the reference's); "rmsprop" takes torch's
    alpha (0.99), eps (1e-8) and momentum (0); centered / weight_decay other than torch's defaults, unknown keys
    and out-of-range values raise ValueError naming them.  lr_lambda (a LambdaLR lambda) is tabulated over
    hp.max_updates epochs; None is the reference's lambda e: 0.95.  lr_table (instead of lr_lambda) is an
    already tabulated schedule, e.g. the one a data-parallel worker rank receives."""
    if optimizer not in _cabi.OPT_RULES:
        raise ValueError(f"optimizer must be one of {sorted(_cabi.OPT_RULES)}, got {optimizer!r}")
    kw = dict(optimizer_kwargs or {})
    if optimizer == "adam":
        if kw:
            raise ValueError(f"optimizer='adam' takes no optimizer_kwargs (its betas {ADAM_BETAS} and eps {ADAM_EPS} "
                             f"are the reference's), got {sorted(kw)}")
        h0, h1, eps = ADAM_BETAS[0], ADAM_BETAS[1], ADAM_EPS
    else:
        unknown = sorted(set(kw) - set(RMSPROP_DEFAULTS) - set(_RMSPROP_OFF))
        if unknown:
            raise ValueError(f"optimizer='rmsprop': unknown optimizer_kwargs {unknown}; "
                             f"it takes {sorted(RMSPROP_DEFAULTS)}")
        for key, off in _RMSPROP_OFF.items():
            if key in kw and kw[key] != off:
                raise ValueError(f"optimizer='rmsprop': {key}={kw[key]!r} is not supported (only {key}={off!r})")
        vals = {k: _finite_number(f"rmsprop {k}", kw.get(k, d)) for k, d in RMSPROP_DEFAULTS.items()}
        if not (0.0 <= vals["alpha"] < 1.0 and np.float32(vals["alpha"]) < 1.0):  # the kernel takes float32
            raise ValueError(f"rmsprop alpha must be in [0, 1), got {vals['alpha']!r}")
        if vals["eps"] < 0.0:
            raise ValueError(f"rmsprop eps must be >= 0, got {vals['eps']!r}")
        if vals["momentum"] < 0.0:
            raise ValueError(f"rmsprop momentum must be >= 0, got {vals['momentum']!r}")
        h0, h1, eps = vals["alpha"], vals["momentum"], vals["eps"]
    lr = _finite_number("hp.lr", hp.lr)
    scalar = REFERENCE_LR_FACTOR * lr  # LambdaLR(lambda e: 0.95): constant factor, learner.py:42
    if lr_lambda is not None and lr_table is not None:
        raise ValueError("pass lr_lambda or lr_table, not both")
    if lr_table is not None:
        table = _check_table(lr_table, "lr_table")
    elif lr_lambda is not None:
        table = tabulate_lr(lr, lr_lambda, int(hp.max_updates))
    elif optimizer != "adam":
        table = _check_table([scalar], "the reference's schedule")
    else:
        table = None
    return OptimConfig(optimizer, float(h0), float(h1), float(eps), table, scalar)


POPART_BETA = 3e-4  # step size of the PopArt statistics (van Hasselt et al. 2016)


def check_popart_args(popart, popart_beta) -> float:
    """Check LearnerEngine / Learner's PopArt switch and step size; returns beta.  The kernel takes beta as a
    float32 in (0, 1]; a value that rounds outside raises ValueError."""
    if not isinstance(popart, (bool, np.bool_)):
        raise ValueError(f"popart must be True or False, got {popart!r}")
    beta = _finite_number("popart_beta", popart_beta)
    if not (0.0 < np.float32(beta) <= 1.0):
        raise ValueError(f"popart_beta must be in (0, 1], got {popart_beta!r}")
    return beta
