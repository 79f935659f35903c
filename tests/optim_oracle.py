"""TEST INFRASTRUCTURE - float64 restatement of the optimizers the learner offers beyond the reference's Adam.

`oracle.impala_oracle` states the reference's update (Adam at 0.95 * lr, learner.py:39-42).  This module adds,
on top of it and in the same numpy style:

  * `Adam(params, lr, lr_lambda)`: torch.optim.Adam (betas (0.9, 0.999), eps 1e-8) under
    LambdaLR(lr_lambda) - step n uses lr * lr_lambda(n - 1); lr_lambda=None is the reference's 0.95;
  * `RMSprop(params, lr, alpha, eps, momentum, lr_lambda)`: torch.optim.RMSprop (not centered, no weight
    decay; eps outside the square root) under the same schedule;
  * `BatchedLearner(params, hp, optimizer, optimizer_kwargs, lr_lambda)`: the oracle's learner with either
    optimizer; the default arguments build the reference's Adam unchanged.
"""
from __future__ import annotations

import numpy as np

from oracle import impala_oracle as orc


def _reference_lambda(e):
    return 0.95


class Adam(orc.Adam):
    def __init__(self, params, lr, lr_lambda=None):
        super().__init__(params, lr)
        self.base_lr, self.lr_lambda = lr, lr_lambda or _reference_lambda

    def step(self, params, grads):
        self.lr = self.base_lr * self.lr_lambda(self.t)  # self.t = completed steps = LambdaLR's epoch
        super().step(params, grads)


class RMSprop:
    def __init__(self, params, lr, alpha=0.99, eps=1e-8, momentum=0.0, lr_lambda=None):
        self.base_lr, self.lr_lambda = lr, lr_lambda or _reference_lambda
        self.alpha, self.eps, self.momentum = alpha, eps, momentum
        self.sq = [np.zeros_like(p) for p in params]
        self.buf = [np.zeros_like(p) for p in params]
        self.t = 0

    def step(self, params, grads):
        lr = self.base_lr * self.lr_lambda(self.t)
        self.t += 1
        for p, g, sq, buf in zip(params, grads, self.sq, self.buf):
            sq *= self.alpha
            sq += (1.0 - self.alpha) * g * g
            avg = np.sqrt(sq) + self.eps
            if self.momentum > 0:
                buf *= self.momentum
                buf += g / avg
                p -= lr * buf
            else:
                p -= lr * (g / avg)


class BatchedLearner(orc.BatchedLearner):
    def __init__(self, params, hp, optimizer="adam", optimizer_kwargs=None, lr_lambda=None):
        super().__init__(params, hp)
        kw = dict(optimizer_kwargs or {})
        if optimizer == "rmsprop":
            self.opt = RMSprop(self.pi + self.vf, hp.lr, lr_lambda=lr_lambda, **kw)
        elif optimizer != "adam" or kw:
            raise ValueError(f"optimizer {optimizer!r} with {kw}")
        elif lr_lambda is not None:
            self.opt = Adam(self.pi + self.vf, hp.lr, lr_lambda)
