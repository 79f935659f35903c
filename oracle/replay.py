"""TEST INFRASTRUCTURE - numpy restatement of the replay batch composition (impala_batch_compose).

The reference learner has no experience replay; what a replayed batch must be is defined by the sampling
rule alone, so this is the whole reference: copy columns.
"""
from __future__ import annotations

import numpy as np

FIELDS = ("obs", "beh_logits", "actions", "rewards", "done", "lens")


def compose_batch(history: dict, plan) -> dict:
    """The B-column batch of one update.  history: store slot -> the fresh batch kept in it (dicts of the six
    batch arrays, Bf columns each).  plan: (B, 2) of (slot, column); column j of the result is that column of
    that batch, a negative slot the empty trajectory (zeros, lens 0)."""
    plan = np.asarray(plan)
    any_batch = next(iter(history.values()))
    out = {}
    for name in FIELDS:
        a = np.asarray(any_batch[name])
        col = np.zeros(len(plan), a.dtype) if name == "lens" else \
            np.zeros((a.shape[0], len(plan)) + a.shape[2:], a.dtype)
        for slot in np.unique(plan[:, 0]):
            if slot < 0:
                continue
            src, js = np.asarray(history[int(slot)][name]), np.flatnonzero(plan[:, 0] == slot)
            if name == "lens":
                col[js] = src[plan[js, 1]]
            else:
                col[:, js] = src[:, plan[js, 1]]
        out[name] = col
    return out
