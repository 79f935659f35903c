"""TEST INFRASTRUCTURE - per-trajectory float64 torch port of the reference update.

This is the second restatement: it keeps the reference's *execution structure*
(python loop over trajectories, python loop over time for the V-trace recurrence,
torch autograd, `clip_grad_norm_`, `torch.optim.Adam` + `LambdaLR`) so that, timed
on host cores, it costs what the reference learner costs
(`learner.py:75-183`).  It is what `bench.py` times as the CPU
baseline (`cpu_baseline.kind = "port"`) on machines where the reference checkout is not
present, and `tests/test_oracle_golden.py` pins it against outputs of the real
reference.  Dropout (models.py:15,44) is the identity here: the parity setting is
`.eval()` for both nets (SURVEY.md section 0.4).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

F64 = torch.float64
PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")


def _mlp(x, p):
    """models.py:12-25 / :40-52, eval mode."""
    return F.linear(torch.relu(F.linear(x, p[0], p[1])), p[2], p[3])


def _taken_lp(logits, actions):
    """learner.py:298-303."""
    return torch.log_softmax(logits, -1).gather(-1, actions.reshape(-1, 1))


class CpuLearnerPort:
    def __init__(self, params, hp, threads: int | None = None):
        if threads is not None:
            torch.set_num_threads(threads)
        self.hp = hp
        self.pi = [torch.tensor(params["policy"][k], dtype=F64, requires_grad=True) for k in PKEYS]
        self.vf = [torch.tensor(params["value_fn"][k], dtype=F64, requires_grad=True) for k in PKEYS]
        self.opt = torch.optim.Adam(self.pi + self.vf, lr=hp.lr)                      # :39-41
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda e: 0.95)       # :42
        self.last = {}

    def _one_trajectory(self, tr, keep):
        hp = self.hp
        n = len(tr.r)                                                                  # :104
        x = torch.stack(tr.obs)
        a = torch.stack(tr.a)
        rew = torch.stack(tr.r)
        disc = hp.gamma * (~torch.stack(tr.d))                                         # :109 (float32)
        val = _mlp(x, self.vf).squeeze(1)                                              # :112
        z = _mlp(x[:-1], self.pi)                                                      # :113
        lp_now = _taken_lp(z, a)
        lp_beh = _taken_lp(torch.stack(tr.logits), a)
        with torch.no_grad():                                                          # :120-135
            ratio = (lp_now - lp_beh).exp().squeeze(1)
            rho = ratio.clamp(max=hp.rho_bar)
            cc = ratio.clamp(max=hp.c_bar)
            td = rho * (rew + hp.gamma * val[1:] - val[:1])                            # v[:1] quirk
            acc = torch.zeros(n + 1, dtype=F64)
            for i in reversed(range(n)):
                acc[i] = td[i] + disc[i] * cc[i] * (acc[i + 1] - val[i + 1])
            tgt = acc + val
            adv = rho * (rew + disc * tgt[1:] - val[:-1])
        lsm = torch.log_softmax(z, -1)
        vl = 0.5 * ((val - tgt) ** 2).sum()                                            # :149
        pl = (-lsm.gather(-1, a.reshape(-1, 1)).reshape(-1) * adv).sum()              # :150-152
        ent = -(lsm.exp() * lsm).sum()                                                 # :153
        if keep is not None:
            keep.append((tgt.clone(), adv.clone()))
        return vl, pl, ent, rew.sum().item()

    def update(self, trajectories, keep_elements: bool = False):
        """One pass of learner.py:75-183 over `hp.batch_size` trajectories."""
        hp = self.hp
        bs = hp.batch_size
        total = torch.zeros(1, dtype=F64, requires_grad=True)                          # :85
        vl_s = pl_s = ent_s = rew_s = 0.0
        keep = [] if keep_elements else None
        for tr in trajectories:
            vl, pl, ent, rsum = self._one_trajectory(tr, keep)
            tl = hp.v_loss_c * vl + hp.policy_loss_c * pl - hp.entropy_c * ent          # :154-158
            total = total + tl / bs                                                    # :159
            vl_s += vl.item() / bs
            pl_s += pl.item() / bs
            ent_s += ent.item() / bs
            rew_s += rsum / bs
        self.opt.zero_grad()
        total.backward()                                                               # :174-175
        raw = [p.grad.clone() for p in self.pi + self.vf] if keep_elements else None
        torch.nn.utils.clip_grad_norm_(self.pi, hp.max_norm)                           # :176-181
        torch.nn.utils.clip_grad_norm_(self.vf, hp.max_norm)
        self.opt.step()
        self.sched.step()
        self.last = dict(value_fn_loss=vl_s, policy_loss=pl_s, policy_entropy=ent_s,
                         total_loss=total.item(), batch_mean_reward=rew_s, elements=keep,
                         raw_grads=raw)
        return self.last

    def state(self):
        return {"policy": {k: p.detach().numpy().copy() for k, p in zip(PKEYS, self.pi)},
                "value_fn": {k: p.detach().numpy().copy() for k, p in zip(PKEYS, self.vf)}}
