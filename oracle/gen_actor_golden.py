"""TEST INFRASTRUCTURE - record trajectories of the REAL reference actor as tests/golden/actor/*.npz.

Run where the unmodified reference can be imported (oracle/refload.py):

    python -m oracle.gen_actor_golden

The reference's own actor.py (`Actor._act`) plays the in-repo old-API CartPole with a seeded
MlpPolicy(4, 2, 16) until it has queued B = 6 trajectories of at most T = 20 steps.  Every field
of every trajectory (obs, a, r, d, logits - lists of tensors, utils.py:48-73) is stored
concatenated over the trajectories, with the per-trajectory lengths, so that
tests/test_host_boundary.py can replay them through the packer without the reference present.
"""
from __future__ import annotations

import os
import queue
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refload  # noqa: E402
from oracle.cartpole_env import make as make_cartpole  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "actor", "reference_actor_trajectories.npz")
B, T = 6, 20
FIELDS = ("obs", "a", "r", "d", "logits")


def main() -> None:
    import torch

    refload.load(env_factory=make_cartpole)
    import actor as ref_actor
    import models as ref_models
    import utils as ref_utils

    hp = ref_utils.Hyperparameters(**default_hparams(batch_size=B, max_timesteps=T, verbose=0)._asdict())
    torch.manual_seed(0)
    shared = ref_models.MlpPolicy(4, 2, 16)

    class FakeLearner:  # what actor.py touches: .completion.is_set() and .policy_weights
        class completion:
            calls = 0

            @classmethod
            def is_set(cls):
                cls.calls += 1
                return cls.calls > B

        policy_weights = shared.state_dict()

    q = queue.Queue()
    ref_actor.Actor(1, hp, ref_models.MlpPolicy(4, 2, 16), FakeLearner, q, ref_utils.Counter(0))._act()
    trajs = [q.get_nowait() for _ in range(B)]
    arrays = {"T": np.int64(T), "steps": np.array([len(t.r) for t in trajs], dtype=np.int64)}
    for f in FIELDS:
        arrays[f] = np.concatenate([torch.stack(getattr(t, f)).numpy() for t in trajs])
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **arrays)
    print(f"[gen_actor_golden] {OUT}: steps {arrays['steps'].tolist()}")


if __name__ == "__main__":
    main()
