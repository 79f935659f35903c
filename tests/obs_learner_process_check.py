"""Run the drop-in Learner with wide observations (4 stacked Atari RAM frames) as a forked process behind a RingQueue.

Executed by test_gpu_obs_wide.py in a fresh interpreter (the parent of a forked CUDA process must
never have initialised CUDA).  MlpPolicy(512, 18, 256) and MlpValueFn(512, 256) take 3 updates on
seeded synthetic ragged trajectories; the shared-memory policy the actors would read is compared with
the float64 oracle's parameters after the same 3 updates.
"""
import os
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from conftest import PKEYS  # noqa: E402
from oracle.impala_oracle import BatchedLearner  # noqa: E402
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.learner import Learner  # noqa: E402
from torched_impala_b200.models import MlpPolicy, MlpValueFn  # noqa: E402
from torched_impala_b200.ring import RingQueue  # noqa: E402
from torched_impala_b200.utils import Counter, default_hparams  # noqa: E402

T, B, O, A, H, UPDATES = 20, 64, 512, 18, 256, 3


def main():
    mp.set_start_method("fork", force=True)
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=UPDATES, policy_hidden_dims=H,
                         value_fn_hidden_dims=H)
    init = synth.init_params(21, O, A, H)
    batches = [synth.make_batch(40 + u, T, B, O, A, ragged=True) for u in range(UPDATES)]
    policy, value_fn = MlpPolicy(O, A, H), MlpValueFn(O, H)
    policy.load_state_dict({k: torch.from_numpy(init["policy"][k]).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.from_numpy(init["value_fn"][k]).double() for k in PKEYS})
    policy.share_memory()
    q = RingQueue(T, B, O, A, slabs=2)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, timeout=60)

    def feed():  # stands in for actor processes
        for b in batches:
            for tr in synth.to_trajectories(b):
                q.put(tr, timeout=60)

    lrn.start()
    t = threading.Thread(target=feed, daemon=True)
    t.start()
    ok = lrn.completion.wait(timeout=180)
    lrn.join()
    t.join(timeout=5)
    q.close()
    assert ok, "learner never signalled completion"
    assert lrn.p.exitcode == 0, f"learner exit code {lrn.p.exitcode}"
    assert counter.value == UPDATES, counter.value
    ref = BatchedLearner(init, hp)
    for b in batches:
        ref.update(b)
    want = ref.state()["policy"]
    worst = max(float(np.abs(policy.state_dict()[k].numpy() - want[k]).max()) for k in PKEYS)
    assert worst < 5e-5, worst
    assert not np.allclose(policy.state_dict()[PKEYS[0]].numpy(), init["policy"][PKEYS[0]])
    print(f"OBS_LEARNER_OK updates={counter.value} max|dW|={worst:.2e}")


if __name__ == "__main__":
    main()
