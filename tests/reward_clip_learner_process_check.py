"""Run the drop-in Learner as a forked process behind a RingQueue, with or without reward clipping.

    python tests/reward_clip_learner_process_check.py <log dir> clip|plain <out.npz>

Executed by test_gpu_reward_clip.py in a fresh interpreter (the parent of a forked CUDA process must not have
initialised CUDA).  "clip" feeds raw rewards to Learner(reward_clip="abs_one"); "plain" feeds the same
trajectories with the rewards clipped on the host to a Learner without clipping.  The final weights, the logged
rewards/batch_mean_reward of every update and the raw and clipped batch means go to <out.npz>.
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
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.learner import Learner  # noqa: E402
from torched_impala_b200.models import MlpPolicy, MlpValueFn  # noqa: E402
from torched_impala_b200.ring import RingQueue  # noqa: E402
from torched_impala_b200.utils import Counter, default_hparams  # noqa: E402

T, B, O, A, H, UPDATES = 20, 32, 4, 2, 32, 4


def main():
    mp.set_start_method("fork", force=True)
    log_dir, mode, out = sys.argv[1], sys.argv[2], sys.argv[3]
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=UPDATES, policy_hidden_dims=H,
                         value_fn_hidden_dims=H, save_every=UPDATES)
    init = synth.init_params(7, O, A, H)
    policy, value_fn = MlpPolicy(O, A, H), MlpValueFn(O, H)
    policy.load_state_dict({k: torch.as_tensor(np.asarray(init["policy"][k])).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.as_tensor(np.asarray(init["value_fn"][k])).double() for k in PKEYS})
    policy.share_memory()
    value_fn.share_memory()  # the learner process writes both modules back at the end
    batches = []
    for u in range(UPDATES):
        b = synth.make_batch(30 + u, T, B, O, A, ragged=(u % 2 == 1))
        b["rewards"] = b["rewards"] * np.float32(3.0)
        batches.append(b)
    valid = [np.arange(T)[:, None] < b["lens"][None, :] for b in batches]
    raw = [float(b["rewards"].astype(np.float64)[m].sum() / B) for b, m in zip(batches, valid)]
    clipped = [float(np.clip(b["rewards"], -1, 1).astype(np.float64)[m].sum() / B) for b, m in zip(batches, valid)]
    q = RingQueue(T, B, O, A, slabs=2)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, log_path=log_dir, timeout=60,
                  reward_clip="abs_one" if mode == "clip" else None)

    def feed():
        for b in batches:
            fed = b if mode == "clip" else dict(b, rewards=np.clip(b["rewards"], -1.0, 1.0))
            for tr in synth.to_trajectories(fed):
                q.put(tr, timeout=60)

    lrn.start()
    t = threading.Thread(target=feed, daemon=True)
    t.start()
    ok = lrn.completion.wait(timeout=180)
    lrn.join()
    t.join(timeout=5)
    q.close()
    assert ok and lrn.p.exitcode == 0, f"learner failed (exit code {lrn.p.exitcode})"
    assert counter.value == UPDATES, counter.value

    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator

    acc = EventAccumulator(os.path.join(log_dir, "l1"))
    acc.Reload()
    ev = acc.Scalars("learner_1/rewards/batch_mean_reward")
    assert [e.step for e in ev] == list(range(1, UPDATES + 1)), [e.step for e in ev]
    np.savez(out, **{f"policy/{k}": v.numpy() for k, v in policy.state_dict().items()},
             **{f"value_fn/{k}": v.numpy() for k, v in value_fn.state_dict().items()},
             logged_reward=np.array([e.value for e in ev]), raw_reward=np.array(raw), clipped_reward=np.array(clipped))
    print(f"REWARD_CLIP_LEARNER_OK mode={mode} updates={counter.value}")


if __name__ == "__main__":
    main()
