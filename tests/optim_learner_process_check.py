"""Run the drop-in Learner with RMSprop and a learning-rate schedule as a forked process behind a RingQueue.

    python tests/optim_learner_process_check.py <log dir> <weights.npz>

Executed by test_gpu_optim_sched.py in a fresh interpreter (the parent of a forked CUDA process must not have
initialised CUDA).  Feeds the golden c1 batches, saves the final policy / value weights to <weights.npz> and
checks that rank 0's event file holds optim/lr = hp.lr * lambda(n - 1) at every update n.
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

from conftest import PKEYS, Golden  # noqa: E402
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.learner import Learner  # noqa: E402
from torched_impala_b200.models import MlpPolicy, MlpValueFn  # noqa: E402
from torched_impala_b200.ring import RingQueue  # noqa: E402
from torched_impala_b200.utils import Counter  # noqa: E402


def main():
    mp.set_start_method("fork", force=True)
    log_dir, out = sys.argv[1], sys.argv[2]
    g = Golden("c1_cartpole_ragged")
    c = g.case
    hp = g.hp._replace(max_updates=g.updates, verbose=0, eval_every=None)
    policy, value_fn = MlpPolicy(c["O"], c["A"], c["H_pi"]), MlpValueFn(c["O"], c["H_v"])
    init = g.init_params()
    policy.load_state_dict({k: torch.from_numpy(init["policy"][k]).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.from_numpy(init["value_fn"][k]).double() for k in PKEYS})
    policy.share_memory()
    value_fn.share_memory()  # the learner process writes both modules back at the end
    q = RingQueue(c["T"], c["B"], c["O"], c["A"], slabs=2)
    counter = Counter(0)

    def lam(e):  # a closure over local state: it would not pickle, the Learner tabulates it before forking
        return 1.0 - e / g.updates

    lrn = Learner(1, hp, policy, value_fn, q, counter, log_path=log_dir, timeout=60, optimizer="rmsprop",
                  optimizer_kwargs=dict(eps=0.01, momentum=0.5), lr_lambda=lam)

    def feed():
        for u in range(g.updates):
            for tr in synth.to_trajectories(g.batch(u)):
                q.put(tr, timeout=60)

    lrn.start()
    t = threading.Thread(target=feed, daemon=True)
    t.start()
    ok = lrn.completion.wait(timeout=180)
    lrn.join()
    t.join(timeout=5)
    q.close()
    assert ok and lrn.p.exitcode == 0, f"learner failed (exit code {lrn.p.exitcode})"
    assert counter.value == g.updates, counter.value
    np.savez(out, **{f"policy/{k}": v.numpy() for k, v in policy.state_dict().items()},
             **{f"value_fn/{k}": v.numpy() for k, v in value_fn.state_dict().items()})

    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator

    acc = EventAccumulator(os.path.join(log_dir, "l1"))
    acc.Reload()
    events = acc.Scalars("learner_1/optim/lr")
    assert [e.step for e in events] == list(range(1, g.updates + 1)), [e.step for e in events]
    for e in events:
        want = float(np.float32(hp.lr * lam(e.step - 1)))
        assert e.value == want, (e.step, e.value, want)
    print(f"OPTIM_LEARNER_OK updates={counter.value} lr={[e.value for e in events]}")


if __name__ == "__main__":
    main()
