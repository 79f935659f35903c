"""Run the drop-in Learner with or without off-policy diagnostics as a forked process behind a RingQueue.

    python tests/diag_learner_process_check.py <log dir> <on|off> <weights.npz> [n devices]

Executed by test_gpu_diagnostics.py in a fresh interpreter (the parent of a forked CUDA process must not
have initialised CUDA).  Feeds the golden c1 batches, saves the final policy / value weights to
<weights.npz> and, with diagnostics on, checks that rank 0's event file holds the five diagnostic tags at
every logged update (and that no other learner directory was written).
"""
import glob
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

DIAG_TAGS = ("offpolicy/log_ratio_mean", "offpolicy/rho_clip_fraction", "offpolicy/c_clip_fraction",
             "offpolicy/kl_behaviour_current", "value/explained_variance")


def main():
    mp.set_start_method("fork", force=True)
    log_dir, diag, out, n_dev = sys.argv[1], sys.argv[2] == "on", sys.argv[3], int(sys.argv[4]) if len(sys.argv) > 4 else 1
    g = Golden("c1_cartpole_ragged")
    c = g.case
    hp = g.hp._replace(max_updates=g.updates, verbose=1, eval_every=None)
    policy, value_fn = MlpPolicy(c["O"], c["A"], c["H_pi"]), MlpValueFn(c["O"], c["H_v"])
    init = g.init_params()
    policy.load_state_dict({k: torch.from_numpy(init["policy"][k]).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.from_numpy(init["value_fn"][k]).double() for k in PKEYS})
    policy.share_memory()
    q = RingQueue(c["T"], c["B"], c["O"], c["A"], slabs=2)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, log_path=log_dir, timeout=60,
                  devices=[f"cuda:{i}" for i in range(n_dev)], diagnostics=diag)

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

    assert sorted(os.listdir(log_dir)) == ["l1"], os.listdir(log_dir)  # one writer: rank 0's
    acc = EventAccumulator(glob.glob(os.path.join(log_dir, "l1"))[0])
    acc.Reload()
    tags = set(acc.Tags()["scalars"])
    steps = sorted(e.step for e in acc.Scalars("learner_1/loss/total_loss"))
    assert steps == list(range(1, g.updates + 1)), steps
    for tag in DIAG_TAGS:
        full = f"learner_1/{tag}"
        if diag:
            assert full in tags, (full, tags)
            assert sorted(e.step for e in acc.Scalars(full)) == steps, full
        else:
            assert full not in tags, full
    if diag:
        clip = [e.value for e in acc.Scalars("learner_1/offpolicy/rho_clip_fraction")]
        assert all(0.0 <= x <= 1.0 for x in clip), clip
    print(f"DIAG_LEARNER_OK diagnostics={diag} updates={counter.value} devices={n_dev}")


if __name__ == "__main__":
    main()
