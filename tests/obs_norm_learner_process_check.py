"""Run the drop-in Learner with observation normalization as a forked process behind a RingQueue, then resume from
its checkpoint.

    python tests/obs_norm_learner_process_check.py <log dir> <out.npz>

Executed by test_gpu_obs_norm.py in a fresh interpreter (the parent of a forked CUDA process must not have
initialised CUDA).  Feeds the golden c1 batches with obs_norm=True, checks that the checkpoint holds the folded
networks (the modules' weights) and the "obs_norm" key with the statistics of every trained row.  Then load()s the
checkpoint into a new Learner and builds its engine in this process (no fork follows): its statistics must be the
checkpoint's exactly, and its weights are saved to <out.npz> next to the forked run's folded weights, for the test
to compare.
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

def modules(c, init):
    policy, value_fn = MlpPolicy(c["O"], c["A"], c["H_pi"]), MlpValueFn(c["O"], c["H_v"])
    policy.load_state_dict({k: torch.as_tensor(np.asarray(init["policy"][k])).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.as_tensor(np.asarray(init["value_fn"][k])).double() for k in PKEYS})
    return policy, value_fn


def main():
    mp.set_start_method("fork", force=True)
    log_dir, out = sys.argv[1], sys.argv[2]
    g = Golden("c1_cartpole_ragged")
    c = g.case
    hp = g.hp._replace(max_updates=g.updates, verbose=0, eval_every=None, save_every=g.updates)
    policy, value_fn = modules(c, g.init_params())
    policy.share_memory()
    value_fn.share_memory()  # the learner process writes both modules back at the end
    q = RingQueue(c["T"], c["B"], c["O"], c["A"], slabs=2)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, log_path=log_dir, timeout=60, obs_norm=True)

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

    ckpts = glob.glob(os.path.join(log_dir, "l1", "*.pt"))
    assert len(ckpts) == 1, ckpts
    ck = torch.load(ckpts[0])
    assert set(ck) == {"policy_state_dict", "value_fn_state_dict", "obs_norm"}, set(ck)
    st = ck["obs_norm"]
    rows = sum(int(np.minimum(g.batch(u)["lens"], c["T"]).sum()) for u in range(g.updates))
    assert st["count"] == rows, (st["count"], rows)
    for k in PKEYS:  # the checkpoint's networks are the modules': folded into raw-observation coordinates
        assert torch.equal(ck["value_fn_state_dict"][k], value_fn.state_dict()[k]), k
        assert torch.equal(ck["policy_state_dict"][k], policy.state_dict()[k]), k

    # resume: a new Learner load()s the checkpoint and builds its engine here
    p2, v2 = modules(c, g.init_params())
    lrn2 = Learner(2, hp, p2, v2, RingQueue(c["T"], c["B"], c["O"], c["A"], slabs=2), Counter(0), obs_norm=True)
    lrn2.load(ckpts[0])
    eng = lrn2._make_engine()
    st2 = eng.obs_norm_stats()
    assert st2["count"] == st["count"]
    assert (st2["mean"] == st["mean"].numpy()).all() and (st2["var"] == st["var"].numpy()).all()
    resumed = eng.state()
    np.savez(out, **{f"policy/{k}": v.numpy() for k, v in policy.state_dict().items()},
             **{f"value_fn/{k}": v.numpy() for k, v in value_fn.state_dict().items()},
             **{f"resumed/{g_}/{k}": resumed[g_][k].numpy() for g_ in resumed for k in PKEYS},
             count=st["count"], mean=st["mean"].numpy(), var=st["var"].numpy())
    print(f"OBS_NORM_LEARNER_OK updates={counter.value} count={st['count']:.0f}")


if __name__ == "__main__":
    main()
