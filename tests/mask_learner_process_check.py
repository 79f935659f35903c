"""Run the drop-in Learner with a masked categorical policy as a forked process behind a masked RingQueue, or behind
a plain mp.Queue of trajectories that carry action_mask.

    python tests/mask_learner_process_check.py <log dir> <out.npz> ring|queue

Executed by test_gpu_action_mask_host.py in a fresh interpreter (the parent of a forked CUDA process must not have
initialised CUDA).  Synthetic actors put reference-format trajectories (a (1,) int64, logits (A,) float64 with garbage
at the illegal entries, action_mask (A,) bool) into the queue; the final weights go to <out.npz>.  `oracle_run()` is
the float64 oracle learner on the same batches, for the test to compare with.
"""
import os
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.utils import default_hparams  # noqa: E402

T, B, O, A, H, UPDATES = 20, 32, 6, 8, 32, 4
PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")


def setup():
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=UPDATES, policy_hidden_dims=H,
                         value_fn_hidden_dims=H, save_every=UPDATES, rho_bar=1.0, c_bar=1.0)
    init = synth.init_params(7, O, A, H)
    batches = [synth.make_masked_batch(30 + u, T, B, O, A, density=0.5, ragged=(u % 2 == 1), params=init)
               for u in range(UPDATES)]
    return hp, init, batches


def oracle_run():
    import action_mask_oracle as aorc

    hp, init, batches = setup()
    lrn = aorc.MaskLearner(init, hp, (A,))
    for b in batches:
        lrn.update(b)
    return lrn.state()


def main():
    import torch.multiprocessing as mp

    from torched_impala_b200.learner import Learner
    from torched_impala_b200.models import MlpPolicy, MlpValueFn
    from torched_impala_b200.ring import RingQueue
    from torched_impala_b200.utils import Counter

    mp.set_start_method("fork", force=True)
    log_dir, out, kind = sys.argv[1], sys.argv[2], sys.argv[3]
    hp, init, batches = setup()
    policy, value_fn = MlpPolicy(O, A, H), MlpValueFn(O, H)
    policy.load_state_dict({k: torch.as_tensor(np.asarray(init["policy"][k])).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.as_tensor(np.asarray(init["value_fn"][k])).double() for k in PKEYS})
    policy.share_memory()
    value_fn.share_memory()  # the learner process writes both modules back at the end
    q = RingQueue(T, B, O, A, slabs=2, action_mask=True) if kind == "ring" else mp.Queue()
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, log_path=log_dir, timeout=60, action_mask=True)

    def feed():
        for b in batches:
            for tr in synth.to_trajectories(b):
                q.put(tr, timeout=60) if kind == "ring" else q.put(tr)

    lrn.start()
    t = threading.Thread(target=feed, daemon=True)
    t.start()
    ok = lrn.completion.wait(timeout=180)
    lrn.join()
    t.join(timeout=5)
    if kind == "ring":
        q.close()
    assert ok and lrn.p.exitcode == 0, f"learner failed (exit code {lrn.p.exitcode})"
    assert counter.value == UPDATES, counter.value
    assert policy.state_dict()["model.3.weight"].shape == (A, H)
    np.savez(out, **{f"policy/{k}": v.numpy() for k, v in policy.state_dict().items()},
             **{f"value_fn/{k}": v.numpy() for k, v in value_fn.state_dict().items()})
    print(f"MASK_LEARNER_OK updates={counter.value}")


if __name__ == "__main__":
    main()
