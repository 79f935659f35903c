"""Run the drop-in Learner with byte observations as a forked process behind a uint8 RingQueue, and the
float32 Learner on the same trajectories; both must end with the same weights.

Executed by test_gpu_obs_u8.py in a fresh interpreter (the parent of a forked CUDA process must never have
initialised CUDA).  Usage: obs_u8_learner_process_check.py O A H  (O > 128: the byte kernels; O <= 128:
the widened float path).  MinAtar-style 0/1 planes, ragged trajectories, 3 updates.
"""
import os
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from conftest import PKEYS  # noqa: E402
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.learner import Learner  # noqa: E402
from torched_impala_b200.models import MlpPolicy, MlpValueFn  # noqa: E402
from torched_impala_b200.ring import RingQueue  # noqa: E402
from torched_impala_b200.utils import Counter, default_hparams  # noqa: E402

T, B, UPDATES = 20, 64, 3


def run(obs_dtype, O, A, H, hp, init, batches):
    policy, value_fn = MlpPolicy(O, A, H), MlpValueFn(O, H)
    policy.load_state_dict({k: torch.from_numpy(init["policy"][k]).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.from_numpy(init["value_fn"][k]).double() for k in PKEYS})
    policy.share_memory()
    value_fn.share_memory()
    q = RingQueue(T, B, O, A, slabs=2, obs_dtype=obs_dtype)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, timeout=60, obs_dtype=obs_dtype)

    def feed():  # stands in for actor processes: the reference wire format (float64 obs)
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
    assert ok, f"{obs_dtype} learner never signalled completion"
    assert lrn.p.exitcode == 0, f"{obs_dtype} learner exit code {lrn.p.exitcode}"
    assert counter.value == UPDATES, counter.value
    return {"policy": {k: v.clone() for k, v in policy.state_dict().items()},
            "value_fn": {k: v.clone() for k, v in value_fn.state_dict().items()}}


def main():
    O, A, H = (int(v) for v in sys.argv[1:4])
    mp.set_start_method("fork", force=True)
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=UPDATES, policy_hidden_dims=H,
                         value_fn_hidden_dims=H)
    init = synth.init_params(21, O, A, H)
    batches = [synth.make_batch(40 + u, T, B, O, A, ragged=True, obs_kind="planes") for u in range(UPDATES)]
    got = run("uint8", O, A, H, hp, init, batches)
    want = run("float32", O, A, H, hp, init, batches)
    for grp in ("policy", "value_fn"):
        for k in PKEYS:
            assert torch.equal(got[grp][k], want[grp][k]), (grp, k, float((got[grp][k] - want[grp][k]).abs().max()))
    assert not torch.equal(got["policy"][PKEYS[0]], torch.from_numpy(init["policy"][PKEYS[0]]).double())
    print(f"OBS_U8_LEARNER_OK O={O} A={A} H={H} updates={UPDATES}")


if __name__ == "__main__":
    main()
