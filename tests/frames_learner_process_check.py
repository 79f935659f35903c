"""Run the drop-in Learner as a forked process behind a frame RingQueue (frames=k) and behind a dense RingQueue
on the same trajectories; both must end with the same weights.

The dense ring zero-fills observation rows past a trajectory's length; the frame ring keeps the frames those
rows share with valid rows.  Every padded step has zero importance weight, trace coefficient, discount and
output gradients, so the weights must still be identical (DESIGN.md section 3).

Executed by test_gpu_frames.py in a fresh interpreter (the parent of a forked CUDA process must never have
initialised CUDA).  Usage: frames_learner_process_check.py O k A H obs_dtype devices.  Ragged trajectories in
the reference wire format (float64 obs), 3 updates.
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


def run(frames, obs_dtype, devices, O, A, H, hp, init, trajs):
    policy, value_fn = MlpPolicy(O, A, H), MlpValueFn(O, H)
    policy.load_state_dict({k: torch.from_numpy(init["policy"][k]).double() for k in PKEYS})
    value_fn.load_state_dict({k: torch.from_numpy(init["value_fn"][k]).double() for k in PKEYS})
    policy.share_memory()
    value_fn.share_memory()
    q = RingQueue(T, B, O, A, slabs=2, obs_dtype=obs_dtype, frames=frames)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, timeout=60, obs_dtype=obs_dtype, frames=frames,
                  devices=[f"cuda:{i}" for i in range(devices)])

    def feed():  # stands in for actor processes
        for tr in trajs:
            q.put(tr, timeout=60)

    lrn.start()
    t = threading.Thread(target=feed, daemon=True)
    t.start()
    ok = lrn.completion.wait(timeout=240)
    lrn.join()
    t.join(timeout=5)
    q.close()
    assert ok, f"frames={frames} learner never signalled completion"
    assert lrn.p.exitcode == 0, f"frames={frames} learner exit code {lrn.p.exitcode}"
    assert counter.value == UPDATES, counter.value
    return {"policy": {k: v.clone() for k, v in policy.state_dict().items()},
            "value_fn": {k: v.clone() for k, v in value_fn.state_dict().items()}}


def main():
    O, k, A, H = (int(v) for v in sys.argv[1:5])
    obs_dtype, devices = sys.argv[5], int(sys.argv[6])
    mp.set_start_method("fork", force=True)
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=UPDATES, policy_hidden_dims=H,
                         value_fn_hidden_dims=H)
    init = synth.init_params(21, O, A, H)
    kind = "bytes" if obs_dtype == "uint8" else "normal"
    trajs = []
    for u in range(UPDATES):
        fb = synth.make_batch(40 + u, T, B, O, A, ragged=True, obs_kind=kind, frames=k)
        trajs += synth.to_trajectories(synth.stack_frames(fb, k))
    got = run(k, obs_dtype, devices, O, A, H, hp, init, trajs)
    want = run(1, obs_dtype, devices, O, A, H, hp, init, trajs)
    for grp in ("policy", "value_fn"):
        for key in PKEYS:
            assert torch.equal(got[grp][key], want[grp][key]), (grp, key,
                                                                float((got[grp][key] - want[grp][key]).abs().max()))
    assert not torch.equal(got["policy"][PKEYS[0]], torch.from_numpy(init["policy"][PKEYS[0]]).double())
    print(f"FRAMES_LEARNER_OK O={O} frames={k} A={A} H={H} obs_dtype={obs_dtype} devices={devices} updates={UPDATES}")


if __name__ == "__main__":
    main()
