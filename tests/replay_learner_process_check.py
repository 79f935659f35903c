"""Run the drop-in Learner with experience replay as a forked process, then rebuild what it must have computed.

    python tests/replay_learner_process_check.py <ring|queue> O k A H obs_dtype

Executed by test_gpu_replay.py in a fresh interpreter (the parent of a forked CUDA process must not have
initialised CUDA before the fork).  The learner (replay_slabs=2, replay_columns=B/2, diagnostics on) sits behind a
RingQueue of Bf = B/2 columns or an mp.Queue and is fed exactly max_updates * Bf ragged trajectories.  Afterwards
this process recomputes every update's plan from the seed with ReplaySampler, composes the B-column batches on
the host (oracle.replay.compose_batch) and runs them through a plain engine: the learner's final weights must
equal that engine's bit for bit.
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
from oracle.replay import compose_batch  # noqa: E402
from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.learner import Learner  # noqa: E402
from torched_impala_b200.models import MlpPolicy, MlpValueFn  # noqa: E402
from torched_impala_b200.replay import ReplaySampler  # noqa: E402
from torched_impala_b200.ring import RingQueue  # noqa: E402
from torched_impala_b200.utils import Counter, default_hparams  # noqa: E402

T, B, BR, R, UPDATES = 20, 64, 32, 2, 6
BF = B - BR


def main():
    transport = sys.argv[1]
    O, k, A, H = (int(v) for v in sys.argv[2:6])
    obs_dtype = sys.argv[6]
    mp.set_start_method("fork", force=True)
    hp = default_hparams(batch_size=B, max_timesteps=T, max_updates=UPDATES, policy_hidden_dims=H,
                         value_fn_hidden_dims=H, eval_every=None)
    init = synth.init_params(23, O, A, H)
    kind = "bytes" if obs_dtype == "uint8" else "normal"
    fresh = [synth.make_batch(60 + u, T, BF, O, A, ragged=True, obs_kind=kind, frames=k) for u in range(UPDATES)]
    trajs = []
    for fb in fresh:
        trajs += synth.to_trajectories(synth.stack_frames(fb, k) if k > 1 else fb)
    policy, value_fn = MlpPolicy(O, A, H), MlpValueFn(O, H)
    policy.load_state_dict({key: torch.from_numpy(init["policy"][key]).double() for key in PKEYS})
    value_fn.load_state_dict({key: torch.from_numpy(init["value_fn"][key]).double() for key in PKEYS})
    policy.share_memory()
    value_fn.share_memory()
    q = RingQueue(T, BF, O, A, slabs=2, obs_dtype=obs_dtype, frames=k) if transport == "ring" \
        else mp.Queue(maxsize=hp.queue_lim)
    counter = Counter(0)
    lrn = Learner(1, hp, policy, value_fn, q, counter, timeout=60, obs_dtype=obs_dtype, frames=k, diagnostics=True,
                  replay_slabs=R, replay_columns=BR)

    def feed():  # stands in for actor processes
        for tr in trajs:
            q.put(tr, timeout=60)

    lrn.start()
    t = threading.Thread(target=feed, daemon=True)
    t.start()
    ok = lrn.completion.wait(timeout=240)
    lrn.join()
    t.join(timeout=5)
    assert ok and lrn.p.exitcode == 0, f"learner failed (exit code {lrn.p.exitcode})"
    assert counter.value == UPDATES, counter.value
    assert not t.is_alive()  # every one of the UPDATES * BF trajectories was taken
    if transport == "ring":
        q.close()
    else:
        assert q.empty()

    # the same updates on a plain engine (CUDA is first touched here, after the fork)
    from torched_impala_b200.engine import LearnerEngine

    eng = LearnerEngine(T, B, O, A, H, H, hp, obs_dtype=obs_dtype, frames=k, diagnostics=True)
    eng.load_state(init)
    sampler, store = ReplaySampler(0, R, BF, BR), {}
    for n in range(1, UPDATES + 1):
        store[n % sampler.slots] = fresh[n - 1]
        eng.fill_host(compose_batch(store, sampler.plan(n)), 0)
        eng.ingest(0)
        eng.step(0)
        eng.synchronize()
    want = eng.state()
    for grp, mod in (("policy", policy), ("value_fn", value_fn)):
        for key in PKEYS:
            got = mod.state_dict()[key]
            assert torch.equal(got, want[grp][key]), (grp, key, float((got - want[grp][key]).abs().max()))
    assert not torch.equal(policy.state_dict()[PKEYS[0]], torch.from_numpy(init["policy"][PKEYS[0]]).double())
    print(f"REPLAY_LEARNER_OK transport={transport} O={O} frames={k} A={A} H={H} obs_dtype={obs_dtype} "
          f"updates={UPDATES} fresh_trajectories={len(trajs)}")


if __name__ == "__main__":
    main()
