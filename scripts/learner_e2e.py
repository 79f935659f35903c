"""End to end THROUGH the product API: K synthetic actor processes -> RingQueue -> forked `Learner`
-> sm_90a kernels -> weight publication, for a BASELINE config (default c3: 32 CPU actors, one GPU).

    python scripts/learner_e2e.py [--config c3|c4] [--actors 32] [--updates 300] [--devices 1]
                                  [--payload block|trajectory] [--block 128]

Prints ONE JSON line: learner steps/s and trajectories/s measured on the shared update counter
between update `warmup` and the last one (wall clock of the launcher, which never touches CUDA -
fork start method as in reference train.py:42).  payload=block: actors push pre-stacked
(T, n, .) blocks (`RingQueue.put_block`, SURVEY section 7); payload=trajectory: the reference wire
format, one `utils.Trajectory` of ~5T tiny tensors per put (what an unmodified actor.py sends).
Run in a fresh interpreter (bench.py spawns it as a subprocess)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from torched_impala_b200 import synth  # noqa: E402
from torched_impala_b200.learner import Learner  # noqa: E402
from torched_impala_b200.models import MlpPolicy, MlpValueFn  # noqa: E402
from torched_impala_b200.ring import RingQueue  # noqa: E402
from torched_impala_b200.utils import Counter, default_hparams  # noqa: E402

CFG = {"c3": dict(T=20, B=1024, O=24, A=4, H=256), "c4": dict(T=20, B=4096, O=24, A=4, H=256),
       "c1": dict(T=20, B=8, O=4, A=2, H=32), "c5": dict(T=100, B=8192, O=64, A=4, H=512)}


def actor_main(aid, ring, learner_done, w, payload, block, seed):
    """Synthetic actor: a pool of pre-generated trajectories pushed as fast as the ring takes them.
    It reads the published policy version like actor.py:70 reads the weights (once per put)."""
    torch.set_num_threads(1)
    n = block if payload == "block" else 8
    pool = synth.make_batch(seed, w["T"], n, w["O"], w["A"])
    trajs = synth.to_trajectories(pool) if payload == "trajectory" else None
    rsum = pool["rewards"].sum(0, dtype=np.float64)
    i = 0
    while not learner_done.is_set():
        try:
            if payload == "block":
                ring.put_block(pool, rsum, timeout=0.5)
            else:
                ring.put(trajs[i % n], timeout=0.5)
                i += 1
        except Exception:  # queue.Full -> retry until the learner is done (actor.py:116-124)
            continue


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3", choices=sorted(CFG))
    ap.add_argument("--actors", type=int, default=32)
    ap.add_argument("--updates", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--devices", type=int, default=1)
    ap.add_argument("--payload", default="block", choices=["block", "trajectory"])
    ap.add_argument("--block", type=int, default=128)
    ap.add_argument("--publish-every", type=int, default=1)
    ap.add_argument("--deadline", type=float, default=120.0)
    a = ap.parse_args()
    w = CFG[a.config]
    mp.set_start_method("fork", force=True)
    os.environ.setdefault("IMPALA_DEBUG_STACKS", "25")  # a stuck learner shows where
    hp = default_hparams(batch_size=w["B"], max_timesteps=w["T"], policy_hidden_dims=w["H"], value_fn_hidden_dims=w["H"],
                         max_updates=a.updates, verbose=0, eval_every=None, save_every=10 ** 9, n_actors=a.actors)
    policy, value_fn = MlpPolicy(w["O"], w["A"], w["H"]), MlpValueFn(w["O"], w["H"])
    policy.share_memory()
    block = min(a.block, w["B"])
    while w["B"] % block:
        block //= 2
    ring = RingQueue(w["T"], w["B"], w["O"], w["A"], slabs=3)
    counter = Counter(0)
    devices = [f"cuda:{i}" for i in range(a.devices)]
    lrn = Learner(1, hp, policy, value_fn, ring, counter, log_path=None, timeout=120, devices=devices,
                  publish_every=a.publish_every)
    actors = [mp.Process(target=actor_main, args=(i, ring, lrn.completion, w, a.payload, block, 100 + i), daemon=True)
              for i in range(a.actors)]
    for p in actors:
        p.start()
    lrn.start()
    t_w = t_end = None
    v0 = None
    deadline = time.time() + a.deadline
    last_print = time.time()
    while time.time() < deadline and not lrn.completion.is_set():
        c = counter.value
        if time.time() - last_print > 5:
            last_print = time.time()
            print(f"[e2e] {c} updates, filled={[int(x) for x in ring._control()['filled'].sum(1)]} "
                  f"ticket={int(ring._control()['ticket'][0])} released={ring._control()['released'].tolist()} "
                  f"version={lrn.policy_version}", file=sys.stderr, flush=True)
        if t_w is None and c >= a.warmup:
            t_w, c_w, v0 = time.perf_counter(), c, lrn.policy_version
        if c >= a.updates:
            break
        time.sleep(0.0005)
    t_end, c_end = time.perf_counter(), counter.value
    ok = lrn.completion.wait(timeout=30)
    if not ok:
        lrn.terminate()
    lrn.join()
    for p in actors:
        p.join(timeout=5)
        if p.is_alive():
            p.terminate()
    ring.close()
    if not ok or lrn.p.exitcode != 0 or t_w is None or c_end <= c_w:
        print(json.dumps(dict(error=f"learner exit {lrn.p.exitcode}, updates {counter.value}")))
        sys.exit(1)
    sps = (c_end - c_w) / (t_end - t_w)
    print(json.dumps(dict(
        what="steps/s through Learner + RingQueue + synthetic actor processes (wall clock on the shared update counter)",
        config=a.config, **w, actors=a.actors, payload=a.payload, block=block if a.payload == "block" else 1,
        devices=a.devices, updates_timed=c_end - c_w, steps_per_s=sps, trajectories_per_s=sps * w["B"],
        h2d_bytes_per_step=int(ring.slab_bytes), weight_publications=(lrn.policy_version - (v0 or 0)) // 2,
        publish_every=a.publish_every, host_cores=os.cpu_count())))


if __name__ == "__main__":
    main()
