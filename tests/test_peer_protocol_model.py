"""CPU model of the push all-reduce handshake (csrc/optim.cu, tail of csrc/mlp_bwd_tc.cu), LL format.

Protocol: the backward of step s on rank `me` STORES each value of its contribution, tagged with s,
into slot `me` of parity s & 1 in EVERY rank's gather buffer (no flag, no fence); the optimizer of
step s polls its own `world` slots until every element carries tag s, then uses them.  The safety
argument - parity-double-buffered slots need no acknowledgement round trip - is a protocol
property, independent of CUDA: rank threads with random delays run it here, writing element by
element with pauses (so readers do see half-written slots), and check that every value a reader
accepts is exactly the one the writer sent for that step (never a value a fast peer has already
overwritten).  Every rank reads the slots of a step twice, as the optimizer and then the observation-statistics
update (impala_obs_norm_update, csrc/obs_norm.cu) do, the second pass after the first and before the rank's next
push.  The same model with ONE buffer per rank must fail, which shows the test can see the hazard the second
buffer removes.  A reader that waits too long is a failure too (a deadlock, not a pass)."""
import random
import threading
import time

import pytest

ELEMS = 6


def run_ranks(world: int, steps: int, buffers: int, seed: int):
    # gather[owner][parity][writer][element] = (tag, payload)
    gather = [[[[(0, None)] * ELEMS for _ in range(world)] for _ in range(buffers)] for _ in range(world)]
    errors, stop = [], threading.Event()

    def rank(me: int):
        rng = random.Random(seed * 131 + me)
        for s in range(1, steps + 1):
            if stop.is_set():
                return
            time.sleep(rng.random() * 2e-4)              # forward / V-trace / backward of step s ...
            for e in range(ELEMS):                       # ... whose tail pushes tagged values to everyone
                for p in range(world):
                    gather[p][s % buffers][me][e] = (s, (me, s, e))
                if rng.random() < 0.2:
                    time.sleep(0)                        # a reader may observe a half-written slot
            # the optimizer, then the statistics update: each polls the LOCAL slots of step s element by element
            for reader in ("optimizer", "statistics"):
                t0 = time.time()
                got = []
                for r in range(world):
                    for e in range(ELEMS):
                        while True:
                            tag, val = gather[me][s % buffers][r][e]
                            if tag == s:
                                break
                            if stop.is_set():
                                return
                            if tag > s or time.time() - t0 > 20:  # overwritten before it was read, or never written
                                errors.append((reader, me, s, r, e, tag))
                                stop.set()
                                return
                            time.sleep(0)
                        got.append(val)
                    if rng.random() < 0.1:
                        time.sleep(rng.random() * 3e-4)  # a slow reader
                if got != [(r, s, e) for r in range(world) for e in range(ELEMS)]:
                    errors.append((reader, me, s, got))
                    stop.set()
                    return

    ts = [threading.Thread(target=rank, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=90)
    return errors


@pytest.mark.parametrize("world", [2, 4, 8])
def test_parity_buffers_need_no_acknowledgement(world):
    for seed in range(3):
        assert run_ranks(world, steps=150, buffers=2, seed=seed) == []


def test_single_buffer_is_unsafe_without_acknowledgement():
    """Sanity of the model itself: with one buffer a fast rank overwrites what a slow rank has not
    read yet - the hazard must show up within a few attempts."""
    assert any(run_ranks(4, steps=150, buffers=1, seed=seed) for seed in range(8))
