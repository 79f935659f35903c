"""Drop-in `Learner` for the reference's actor/learner split, running the update on the GPU.

Same constructor, lifecycle methods, events, checkpoint format and module-level loss
helpers as `learner.py` (constructor `:18-28`, `start/terminate/join`
`:55-65`, `_learn` `:67-275`, `save/load/policy_weights` `:277-295`, helpers `:298-321`),
so `train.py:69` and the unmodified `actor.py` (`:68,70,118,121`) work against it:

  * trajectories arrive as pickled `utils.Trajectory` objects through the same `mp.Queue`
    (or through `ring.RingQueue`, same `put()` call); `queue.Empty` after `timeout` seconds sets
    `completion` and re-raises (`:91-100`);
  * new policy weights are copied IN PLACE into the (shared-memory, float64) `policy` module the
    actors read through `learner.policy_weights` (`actor.py:70`);
  * `update_counter.increment()` once per update; TensorBoard scalars under the same tags;
    checkpoints with keys `policy_state_dict` / `value_fn_state_dict`.

What changes is where the arithmetic happens and that nothing on the host sits on the critical
path of the device (SURVEY 8f-2, 8f-4):

  * `_learn` packs each trajectory into a pinned, zero-padded time-major host slab (replacing the
    torch.stack calls at `:104-109,117`) and hands the batch to `engine.LearnerEngine`, i.e. to the
    sm_90a kernels behind include/impala_b200.h; batch i+1 is collected and DMA'd while the
    kernels of batch i run;
  * weight publication: only the POLICY is published (it is all `actor.py:70` reads; `train.py:67`
    shares only the policy): after the step an in-stream device copy freezes the policy block, a
    side stream brings it to a double-buffered pinned snapshot, and a publisher thread writes it
    into the shared tensors under a version counter (`policy_version`, odd while a write is in
    progress; `policy_snapshot()` returns a consistent copy).  `publish_every` thins it out.  The
    value function reaches its module at checkpoints and at the end;
  * the logged scalars of update n are read while update n + 1 runs;
  * evaluation (`learner.py:195-214`) runs on a frozen copy of the policy in a background thread,
    it no longer blocks updates and no longer flips the training module's mode;
  * `devices=[...]`: data-parallel over the GPUs of one node, still ONE learner object/process
    for the launcher (dp.py): rank 0 lives here, publishes weights and logs.

CUDA is initialised inside the learner process only (`train.py:42` forces the fork start method,
so the parent must never touch the device); a policy / value_fn that already lives on a CUDA
device is rejected with instructions (the reference picks `cuda` at import when it is visible).

Dropout: the reference MLPs carry `Dropout(p=0.8)` (models.py:15,44) and never call `.eval()` on
the learner's nets before the first evaluation.  This learner implements the deterministic
(`.eval()`) forward, the setting every parity number is quoted in (SURVEY.md section 0.4) -
swapping the class therefore changes training dynamics, not only speed (INTEGRATION.md).
"""
from __future__ import annotations

import copy
import queue
import sys
import threading
import time
from pathlib import Path

import numpy as np
import torch
import torch.multiprocessing as mp

PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")


def _np(t, dtype):
    """Stacked trajectory field -> numpy of `dtype` (tensors an actor left on a GPU are fetched)."""
    return t.detach().to(dtype).cpu().numpy()


def check_trajectory(traj, T: int) -> int:
    """Length checks of learner.py:104-109's implicit contract; returns the number of steps."""
    L = len(traj.r)
    if L < 1 or L > T:
        raise ValueError(f"trajectory {getattr(traj, 'id', '?')} has {L} steps; the learner was "
                         f"built for 1..{T} (hp.max_timesteps)")
    if len(traj.obs) != L + 1 or len(traj.a) != L or len(traj.d) != L or len(traj.logits) != L:
        raise ValueError("malformed trajectory: obs must have one more entry than a/r/d/logits")
    return L


def pack_trajectory(views: dict, b: int, traj, T: int) -> float:
    """Write one reference-format trajectory into column `b` of a host batch slab.

    Replaces learner.py:104-109,117 (five torch.stack calls + `disc`): float64 -> float32,
    int64 -> int32, bool -> u8, zero padding past the trajectory's length.  Returns the
    trajectory's reward sum (learner.py:108)."""
    L = check_trajectory(traj, T)
    views["obs"][:L + 1, b] = _np(torch.stack(traj.obs), torch.float32)
    views["obs"][L + 1:, b] = 0
    views["beh_logits"][:L, b] = _np(torch.stack(traj.logits), torch.float32)
    views["beh_logits"][L:, b] = 0
    views["actions"][:L, b] = _np(torch.stack(traj.a).reshape(L), torch.int32)
    views["actions"][L:, b] = 0
    r = torch.stack(traj.r)
    views["rewards"][:L, b] = _np(r, torch.float32)
    views["rewards"][L:, b] = 0
    views["done"][:L, b] = _np(torch.stack(traj.d), torch.uint8)
    views["done"][L:, b] = 0
    views["lens"][b] = L
    return float(r.sum(dtype=torch.float64))  # summed as received (float64 from actor.py), like learner.py:108


def _dims(policy, value_fn):
    sd_p, sd_v = policy.state_dict(), value_fn.state_dict()
    H_pi, O = sd_p[PKEYS[0]].shape
    A = sd_p[PKEYS[2]].shape[0]
    H_v = sd_v[PKEYS[0]].shape[0]
    return int(O), int(A), int(H_pi), int(H_v)


class _Publisher:
    """Asynchronous policy-weight publication (SURVEY 8f-2; replaces the per-update full
    state_dict copy behind learner.py:293-295 / actor.py:70).

    post(n): [learner stream] policy block -> device staging buffer (freezes update n's weights
    without stalling the next update), [side stream] staging -> pinned host snapshot; the
    publisher thread waits for that copy and writes the float64 shared tensors under a seqlock.
    Two snapshot slots; publications coalesce when the host cannot keep up with the updates."""

    def __init__(self, eng, policy, version):
        self.eng, self.policy, self.version = eng, policy, version
        n = eng.n_pi
        self.stream = torch.cuda.Stream(device=eng.dev)
        self.stage = [torch.empty(n, dtype=torch.float32, device=eng.dev) for _ in range(2)]
        self.host = [torch.empty(n, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.free = [threading.Event(), threading.Event()]
        for e in self.free:
            e.set()
        # CUDA events of a slot are reused: a slot is posted again only after its previous publication
        # has been written (free[s] set after landed.synchronize())
        self.ev_frozen = [torch.cuda.Event() for _ in range(2)]
        self.ev_landed = [torch.cuda.Event() for _ in range(2)]
        self.views = []  # (flat offset, shared tensor) of the policy's four parameters
        sd = policy.state_dict()
        for grp, key, off, shp in eng._segments():
            if grp == "policy":
                self.views.append((off, int(np.prod(shp)), sd[key]))
        self.q: queue.SimpleQueue = queue.SimpleQueue()
        self.i = 0
        self.published = 0
        self.error = None
        self.thread = threading.Thread(target=self._run, name="impala-publisher", daemon=True)
        self.thread.start()

    def post(self, n: int, force: bool = False) -> bool:
        """Publish the weights of update n.  Coalescing: if the previous publication is still being
        written the call returns False at once (the next one carries newer weights anyway) - the
        actors always see the newest weights the host can deliver, the update loop never waits.
        force=True (evaluation / checkpoint points, last update) waits for a free snapshot slot."""
        s = self.i & 1
        if not self.free[s].is_set():
            if not force:
                return False
            self.free[s].wait()
        self.i += 1
        self.free[s].clear()
        eng = self.eng
        frozen, landed = self.ev_frozen[s], self.ev_landed[s]
        with eng._on_stream():
            self.stage[s].copy_(eng.params[:eng.n_pi], non_blocking=True)
            frozen.record(eng.stream)
        self.stream.wait_event(frozen)
        with torch.cuda.stream(self.stream):
            self.host[s].copy_(self.stage[s], non_blocking=True)
            landed.record(self.stream)
        self.q.put((s, n, landed))
        return True

    def _run(self) -> None:
        try:
            while True:
                item = self.q.get()
                if item is None:
                    return
                s, n, landed = item
                landed.synchronize()
                self._write(self.host[s])
                self.published = n
                self.free[s].set()
        except BaseException as e:  # noqa: BLE001 - surfaced by the learner loop
            self.error = e
            for ev in self.free:
                ev.set()

    def _write(self, flat: torch.Tensor) -> None:
        v = self.version
        with torch.no_grad():
            v.value += 1             # odd: a write is in progress
            for off, cnt, dst in self.views:
                dst.copy_(flat[off:off + cnt].view(dst.shape))  # float32 -> float64, in place
            v.value += 1

    def drain(self) -> None:
        """Block until everything posted so far is in the shared tensors."""
        for e in self.free:
            e.wait()
        if self.error is not None:
            raise self.error

    def close(self) -> None:
        self.q.put(None)
        self.thread.join(timeout=10)


class Learner:
    def __init__(self, id, hparams, policy, value_fn, q, update_counter, log_path=None,
                 timeout=200, device="cuda:0", mode="reference", devices=None, publish_every=1,
                 evaluator=None):
        self.id = id
        self.hp = hparams
        self.policy = policy
        self.value_fn = value_fn
        self.timeout = timeout
        self.q = q
        self.update_counter = update_counter
        self.devices = [str(d) for d in devices] if devices else [str(device)]
        self.device = self.devices[0]
        self.mode = mode
        self.publish_every = max(1, int(publish_every))
        for name, mod in (("policy", policy), ("value_fn", value_fn)):
            if any(p.is_cuda for p in mod.parameters()):
                raise ValueError(
                    f"{name} lives on a CUDA device: the reference's models.py / actor.py pick `cuda` at import "
                    "when a GPU is visible, which initialises CUDA in the launcher (fork start method, "
                    "train.py:42) and makes policy.share_memory() a no-op.  Hide the GPUs from the launcher "
                    "and the actors (CUDA_VISIBLE_DEVICES='' before importing the reference modules; see "
                    "INTEGRATION.md) - this learner restores visibility inside its own process "
                    "(IMPALA_LEARNER_VISIBLE_DEVICES)")
        self.log_path = log_path
        if self.log_path is not None:
            self.log_path = Path(log_path) / Path(f"l{self.id}")
            self.log_path.mkdir(parents=True, exist_ok=False)
        self.evaluator = evaluator  # optional callable(policy) -> (mean_reward, std); see _evaluate
        self._version = mp.Value("q", 0, lock=False)   # published-weights seqlock (shared with the actors)
        self._stage_ring = None
        self.completion = mp.Event()
        self.p = mp.Process(target=self._learn, name=f"learner_{self.id}")
        print(f"[main] learner_{self.id} Initialized")

    # -------------------------------------------------------------- lifecycle (learner.py:55-65)
    def start(self):
        self.completion.clear()
        if len(self.devices) > 1 and not hasattr(self.q, "collect_batch"):
            # data-parallel + reference wire format: rank 0 packs trajectories into a shared-memory
            # staging ring every rank can DMA its shard from (created before the fork)
            from .ring import RingQueue

            O, A, _, _ = _dims(self.policy, self.value_fn)
            self._stage_ring = RingQueue(self.hp.max_timesteps, self.hp.batch_size, O, A, slabs=2)
        self.p.start()
        print(f"[main] Started learner_{self.id} with pid {self.p.pid}")

    def terminate(self):
        self.p.terminate()
        print(f"[main] Terminated learner_{self.id}")

    def join(self):
        self.p.join()
        if self._stage_ring is not None:
            self._stage_ring.close()
            self._stage_ring = None

    # ------------------------------------------------------------------ helpers
    def _cfg(self):
        O, A, H_pi, H_v = _dims(self.policy, self.value_fn)
        hp = self.hp._asdict() if hasattr(self.hp, "_asdict") else dict(self.hp)
        hp["log_path"] = None if hp.get("log_path") is None else str(hp["log_path"])
        return dict(T=self.hp.max_timesteps, B=self.hp.batch_size, O=O, A=A, H_pi=H_pi, H_v=H_v, mode=self.mode, hp=hp)

    def _make_engine(self, process_group=None, world=1):
        from .engine import LearnerEngine

        c = self._cfg()
        if c["B"] % world:
            raise ValueError(f"batch_size {c['B']} does not divide over {world} devices")
        eng = LearnerEngine(c["T"], c["B"] // world, c["O"], c["A"], c["H_pi"], c["H_v"], self.hp,
                            global_batch=c["B"], device=self.device, mode=self.mode, process_group=process_group)
        eng.load_state(self._init_state())
        return eng

    def _init_state(self):
        return {"policy": {k: v.detach().cpu() for k, v in self.policy.state_dict().items()},
                "value_fn": {k: v.detach().cpu() for k, v in self.value_fn.state_dict().items()}}

    def _sync_modules(self, eng, pub):
        """Blocking: everything published so far is visible AND both float64 modules hold the current
        weights (checkpoints, end of run).  The per-update path is `_Publisher.post`."""
        pub.drain()
        st = eng.state()
        with torch.no_grad():
            self._version.value += 1
            for mod, grp in ((self.policy, "policy"), (self.value_fn, "value_fn")):
                for k, t in mod.state_dict().items():
                    t.copy_(st[grp][k].to(t.dtype))
            self._version.value += 1

    @property
    def policy_version(self) -> int:
        """Even: number of completed weight publications x 2; odd: a publication is in progress."""
        return int(self._version.value)

    def policy_snapshot(self):
        """(version, state_dict copy) that is guaranteed not to be torn by a concurrent publication
        (seqlock read; `policy_weights` keeps the reference's lock-free semantics, actor.py:70)."""
        while True:
            v0 = self._version.value
            if v0 & 1:
                continue
            sd = {k: t.clone() for k, t in self.policy.state_dict().items()}
            if self._version.value == v0:
                return v0, sd

    def _evaluate(self, policy):
        """learner.py:195-214 runs utils.test_policy (a gym rollout) inside the update loop.  Here it
        runs on a frozen copy in a background thread: `self.evaluator` if set, else the reference's
        own `utils.test_policy` when this class is deployed inside that repo."""
        if self.evaluator is not None:
            return self.evaluator(policy)
        try:
            import utils as ref_utils  # the reference's utils.py, if on sys.path

            return ref_utils.test_policy(policy, self.hp.env_name, self.hp.eval_eps, True, self.hp.max_timesteps)
        except Exception as e:  # no gym / not inside the reference tree
            print(f"[learner_{self.id}] evaluation skipped: {e!r}")
            return None

    def _start_evaluation(self, writer, n):
        """Evaluate the weights of update n without blocking update n + 1."""
        prev = getattr(self, "_eval_thread", None)
        if prev is not None and prev.is_alive():
            print(f"[learner_{self.id}] update {n}: previous evaluation still running - skipped")
            return
        _, sd = self.policy_snapshot()
        frozen = copy.deepcopy(self.policy)
        frozen.load_state_dict(sd)

        def work():
            res = self._evaluate(frozen)
            if res is None:
                return
            if self.hp.verbose >= 1:
                print(f"[learner_{self.id}] update {n}: evaluation reward {res[0]:.2f} +- {res[1]:.2f}")
            if writer is not None:
                writer.add_scalar(f"learner_{self.id}/rewards/evaluation_reward", res[0], n)

        self._eval_thread = threading.Thread(target=work, name="impala-eval", daemon=True)
        self._eval_thread.start()

    # ---------------------------------------------------------------- the update loop
    def _collect(self, views, writer):
        """Pull hp.batch_size trajectories off the queue into one host slab (learner.py:89-109)."""
        hp = self.hp
        reward = 0.0
        for b in range(hp.batch_size):
            try:
                traj = self.q.get(timeout=self.timeout)
            except queue.Empty:
                print(f"[learner_{self.id}] queue empty for {self.timeout} s - giving up")
                if writer is not None:
                    writer.close()
                self.completion.set()  # lets the actors leave their put() retry loop (actor.py:121)
                raise
            if hp.verbose >= 2:
                print(f"[learner_{self.id}] packing traj_{traj.id} into column {b}")
            reward += pack_trajectory(views, b, traj, hp.max_timesteps) / hp.batch_size
            del traj  # drop the shared-memory handles of its ~5T tensors right away
        return reward

    def _report(self, writer, n, reward, sc):
        """Console line + the five TensorBoard scalars of learner.py:188-192,217-240."""
        if self.hp.verbose >= 1:
            print(f"[learner_{self.id}] update {n}: batch mean reward {reward:.2f}, "
                  f"loss {sc['total_loss']:.2f}")
        if writer is None:
            return
        tag = f"learner_{self.id}"
        for name, val in (("rewards/batch_mean_reward", reward), ("loss/policy_loss", sc["policy_loss"]),
                          ("loss/value_fn_loss", sc["value_fn_loss"]),
                          ("loss/policy_entropy", sc["policy_entropy"]),
                          ("loss/total_loss", sc["total_loss"])):
            writer.add_scalar(f"{tag}/{name}", val, n)

    def _due(self, n) -> bool:
        hp = self.hp
        return ((hp.eval_every is not None and n % hp.eval_every == 0)
                or (self.log_path is not None and n % hp.save_every == 0))

    def _periodic(self, writer, n, eng, pub):
        hp = self.hp
        if hp.eval_every is not None and n % hp.eval_every == 0:          # learner.py:195-214
            pub.drain()
            self._start_evaluation(writer, n)
        if self.log_path is not None and n % hp.save_every == 0:          # learner.py:243-251
            self._sync_modules(eng, pub)
            path = self.log_path / f"IMPALA_{hp.env_name}_l{self.id}_{n}.pt"
            self.save(path)
            print(f"[learner_{self.id}] checkpoint -> {path}")

    def _restore_gpu_visibility(self):
        """The launcher may have hidden the GPUs so that the reference's import-time device choice
        stays on the CPU (see __init__); the learner process gets them back before its first CUDA call."""
        import os

        vis = os.environ.get("IMPALA_LEARNER_VISIBLE_DEVICES")
        if vis is not None:
            os.environ["CUDA_VISIBLE_DEVICES"] = vis

    def _learn(self):
        """Process target (learner.py:67): loop until the shared counter reaches max_updates."""
        writer, pub, leader, eng = None, None, None, None
        try:
            import os

            if os.environ.get("IMPALA_DEBUG_STACKS"):  # dump every thread's stack if the process is still alive then
                import faulthandler

                faulthandler.dump_traceback_later(float(os.environ["IMPALA_DEBUG_STACKS"]), repeat=True, file=sys.stderr)
            # The forked child inherits the launcher's OpenMP state without its worker threads: the first
            # multi-threaded CPU op (e.g. zero-filling a multi-megabyte pinned slab) would wait forever
            # for them.  The learner's host work is tiny copies; one intra-op thread is also the fastest.
            torch.set_num_threads(1)
            self._restore_gpu_visibility()
            world = len(self.devices)
            ring = self.q if hasattr(self.q, "collect_batch") else None  # ring.RingQueue (SURVEY 8f-1)
            stage = self._stage_ring  # data-parallel + mp.Queue: shared staging slabs filled by this process
            pg = None
            if world > 1:
                from . import dp

                slabs = ring if ring is not None else stage
                leader = dp.DpLeader(self.devices, self._cfg(), self._init_state(), slabs.shm.name,
                                     slabs.slab_bytes, slabs.K, timeout=max(60.0, float(self.timeout)))
                torch.cuda.set_device(torch.device(self.device))
                pg = leader.init_process_group(self.device)
            eng = self._make_engine(pg, world)  # first CUDA call of this process (post-fork)
            pub = _Publisher(eng, self.policy, self._version)
            if self.log_path is not None:
                from torch.utils.tensorboard import SummaryWriter

                writer = SummaryWriter(self.log_path)
                writer.add_text("hyperparameters", f"{self.hp}")
            shared = ring if ring is not None else stage
            if shared is not None:
                if world == 1 and shared.slab_bytes != eng.slab_bytes:
                    raise ValueError("RingQueue and learner disagree on (T, B, obs, actions)")
                eng.register_host(shared.slab_address(0), shared.slab_bytes * shared.K)
            if leader is not None:
                leader.wait_ready()
            done, slot, pending, stage_k = 0, 0, None, 0
            eng.loop_stream(True)  # this thread's current stream is the engine's for the whole loop
            # IMPALA_LOOP_STATS=1: where the host time of the update loop goes (printed at the end)
            stats = {"release_wait": 0.0, "collect": 0.0, "enqueue": 0.0, "post": 0.0, "finish": 0.0} \
                if os.environ.get("IMPALA_LOOP_STATS") else None
            clock = time.perf_counter
            to_release = []  # (DMA-done event, ring slab): released one iteration later, off the critical path
            while done < self.hp.max_updates:
                # ---- batch i: collect (host), DMA (copy stream) - the kernels of batch i-1 are running
                # a slab goes back to the actors when its DMA has completed.  Do not WAIT for that here
                # unless the ring would otherwise run dry (or both device slabs' events are in use): the
                # next batch is collected and its DMA queued right behind the running one, so the copy
                # engine never idles for the host part of an iteration (IMPALA_LOOP_STATS=1 shows how long
                # an update still waits here)
                t0 = clock()
                while to_release:
                    ev, kk = to_release[0]
                    if not ev.query() and len(to_release) < min(ring.K - 1, 2):
                        break
                    ev.synchronize()
                    ring.release(kk)
                    to_release.pop(0)
                t1 = clock()
                if ring is not None:
                    try:
                        k, reward = ring.collect_batch(self.timeout)
                    except queue.Empty:
                        print(f"[learner_{self.id}] no trajectory for {self.timeout} s - giving up")
                        self.completion.set()
                        raise
                elif stage is not None:
                    k, stage_k = stage_k, (stage_k + 1) % stage.K
                    reward = self._collect(stage.views(k), writer)
                else:
                    k = None
                    reward = self._collect(eng.host_batch(slot), writer)
                t2 = clock()
                if world > 1:
                    step_no = leader.publish(k)                       # every rank: DMA your shard of slab k
                    eng.ingest_shard_from(shared.slab_address(k), 0, self.hp.batch_size, slot)
                    eng.slab_ready[slot].synchronize()
                    leader.ack_dma(0, step_no)
                    leader.wait_dma(step_no)
                    if ring is not None:
                        ring.release(k)
                elif ring is not None:
                    eng.ingest_from(ring.slab_address(k), slot)   # DMA straight out of shared memory
                    to_release.append((eng.slab_ready[slot], k))  # handed back to the actors once the DMA is done
                else:
                    eng.ingest(slot)
                eng.step(slot)
                t3 = clock()
                n = done + 1
                # the logged scalars: read back when somebody consumes them (TensorBoard / console), else
                # every 64th update (keeps the data-parallel error word checked)
                want_scalars = writer is not None or self.hp.verbose >= 1 or n % 64 == 0 or n >= self.hp.max_updates
                ticket = eng.post_scalars() if want_scalars else None
                due = self._due(n)  # evaluation / checkpoint of exactly update n
                if due and ticket is None:
                    ticket = eng.post_scalars()
                if due or n % self.publish_every == 0 or n >= self.hp.max_updates:
                    pub.post(n, force=due or n >= self.hp.max_updates)
                if pub.error is not None:
                    raise pub.error
                t4 = clock()
                # ---- while update n runs: log update n - 1
                if pending is not None:
                    self._finish_update(writer, eng, pub, *pending)
                    pending = None
                if due:
                    self._finish_update(writer, eng, pub, ticket, n, reward)  # waits for update n
                else:
                    pending = (ticket, n, reward)
                slot ^= 1
                self.update_counter.increment()                            # learner.py:254-255
                done = self.update_counter.value
                if stats is not None:
                    t5 = clock()
                    for key, dt in (("release_wait", t1 - t0), ("collect", t2 - t1), ("enqueue", t3 - t2),
                                    ("post", t4 - t3), ("finish", t5 - t4)):
                        stats[key] += dt
            if stats is not None:
                print(f"[learner_{self.id}] host time per update (us): "
                      + ", ".join(f"{k} {1e6 * v / max(1, done):.1f}" for k, v in stats.items()), file=sys.stderr, flush=True)
            if pending is not None:
                self._finish_update(writer, eng, pub, *pending)
            self._sync_modules(eng, pub)
            t = getattr(self, "_eval_thread", None)
            if t is not None:
                t.join(timeout=600)
            print(f"[learner_{self.id}] done after {done} updates")
            self.completion.set()
        except KeyboardInterrupt:
            print(f"[learner_{self.id}] interrupted")
            self.completion.set()
        except Exception:
            # The reference re-raises without setting `completion` (learner.py:271-275), which
            # leaves train.py:84 waiting forever; here the actors are released as well.
            print(f"[learner_{self.id}] failed")
            self.completion.set()
            raise
        finally:
            if pub is not None:
                pub.close()
            if leader is not None:
                leader.stop()
            if writer is not None:
                writer.close()

    def _finish_update(self, writer, eng, pub, ticket, n, reward):
        if ticket is not None:
            sc = eng.fetch_scalars(ticket)
            self._report(writer, n, reward, sc)
        self._periodic(writer, n, eng, pub)

    # ------------------------------------------------------ checkpoints (learner.py:277-295)
    def save(self, path):
        torch.save({"policy_state_dict": self.policy.state_dict(),
                    "value_fn_state_dict": self.value_fn.state_dict()}, path)

    def load(self, path):
        checkpoint = torch.load(path)
        self.policy.load_state_dict(checkpoint["policy_state_dict"])
        self.value_fn.load_state_dict(checkpoint["value_fn_state_dict"])

    @property
    def policy_weights(self):
        return self.policy.state_dict()


# ----------------------------------------------------------------------------------------------
# Module-level loss helpers with the reference's names, signatures and sign conventions
# (learner.py:298-321), backed by the C ABI.  Inputs are CUDA tensors (any float dtype; the
# kernels compute in float32 and reduce in float64); results come back in the input dtype and
# are differentiable with respect to the logits / advantages exactly where the reference's are.
# ----------------------------------------------------------------------------------------------
def _lib_and_stream():
    import ctypes as C

    from . import _cabi

    return _cabi, _cabi.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream), C


def _cuda_f32(t):
    from . import _cabi

    if not (torch.is_tensor(t) and t.is_cuda):
        raise _cabi.ImpalaCudaError("loss helpers need CUDA tensors (there is no CPU fallback)")
    return t.detach().to(torch.float32).contiguous()


class _PolicyTerms(torch.autograd.Function):
    """(logits, actions) -> (log pi(a), sum_k p_k log p_k) per row."""

    @staticmethod
    def forward(ctx, logits, actions):
        _cabi, lib, st, C = _lib_and_stream()
        z = _cuda_f32(logits).reshape(-1, logits.shape[-1])
        a = actions.detach().reshape(-1).to(torch.int32).contiguous()
        M, A = z.shape
        lp = torch.empty(M, dtype=torch.float32, device=z.device)
        ne = torch.empty(M, dtype=torch.float32, device=z.device)
        _cabi.check(lib.impala_policy_terms(C.c_void_p(z.data_ptr()), C.c_void_p(a.data_ptr()),
                                            C.c_void_p(lp.data_ptr()), C.c_void_p(ne.data_ptr()), M, A, st),
                    "impala_policy_terms")
        ctx.save_for_backward(z, a)
        ctx.in_shape, ctx.in_dtype = logits.shape, logits.dtype
        return lp.to(logits.dtype), ne.to(logits.dtype)

    @staticmethod
    def backward(ctx, g_lp, g_ne):
        _cabi, lib, st, C = _lib_and_stream()
        z, a = ctx.saved_tensors
        M, A = z.shape
        gl = None if g_lp is None else g_lp.to(torch.float32).contiguous()
        gn = None if g_ne is None else g_ne.to(torch.float32).contiguous()
        dz = torch.empty_like(z)
        _cabi.check(lib.impala_policy_terms_backward(
            C.c_void_p(z.data_ptr()), C.c_void_p(a.data_ptr()),
            C.c_void_p(gl.data_ptr()) if gl is not None else None,
            C.c_void_p(gn.data_ptr()) if gn is not None else None,
            C.c_void_p(dz.data_ptr()), M, A, st), "impala_policy_terms_backward")
        return dz.reshape(ctx.in_shape).to(ctx.in_dtype), None


class _Reduce(torch.autograd.Function):
    """float64-accumulated scalar reductions: mode 0 sum(a), 1 0.5*sum(a^2), 2 sum(a*b) (b constant)."""

    @staticmethod
    def forward(ctx, a, b, mode):
        _cabi, lib, st, C = _lib_and_stream()
        af = _cuda_f32(a).reshape(-1)
        bf = _cuda_f32(b).reshape(-1) if b is not None else None
        out = torch.empty(1, dtype=torch.float64, device=af.device)
        _cabi.check(lib.impala_reduce(C.c_void_p(af.data_ptr()),
                                      C.c_void_p(bf.data_ptr()) if bf is not None else None,
                                      af.numel(), mode, C.c_void_p(out.data_ptr()), st), "impala_reduce")
        ctx.mode, ctx.shape, ctx.dtype = mode, a.shape, a.dtype
        ctx.save_for_backward(af, bf if bf is not None else af)
        return out[0].to(a.dtype)

    @staticmethod
    def backward(ctx, g):
        af, bf = ctx.saved_tensors
        if ctx.mode == 0:
            ga = g.to(torch.float32).expand(af.shape)
        elif ctx.mode == 1:
            ga = g.to(torch.float32) * af
        else:
            ga = g.to(torch.float32) * bf
        return ga.reshape(ctx.shape).to(ctx.dtype), None, None


def action_log_probs(policy_logits, actions):
    """log pi(a|x) of the taken actions, shaped like `actions` (learner.py:298-303)."""
    return _PolicyTerms.apply(policy_logits, actions)[0].view_as(actions)


def compute_baseline_loss(advantages):
    """0.5 * sum(advantages ** 2)  (learner.py:306-307)."""
    return _Reduce.apply(advantages, None, 1)


def compute_entropy_loss(logits):
    """The NEGATIVE entropy sum(p * log p), as in the reference (learner.py:310-314)."""
    return _Reduce.apply(_PolicyTerms.apply(logits, torch.zeros(logits.shape[:-1], dtype=torch.int32,
                                                                 device=logits.device))[1], None, 0)


def compute_policy_gradient_loss(logits, actions, advantages):
    """sum(-log pi(a|x) * advantages.detach())  (learner.py:317-321)."""
    lp = _PolicyTerms.apply(logits, actions)[0]
    return _Reduce.apply(lp, -advantages.detach().reshape(-1), 2)
