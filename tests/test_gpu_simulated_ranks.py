"""GPU, one device: the data-parallel learner step with W simulated ranks, through LearnerEngine for every feature, and
the observation-normalization exchange kernels at the C ABI against float64.

The peer route takes every rank's gather buffer as a plain device address (LearnerEngine._use_peers), so W engines on
cuda:0, each with its own zero-filled gather buffer, run the launches, layout, tags, parities and rank-ordered sums of
W GPUs of a node.  What this cannot cover - the IPC mapping, the cross-device timing (tests/test_peer_protocol_model.py
models that), the NCCL route and the forked Learner with its worker ranks - needs two GPUs (tests/multi_gpu_*_check.py).

Harness rules, which keep every consumer from waiting:
  * all W engines live on cuda:0 and every launch goes on ONE stream; step u is every rank's `_enqueue_main(slot)` in
    rank order, then every rank's `_enqueue_opt()`, so no consumer starts before every producer of its step is done;
  * `eng.step()` is never called on a simulated rank with W > 1: its captured graph holds the consumer, which would
    wait for a push enqueued after it (W = 1 may, and does);
  * timeout_s is a few seconds, so a broken build fails in bounded time, and every rank's error word is read after
    every step: a nonzero value is a failure, never retried;
  * the timeout is never provoked: the error paths are exercised by presetting *err = 1, with every slot written;
  * batches reach the ranks as `load_device_batch(synth.shard_batch(batch, r, W))`; no replay (one device by design).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import obs_norm_oracle as onorc
import test_gpu_optim_exchange as ex
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.engine import LearnerEngine
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu

TIMEOUT_S = 5.0
T, B, UPDATES = 20, 48, 3  # W in {1, 2, 3, 8} divides B; three updates cover parities 1, 0, 1
WORLDS = (1, 2, 3, 8)
POPART0 = {"mu": 0.4, "nu": 1.5}


def _lr_lambda(e):
    return 0.95 / (1.0 + e / 4)


# name: (engine options, O, A, H, fused push expected)
CASES = {
    "plain": ({}, 24, 4, 256, True),
    "a6": ({}, 24, 6, 256, False),
    "diag_popart": (dict(diagnostics=True, popart=True, popart_beta=0.1), 24, 4, 256, True),
    "popart_rmsprop": (dict(popart=True, optimizer="rmsprop", optimizer_kwargs=dict(eps=0.01)), 24, 4, 256, True),
    "rclip_paper": (dict(reward_clip="soft_asymmetric"), 24, 4, 256, True),
    "gauss": (dict(action_dist="gaussian", diagnostics=True), 28, 2, 256, True),
    "md": (dict(action_dist="multi_discrete", action_heads=(2, 2)), 24, 4, 256, True),
    "md_mask": (dict(action_dist="multi_discrete", action_heads=(3, 3, 2), action_mask=True), 24, 8, 256, False),
    "mask": (dict(action_mask=True), 24, 4, 256, True),
    "shared_popart": (dict(shared_torso=True, popart=True), 24, 4, 256, False),
    "u8_frames": (dict(obs_dtype="uint8", frames=4), 512, 18, 256, False),
    "obs_norm": (dict(obs_norm=True), 24, 4, 256, True),
    "obs_norm_diag_popart": (dict(obs_norm=True, diagnostics=True, popart=True), 24, 4, 256, True),
    "obs_norm_shared": (dict(obs_norm=True, shared_torso=True), 24, 4, 256, False),
    "obs_norm_u8_frames": (dict(obs_norm=True, obs_dtype="uint8", frames=4), 200, 4, 256, False),
    "obs_norm_1024": (dict(obs_norm=True), 1024, 4, 256, False),
}
ENGINE_KW = {"popart_rmsprop": dict(lr_lambda=_lr_lambda), "rclip_paper": dict(mode="paper")}


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    torch.cuda.set_device(0)
    return _cabi.lib()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bits(t):
    return t.view({torch.float32: torch.int32, torch.float64: torch.int64}.get(t.dtype, t.dtype))


def _same_bits(a, b):
    return a.dtype == b.dtype and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


# ------------------------------------------------------------------------------------------ engine harness
def _obs_stats0(O):
    return {"count": 1000.0, "mean": np.linspace(-2.0, 3.0, O), "var": np.linspace(0.5, 4.0, O)}


def make_batch(case, seed):
    """A ragged batch of the case's kind with two empty columns (lens 0) on different ranks; float32 observations of
    an obs_norm case are scaled per feature (spreads 0.1 to 10, means -50 to 50)."""
    opts, O, A, _, _ = CASES[case]
    frames, heads = opts.get("frames", 1), opts.get("action_heads", ())
    if opts.get("action_dist") == "gaussian":
        b = synth.make_gaussian_batch(seed, T, B, O, A, ragged=True)
    elif opts.get("action_mask"):
        b = synth.make_masked_batch(seed, T, B, O, A, heads, ragged=True)
        b.pop("legal")
    elif heads:
        b = synth.make_md_batch(seed, T, B, O, heads, ragged=True)
    else:
        # byte frames: 0/1 planes (MinAtar) without obs_norm, whole bytes (Atari RAM) with it.  Unnormalized 0..255
        # inputs leave most of the first layer's gradient at float32 sum-order noise (see check_against_one_device)
        kind = ("bytes" if opts.get("obs_norm") else "planes") if opts.get("obs_dtype") == "uint8" else "normal"
        b = synth.make_batch(seed, T, B, O, A, ragged=True, frames=frames, obs_kind=kind)
    b["lens"][[0, B - 1]] = 0
    b["lens"][1] = T
    if opts.get("obs_norm") and b["obs"].dtype == np.float32:
        F = b["obs"].shape[-1]
        b["obs"] = (b["obs"] * np.linspace(0.1, 10.0, F) + np.linspace(-50.0, 50.0, F)).astype(np.float32)
    return b


def make_engine(case, B_local, **kw):
    opts, O, A, H, _ = CASES[case]
    hp = default_hparams(batch_size=B, max_timesteps=T)
    eng = LearnerEngine(T, B_local, O, A, H, H, hp, global_batch=B, **ENGINE_KW.get(case, {}), **kw, **opts)
    init = synth.init_params(3, O, eng.N_pi, H)
    eng.load_state(init, popart=POPART0 if eng.popart else None, obs_norm=_obs_stats0(O) if eng.obs_norm else None)
    return eng


def snapshot(e):
    """Everything an update leaves behind on one rank (the logged scalars: the reduced extras in `comm`)."""
    out = dict(params=e.params, adam_m=e.adam_m, adam_v=e.adam_v, adam_step=e.adam_step, norms=e.norms,
               scalars=e.comm[e.n_total:e.obs_sums_at])
    if e.popart:
        out["popart_buf"] = e.popart_buf
    if e.obs_norm:
        out.update(obs_stats=e.obs_stats, obs_norm_dev=e.obs_norm_dev, folded=e.folded)
    return {k: v.detach().clone() for k, v in out.items()}


class SimRanks:
    """W engines of B / W columns on cuda:0, attached to W gather buffers, stepped in the harness order."""

    def __init__(self, case, W):
        self.W = W
        self.engines = [make_engine(case, B // W) for _ in range(W)]
        nbytes = self.engines[0].gather_bytes(W)
        self.gather = [torch.zeros(nbytes // 8, dtype=torch.int64, device="cuda") for _ in range(W)]
        ptrs = [g.data_ptr() for g in self.gather]
        for r, e in enumerate(self.engines):
            e._use_peers(ptrs[r], ptrs, r, W, timeout_s=TIMEOUT_S)
        self.stream = torch.cuda.Stream()
        torch.cuda.synchronize()

    def load(self, batch):
        for r, e in enumerate(self.engines):
            e.load_device_batch(synth.shard_batch(batch, r, self.W))

    def step(self, batch):
        self.load(batch)
        with torch.cuda.stream(self.stream):
            for e in self.engines:
                e._enqueue_main(0)
            for e in self.engines:
                e._enqueue_opt()
        self.finish()

    def finish(self):
        torch.cuda.synchronize()
        for r, e in enumerate(self.engines):
            assert int(e.peer["err"].item()) == 0, f"rank {r}: a consumer gave up waiting for a slot"

    @property
    def fused(self):
        return {e.peer["fused"] for e in self.engines}


def assert_same_bits(a, b, what):
    for k in a:
        assert _same_bits(a[k], b[k]), (what, k)


def assert_same_values(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), (what, k)


def assert_same_scalars(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert a[k] == b[k] or (np.isnan(a[k]) and np.isnan(b[k])), (what, k, a[k], b[k])


def check_obs_norm(e, run):
    """obs_norm statistics against the float64 oracle over the concatenated valid rows, the float32 statistics
    bitwise theirs, and `folded` the fold of the engine's parameters within float32 rounding."""
    O = e.O
    st = e.obs_stats.cpu().numpy()
    assert st[0] == run.count
    np.testing.assert_allclose(st[1:1 + O], run.mean, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(st[1 + O:], run.var, rtol=1e-12, atol=1e-300)
    mu_f, r_f = onorc.norm_f32(st[1:1 + O], st[1 + O:], e.obs_norm_eps)
    nd = e.obs_norm_dev.cpu().numpy()
    assert np.array_equal(nd.view(np.int32), np.concatenate([mu_f, r_f]).view(np.int32))
    p, f = e.params.cpu().numpy(), e.folded.cpu().numpy()
    rest = np.ones(p.size, bool)
    for w1, b1, H in e.w1_nets:
        W1, b = p[w1:w1 + H * O].reshape(H, O), p[b1:b1 + H]
        Wf, bf = onorc.fold(W1, b, mu_f, r_f)
        assert np.array_equal(f[w1:w1 + H * O].view(np.int32), Wf.astype(np.float32).reshape(-1).view(np.int32))
        tol = np.spacing(np.abs(bf).astype(np.float32)) + 2.0 ** -23 * (np.abs(Wf) @ np.abs(mu_f.astype(np.float64)))
        err = np.abs(f[b1:b1 + H] - bf)
        assert (err <= tol).all(), float((err - tol).max())
        rest[w1:w1 + H * O] = rest[b1:b1 + H] = False
    assert np.array_equal(f[rest].view(np.int32), p[rest].view(np.int32))


def check_against_one_device(e, sc, ref, u):
    """A rank against the one-device engine on the full batch after update u (1-based), within the two-GPU scripts'
    tolerances.  One exception: the float32 sums of the gradient are exact to about 1e-7 of its largest entries, so an
    entry 1e5 times smaller than those (byte-valued or 1024-feature inputs have them) carries sum-order noise of a
    percent or more, and Adam normalizes that into a step of up to lr.  Such entries (sqrt(v) under 1e-5 of the largest
    on the one-device engine) may differ by 2 lr per update after the first, where both start from the same
    parameters.  state() is a function
    of the parameters and the statistics, checked on their own; it is compared where no entry needs the exception."""
    d = (e.params - ref["params"]).abs()
    rms = ref["snap"]["adam_v"].sqrt()
    resolved = rms >= 1e-5 * rms.max()
    assert float(d[resolved].max()) < 2e-5, float(d[resolved].max())
    noise = float(d[~resolved].max()) if (~resolved).any() else 0.0
    assert noise < 2e-5 + 2.0 * 0.95 * e.hp.lr * (u - 1), (noise, int((d >= 2e-5).sum()))
    got_state = e.state() if float(d.max()) < 2e-5 else {}
    for grp in got_state:
        for key in got_state[grp]:
            dd = float((got_state[grp][key] - ref["state"][grp][key]).abs().max())
            assert dd < 2e-5, (grp, key, dd)
    want = ref["scalars"]
    # the clip norms too at update 1, where both start from the same parameters (later, a policy whose gradient has
    # fallen to sum-order noise, as with byte inputs, has a norm of that noise)
    for k in ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward") + (
            ("norm_policy", "norm_value") if u == 1 else ()):
        assert abs(sc[k] - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, sc[k], want[k])
    if e.diagnostics:
        assert sc["valid_steps"] == want["valid_steps"]
    if e.popart:
        got = e.popart_buf.cpu().numpy()
        np.testing.assert_allclose(got[:3], ref["popart"][:3], rtol=0, atol=1e-6)


def _one_device_run(case, batches):
    ref = make_engine(case, B)
    out = []
    for b in batches:
        ref.load_device_batch(b)
        ref.step()
        out.append(dict(scalars=ref.read_scalars(), snap=snapshot(ref), state=ref.state(), params=ref.params.clone(),
                        popart=ref.popart_buf.cpu().numpy() if ref.popart else None))
    return out


# ------------------------------------------------------------------------------------------ engine-level cases
@pytest.mark.parametrize("case", list(CASES))
def test_simulated_ranks(lib, case, monkeypatch):
    """W in {1, 2, 3, 8} simulated ranks, three updates: the route the case names; every rank's error word 0; the
    ranks bitwise equal; W = 1 equal in value to the engine without peers, through the split enqueue and through
    step() (the peer route in one captured graph); the stand-alone push bitwise equal to the fused one; the one-device
    full-batch engine within the two-GPU tolerances; the obs_norm statistics and folded block against float64."""
    opts, O, _, _, want_fused = CASES[case]
    frames = opts.get("frames", 1)
    batches = [make_batch(case, 300 + u) for u in range(UPDATES)]
    ref = _one_device_run(case, batches)
    run = None
    if opts.get("obs_norm"):
        s0 = _obs_stats0(O)
        run = onorc.Running(O)
        run.count, run.mean, run.var = s0["count"], s0["mean"].copy(), s0["var"].copy()
    for W in WORLDS:
        sims = [SimRanks(case, W)]
        assert sims[0].fused == {want_fused}, (case, W, sims[0].fused)
        if W > 1 and want_fused:
            monkeypatch.setenv("IMPALA_PUSH_FUSED", "0")
            sims.append(SimRanks(case, W))
            monkeypatch.delenv("IMPALA_PUSH_FUSED")
            assert sims[1].fused == {False}
        if W == 1:  # the same peer route through step(): eager first, then one graph of main + optimizer
            one = make_engine(case, B)
            g = torch.zeros(one.gather_bytes(1) // 8, dtype=torch.int64, device="cuda")
            one._use_peers(g.data_ptr(), [g.data_ptr()], 0, 1, timeout_s=TIMEOUT_S)
        if run is not None:
            r_w = onorc.Running(O)
            r_w.count, r_w.mean, r_w.var = run.count, run.mean.copy(), run.var.copy()
        for u, batch in enumerate(batches):
            for s in sims:
                s.step(batch)
            e0 = sims[0].engines[0]
            snaps = [snapshot(e) for e in sims[0].engines]
            for r in range(1, W):
                assert_same_bits(snaps[r], snaps[0], (case, W, u, "rank", r))
            for s in sims[1:]:  # stand-alone push: the same bits on every rank
                for r, e in enumerate(s.engines):
                    assert_same_bits(snapshot(e), snaps[r], (case, W, u, "stand-alone push", r))
            if W == 1:
                assert_same_values(snaps[0], ref[u]["snap"], (case, u, "split enqueue"))
                one.load_device_batch(batch)
                one.step()
                one.synchronize()
                assert int(one.peer["err"].item()) == 0
                assert_same_values(snapshot(one), ref[u]["snap"], (case, u, "step()"))
                assert_same_scalars(one.read_scalars(), ref[u]["scalars"], (case, u))
            check_against_one_device(e0, e0.read_scalars(), ref[u], u + 1)
            if run is not None:
                r_w.update(onorc.dense_rows(batch["obs"], T, frames), batch["lens"], T)
                check_obs_norm(e0, r_w)
        print(f"SIMULATED_RANKS {case} W={W} route={'fused' if want_fused else 'stand-alone'}"
              + (" (+ stand-alone, bitwise equal)" if len(sims) > 1 else ""))


@pytest.mark.parametrize("case", ["obs_norm_diag_popart", "obs_norm_shared"])
def test_captured_graphs_replay_in_harness_order(lib, case):
    """W = 8: each rank's main and optimizer enqueues captured once as separate CUDA graphs and replayed in the harness
    order for four steps equal the eager steps bit for bit (seq on the device picks parity and tag)."""
    W = 8
    batches = [make_batch(case, 500 + u) for u in range(4)]
    eager = SimRanks(case, W)
    for b in batches:
        eager.step(b)
    G = SimRanks(case, W)
    assert G.fused == {CASES[case][4]}
    s = G.stream
    mains, opts = [], []
    with torch.cuda.stream(s):
        for e in G.engines:
            for lst, enqueue in ((mains, lambda e=e: e._enqueue_main(0)), (opts, e._enqueue_opt)):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
                    enqueue()
                lst.append(g)
    for b in batches:
        G.load(b)
        with torch.cuda.stream(s):
            for g in mains + opts:
                g.replay()
        G.finish()
    for r in range(W):
        assert_same_bits(snapshot(G.engines[r]), snapshot(eager.engines[r]), (case, r))
        assert _same_bits(G.gather[r], eager.gather[r]), r
        assert int(G.engines[r].peer["seq"].item()) == 4


def test_peers_refuse_replay(lib):
    eng = LearnerEngine(T, B // 2, 24, 4, 64, 64, default_hparams(batch_size=B, max_timesteps=T), global_batch=B,
                        replay_slabs=2, replay_columns=4)
    g = torch.zeros(eng.gather_bytes(2) // 8, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="one device"):
        eng._use_peers(g.data_ptr(), [g.data_ptr()] * 2, 0, 2, timeout_s=TIMEOUT_S)
    assert eng.peer is None and eng.world == 1


# ------------------------------------------------------------------------- obs_norm exchange at the C ABI
def expect_slots(R, before, comms, n, step):
    """Slot r of every rank's buffer at the step's parity holds comms[r][:n] bit for bit, both halves tagged with the
    step; the pad of every slot and the other parity are untouched."""
    par = step & 1
    want_bits = [c.cpu().numpy().view(np.uint64) for c in comms]
    for b in range(R.W):
        got = R.words(b)
        want = before[b].copy()
        for r in range(R.W):
            want[par, r, :n, 0] = (want_bits[r][:n] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            want[par, r, :n, 2] = (want_bits[r][:n] >> np.uint64(32)).astype(np.uint32)
            want[par, r, :n, 1] = want[par, r, :n, 3] = np.uint32(step)
        if not np.array_equal(got, want):
            bad = np.argwhere(got != want)[:5]
            raise AssertionError(f"gather buffer of rank {b} after step {step}: first differing "
                                 f"(parity, slot, element, word) {bad.tolist()}")


@pytest.mark.parametrize("n_extra", [4, 12])
@pytest.mark.parametrize("O", [4, 24, 28])
@pytest.mark.parametrize("W", [1, 3, 8])
def test_fused_push_obs_norm_slots(lib, W, O, n_extra):
    """impala_mlp_backward_pair_push_obs_norm, three steps: slot r of every buffer holds rank r's gradient as
    impala_mlp_backward_pair computes it, then the n_extra + 2 O + 1 extras (past the 32 a single CTA used to write),
    bit for bit and tagged with the step; nothing else moves."""
    net = ex.Net(5, 7, O, 128, 256, 3)
    assert lib.impala_mlp_backward_pair_push_supported(net.M_pi, net.M_vf, O, net.H_pi, net.H_vf, net.A) == 1
    n_ext = n_extra + 2 * O + 1
    R = ex.Ranks(W, net.n_total, n_ext, net.n_pi, net.init_params(O))
    rng = np.random.default_rng(W * 1000 + O * 10 + n_extra)
    for step in (1, 2, 3):
        inputs = [ex.random_inputs(lib, net, rng, n_ext) for _ in range(W)]
        before = R.snapshot()
        comms = [ex.contribution(lib, net, R.params[r], inputs[r], n_ext) for r in range(W)]
        for r in range(W):
            inp, p = inputs[r], R.params[r]
            _cabi.check(lib.impala_mlp_backward_pair_push_obs_norm(
                _p(inp["x"]), _p(p), _p(p[net.n_pi:]), _p(inp["dl"]), _p(inp["dv"]), _p(inp["ws"][0]),
                inp["ws"][0].numel(), _p(inp["ws"][1]), inp["ws"][1].numel(), net.M_pi, net.M_vf, O, net.H_pi,
                net.H_vf, net.A, _p(inp["extra"]), n_extra, _p(R.ptrs), _p(R.seq[r]), R.slot, R.buf, r, W, _st()),
                "impala_mlp_backward_pair_push_obs_norm")
        torch.cuda.synchronize()
        expect_slots(R, before, comms, net.n_total + n_ext, step)
        for s in R.seq:  # what the consumer does once it has read the step
            s.fill_(step)


class ObsNormRanks:
    """W ranks' gather buffers (sums `sums_at` elements into each slot, a pad after them), per-rank seq and the
    update's outputs per rank, next to one local-route copy (gather = NULL) fed the host's rank-ordered sum."""

    def __init__(self, lib, W, O, nets, seed):
        self.lib, self.W, self.O = lib, W, O
        H = 64
        if nets == 2:
            off_pi, n_pi = _cabi.param_layout(O, H, 4)
            off_vf, n_vf = _cabi.param_layout(O, H, 1)
            self.nets = (off_pi[0], off_pi[1], H, n_pi + off_vf[0], n_pi + off_vf[1], H)
            self.n_total = n_pi + n_vf
        else:
            off, self.n_total = _cabi.param_layout(O, H, 5)
            self.nets = (off[0], off[1], H, 0, 0, 0)
        rng = np.random.default_rng(seed)
        self.params = torch.from_numpy(rng.uniform(-0.3, 0.3, self.n_total).astype(np.float32)).cuda()
        self.sums_at = 37
        self.slot = self.sums_at + 2 * O + 1 + 3
        self.buf = W * self.slot
        self.gather = [torch.zeros(2 * self.buf * 2, dtype=torch.int64, device="cuda") for _ in range(W)]
        self.ptrs = torch.tensor([g.data_ptr() for g in self.gather], dtype=torch.int64, device="cuda")
        self.seq = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(W)]
        self.count0, self.mean0, self.var0 = 500.0, rng.uniform(-3.0, 3.0, O), 10.0 ** rng.uniform(-2.0, 2.0, O)
        st = torch.from_numpy(np.concatenate([[self.count0], self.mean0, self.var0]))
        mu_f, r_f = onorc.norm_f32(self.mean0, self.var0, 1e-8)
        nd = torch.from_numpy(np.concatenate([mu_f, r_f]))
        # index W: the local route
        self.stats = [st.cuda() for _ in range(W + 1)]
        self.norm = [nd.cuda() for _ in range(W + 1)]
        self.folded = [torch.zeros(self.n_total, device="cuda") for _ in range(W + 1)]
        self.ctl = [torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(W + 1)]
        self.err = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.step_no = 0

    def update(self, i, sums=None):
        """impala_obs_norm_update of rank i out of its gather buffer, or (i = W) the local route on `sums`."""
        peer = ((None, None, 0, 0, 1, 0, None, 0.0) if i == self.W else
                (_p(self.gather[i]), _p(self.seq[i]), self.slot, self.buf, self.W, self.sums_at, _p(self.err[i]),
                 TIMEOUT_S))
        _cabi.check(self.lib.impala_obs_norm_update(
            _p(self.stats[i]), _p(self.norm[i]), _p(sums) if sums is not None else None, 1e-8, _p(self.params),
            _p(self.folded[i]), self.n_total, self.O, *self.nets, _p(self.ctl[i]), *peer, _st()),
            "impala_obs_norm_update")

    def push(self, rank_sums):
        """Every rank's sums into slot `rank` of every buffer (impala_peer_push at seq = step - 1), then seq = step on
        every rank, as the gather optimizer leaves it."""
        self.step_no += 1
        n = self.sums_at + 2 * self.O + 1
        for r, s in enumerate(rank_sums):
            local = torch.zeros(n, dtype=torch.float64, device="cuda")
            local[:self.sums_at] = torch.arange(self.sums_at, dtype=torch.float64) + 0.5 + r  # what precedes the sums
            local[self.sums_at:] = torch.from_numpy(s)
            _cabi.check(self.lib.impala_peer_push(_p(local), n, _p(self.ptrs), _p(self.seq[r]), self.slot, self.buf,
                                                  r, self.W, _st()), "impala_peer_push")
        torch.cuda.synchronize()
        for s in self.seq:
            s.fill_(self.step_no)

    def step(self, rank_sums):
        """One step: the pushes, every rank's update and the local route on the host's rank-ordered float64 sum.
        Returns the stats, norm and folded of the local route; every rank's are bitwise the same."""
        self.push(rank_sums)
        total = np.zeros(2 * self.O + 1)
        for s in rank_sums:
            total = total + s  # numpy float64 addition rounds like __dadd_rn
        for i in range(self.W):
            self.update(i)
        self.update(self.W, torch.from_numpy(total).cuda())
        torch.cuda.synchronize()
        for i in range(self.W):
            assert int(self.err[i].item()) == 0, i
        for i in range(self.W + 1):
            assert not self.ctl[i].any(), ("ctl left armed", i)
        for i in range(self.W):
            for name in ("stats", "norm", "folded"):
                assert _same_bits(getattr(self, name)[i], getattr(self, name)[self.W]), (name, i, self.step_no)
        return self.stats[self.W].cpu().numpy(), self.norm[self.W].cpu().numpy(), self.folded[self.W].cpu().numpy()


@pytest.mark.parametrize("nets", [2, 1])
@pytest.mark.parametrize("O", [1, 24, 33, 257, 1024])
@pytest.mark.parametrize("W", [1, 2, 3, 8])
def test_obs_norm_update_gather(lib, W, O, nets):
    """impala_obs_norm_update with a gather buffer, four steps (both parities, twice): bitwise the local route on the
    host's rank-ordered float64 sum, including a sum whose value depends on the order; sums of real shards within 1e-12
    of the float64 merge and the fold; zero rows leave the statistics bitwise; a preset *err = 1 leaves statistics,
    norm and folded bitwise untouched; ctl zeroed after every launch."""
    R = ObsNormRanks(lib, W, O, nets, seed=W * 7 + O + nets)
    rng = np.random.default_rng(O * 3 + W)
    # step 1: sums of the shards of a ragged batch
    Tb, Bb = 5, 24
    lens = rng.integers(0, Tb + 1, Bb).astype(np.int32)
    lens[[0, Bb - 1]] = (0, Tb)
    x = onorc.scaled_obs(O + W, Tb, Bb, O, lens).astype(np.float64)
    per = Bb // W
    shard_sums = []
    for r in range(W):
        s1, s2, n = onorc.batch_sums(x[:, r * per:(r + 1) * per], lens[r * per:(r + 1) * per], Tb)
        shard_sums.append(np.concatenate([s1, s2, [n]]))
    stats, norm, folded = R.step(shard_sums)
    S1, S2, N = onorc.batch_sums(x, lens, Tb)
    count, mean, var = onorc.merge(R.count0, R.mean0, R.var0, S1, S2, N)
    assert stats[0] == count == R.count0 + np.minimum(lens, Tb).sum()
    np.testing.assert_allclose(stats[1:1 + O], mean, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(stats[1 + O:], var, rtol=1e-12, atol=1e-300)
    mu_f, r_f = onorc.norm_f32(stats[1:1 + O], stats[1 + O:], 1e-8)
    assert np.array_equal(norm.view(np.int32), np.concatenate([mu_f, r_f]).view(np.int32))
    p = R.params.cpu().numpy()
    rest = np.ones(R.n_total, bool)
    for w1, b1, H in (R.nets[:3], R.nets[3:]):
        if H == 0:
            continue
        Wf, bf = onorc.fold(p[w1:w1 + H * O].reshape(H, O), p[b1:b1 + H], mu_f, r_f)
        assert np.array_equal(folded[w1:w1 + H * O].view(np.int32), Wf.astype(np.float32).reshape(-1).view(np.int32))
        tol = np.spacing(np.abs(bf).astype(np.float32)) + 2.0 ** -23 * (np.abs(Wf) @ np.abs(mu_f.astype(np.float64)))
        assert (np.abs(folded[b1:b1 + H] - bf) <= tol).all()
        rest[w1:w1 + H * O] = rest[b1:b1 + H] = False
    assert np.array_equal(folded[rest].view(np.int32), p[rest].view(np.int32))
    # step 2: feature 0's first sum is 1, 1e17, -1e17 on ranks 0, 1, 2: ((0 + 1) + 1e17) - 1e17 = 0 in rank order,
    # 1 in reverse order
    odd = []
    for r in range(W):
        s = np.concatenate([rng.standard_normal(O) * 10.0, rng.uniform(1.0, 100.0, O) * 100.0, [3.0]])
        if W >= 3:
            s[0] = (1.0, 1e17, -1e17)[r] if r < 3 else 0.0
        odd.append(s)
    before = stats
    stats, _, _ = R.step(odd)
    if W >= 3:  # the batch mean of feature 0 is 0 / (3 W): the merge moves mean_a by -mean_a * n_b / n exactly
        assert stats[1] == before[1] + (0.0 - before[1]) * ((3.0 * W) / (before[0] + 3.0 * W))
    # step 3: zero rows on every rank
    before = R.stats[W].clone()
    norm_before = R.norm[W].clone()
    R.step([np.zeros(2 * O + 1) for _ in range(W)])
    assert _same_bits(R.stats[W], before) and _same_bits(R.norm[W], norm_before)
    # step 4: a preset error word on every rank (the optimizer timed out): nothing moves, the slots are all written
    for i in range(W):
        R.err[i].fill_(1)
        R.folded[i].fill_(7.0)
    keep = [(R.stats[i].clone(), R.norm[i].clone(), R.folded[i].clone()) for i in range(W)]
    R.push([rng.standard_normal(2 * O + 1) ** 2 + 1.0 for _ in range(W)])
    for i in range(W):
        R.update(i)
    torch.cuda.synchronize()
    for i in range(W):
        for got, want in zip((R.stats[i], R.norm[i], R.folded[i]), keep[i]):
            assert _same_bits(got, want), i
        assert not R.ctl[i].any() and int(R.err[i].item()) == 1
        R.err[i].zero_()
    # step 5: the next launch runs as armed
    R.step([np.concatenate([rng.standard_normal(2 * O) ** 2, [2.0]]) for _ in range(W)])
