"""GPU, one device: the optimizer kernels and the peer-memory gradient exchange of the data-parallel learner.

The exchange (include/impala_b200.h, "Data-parallel learners") takes every rank's gather buffer as a plain
device pointer, so W buffers on one device, written by W producer calls and read by W consumer calls in
stream order, run the same code with the same layout, tags, parities and rank-ordered sums as W GPUs of a
node - everything except the cross-device timing (tests/test_peer_protocol_model.py models that).  Every
producer is enqueued before any consumer, so no consumer ever waits; `timeout_s` is a few seconds so a broken
build fails in bounded time through the consumer's error word, which is checked after every step.

Clip + Adam at its edges is compared with a float64 step that starts from the kernel's own float32 state
(`adam_ref`), so the bound covers one step's float32 rounding only, and with torch.nn.utils.clip_grad_norm_ +
torch.optim.Adam for non-finite gradients."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from conftest import PKEYS, Golden
from oracle import impala_oracle as orc
from torched_impala_b200 import _cabi, ops, synth
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu

TIMEOUT_S = 5.0
EPS = 1e-8
# the kernels take float32 betas and keep the running powers of those values in float64
B1, B2 = float(np.float32(0.9)), float(np.float32(0.999))


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
    """Bit pattern of a float tensor (NaN-safe equality); integer tensors as they are."""
    return t.view({torch.float32: torch.int32, torch.float64: torch.int64}.get(t.dtype, t.dtype))


def _same_bits(a, b):
    return a.dtype == b.dtype and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


# ------------------------------------------------------------------------------------------- harness
class Net:
    """Shapes of one learner step: T, B (per rank), O, H_pi, H_vf, A and the parameter layout."""

    def __init__(self, T, B, O, H_pi, H_vf, A):
        self.T, self.B, self.O, self.H_pi, self.H_vf, self.A = T, B, O, H_pi, H_vf, A
        self.M_pi, self.M_vf = T * B, (T + 1) * B
        self.n_pi = _cabi.param_layout(O, H_pi, A)[1]
        self.n_total = self.n_pi + _cabi.param_layout(O, H_vf, 1)[1]

    def init_params(self, seed):
        pi = synth.init_params(seed, self.O, self.A, self.H_pi)["policy"]
        vf = synth.init_params(seed + 1, self.O, 1, self.H_vf)["value_fn"]
        return torch.cat([ops.pack_params(pi), ops.pack_params(vf)])

    def workspaces(self, lib):
        return [torch.zeros(int(lib.impala_mlp_backward_workspace(M, self.O, H, N2)), dtype=torch.uint8,
                            device="cuda")
                for M, H, N2 in ((self.M_pi, self.H_pi, self.A), (self.M_vf, self.H_vf, 1))]


class Ranks:
    """W simulated ranks on cuda:0: every rank's gather buffer (2 parities x W slots x `slot` LL elements of
    16 bytes; `pad` elements at the end of every slot that nothing may write), the device array of their
    addresses and each rank's seq, params, m, v, state, reduced, norms and err."""

    def __init__(self, W, n_total, n_extra, n_policy, params0, pad=3):
        self.W, self.n, self.n_extra, self.n_policy = W, n_total, n_extra, n_policy
        self.slot = n_total + n_extra + pad
        self.buf = W * self.slot
        self.gather = [torch.zeros(2 * self.buf * 2, dtype=torch.int64, device="cuda") for _ in range(W)]
        assert all(g.data_ptr() % 16 == 0 for g in self.gather)
        self.ptrs = torch.tensor([g.data_ptr() for g in self.gather], dtype=torch.int64, device="cuda")
        self.seq = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(W)]
        self.params = [params0.clone() for _ in range(W)]
        self.m = [torch.zeros(n_total, device="cuda") for _ in range(W)]
        self.v = [torch.zeros(n_total, device="cuda") for _ in range(W)]
        self.state = [torch.zeros(3, dtype=torch.int64, device="cuda") for _ in range(W)]
        self.reduced = [torch.zeros(n_total + n_extra, dtype=torch.float64, device="cuda") for _ in range(W)]
        self.norms = [torch.zeros(2, dtype=torch.float64, device="cuda") for _ in range(W)]
        self.err = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(W)]

    # producers
    def push(self, lib, r, local):
        """Stand-alone producer: local[0, n + n_extra) -> slot r of every rank's buffer."""
        _cabi.check(lib.impala_peer_push(_p(local), self.n + self.n_extra, _p(self.ptrs), _p(self.seq[r]), self.slot,
                                         self.buf, r, self.W, _st()), "impala_peer_push")

    def push_fused(self, lib, r, net, inp):
        p = self.params[r]
        _cabi.check(lib.impala_mlp_backward_pair_push(
            _p(inp["x"]), _p(p), _p(p[net.n_pi:]), _p(inp["dl"]), _p(inp["dv"]), _p(inp["ws"][0]),
            inp["ws"][0].numel(), _p(inp["ws"][1]), inp["ws"][1].numel(), net.M_pi, net.M_vf, net.O, net.H_pi,
            net.H_vf, net.A, _p(inp["extra"]) if self.n_extra else None, self.n_extra, _p(self.ptrs),
            _p(self.seq[r]), self.slot, self.buf, r, self.W, _st()), "impala_mlp_backward_pair_push")

    # consumer
    def consume(self, lib, r, max_norm, lr):
        _cabi.check(lib.impala_gather_clip_adam(
            _p(self.params[r]), _p(self.reduced[r]), _p(self.gather[r]), _p(self.seq[r]), self.slot, self.buf,
            self.W, self.n_extra, _p(self.m[r]), _p(self.v[r]), _p(self.state[r]), self.n_policy, self.n,
            float(max_norm), float(lr), B1, B2, EPS, _p(self.norms[r]), _p(self.err[r]), TIMEOUT_S, _st()),
            "impala_gather_clip_adam")

    def words(self, b):
        """Rank b's gather buffer as uint32 (parity, slot, element, [lo32 | step32 | hi32 | step32])."""
        return self.gather[b].cpu().numpy().view(np.uint32).reshape(2, self.W, self.slot, 4)

    def snapshot(self):
        return [self.words(b).copy() for b in range(self.W)]

    def assert_no_error(self):
        for r in range(self.W):
            assert int(self.err[r].item()) == 0, f"rank {r}: the consumer gave up waiting (a slot was never written)"


def contribution(lib, net, params, inp, n_extra):
    """[grad_pi | grad_vf | extra] of one rank through the plain paired backward (the stand-alone producer's
    source, and what the fused push must deliver bit for bit)."""
    comm = torch.zeros(net.n_total + n_extra, dtype=torch.float64, device="cuda")
    _cabi.check(lib.impala_mlp_backward_pair(
        _p(inp["x"]), _p(params), _p(params[net.n_pi:]), _p(inp["dl"]), _p(inp["dv"]), _p(comm),
        _p(comm[net.n_pi:]), _p(inp["ws"][0]), inp["ws"][0].numel(), _p(inp["ws"][1]), inp["ws"][1].numel(),
        net.M_pi, net.M_vf, net.O, net.H_pi, net.H_vf, net.A, _st()), "impala_mlp_backward_pair")
    if n_extra:
        comm[net.n_total:].copy_(inp["extra"])
    return comm


def random_inputs(lib, net, rng, n_extra):
    x = rng.standard_normal((net.M_vf, net.O), dtype=np.float32)
    dl = (rng.standard_normal((net.M_pi, net.A), dtype=np.float32) / net.M_pi).astype(np.float32)
    dv = (rng.standard_normal(net.M_vf, dtype=np.float32) / net.M_vf).astype(np.float32)
    return dict(x=torch.from_numpy(x).cuda(), dl=torch.from_numpy(dl).cuda(), dv=torch.from_numpy(dv).cuda(),
                extra=torch.from_numpy(rng.standard_normal(n_extra)).cuda(), ws=net.workspaces(lib))


def exchange_step(lib, R, net, inputs, fused, max_norm, lr, order=None, check=True):
    """One simulated step: every rank's producer (in `order`), then every rank's consumer.  With `check`, asserts
    what the step must leave behind, bit for bit, and returns the contributions.  The producers' stores are
    checked before any consumer is enqueued: a consumer only ever runs on complete slots."""
    W = R.W
    order = list(range(W)) if order is None else order
    step = int(R.seq[0].item()) + 1 if check else None
    if check:
        before = R.snapshot()
        shadow = dict(p=R.params[0].clone(), m=R.m[0].clone(), v=R.v[0].clone(), state=R.state[0].clone())
    comms = [None] * W
    for r in order:
        if check or not fused:
            comms[r] = contribution(lib, net, R.params[r], inputs[r], R.n_extra)
        if fused:
            R.push_fused(lib, r, net, inputs[r])
        else:
            R.push(lib, r, comms[r])
    if not check:
        for r in range(W):
            R.consume(lib, r, max_norm, lr)
        return None
    torch.cuda.synchronize()
    n = R.n + R.n_extra
    want_bits = [c.cpu().numpy().view(np.uint64) for c in comms]
    par = step & 1
    # producers: slot r of EVERY buffer at this step's parity holds rank r's contribution, both halves tagged
    # with the step; the pad of every slot and the other parity are untouched
    for b in range(W):
        got = R.words(b)
        want = before[b].copy()
        for r in range(W):
            want[par, r, :n, 0] = (want_bits[r] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            want[par, r, :n, 2] = (want_bits[r] >> np.uint64(32)).astype(np.uint32)
            want[par, r, :n, 1] = want[par, r, :n, 3] = np.uint32(step)
        if not np.array_equal(got, want):
            bad = np.argwhere(got != want)[:5]
            raise AssertionError(f"gather buffer of rank {b} after step {step}: first differing "
                                 f"(parity, slot, element, word) {bad.tolist()}")
    for r in range(W):
        R.consume(lib, r, max_norm, lr)
    torch.cuda.synchronize()
    R.assert_no_error()
    # consumer: the rank-ordered float64 sum ((0 + g_0) + g_1) + ..., scalars included, on every rank
    s = np.zeros(n)
    for c in comms:
        s = s + c.cpu().numpy()
    for r in range(W):
        assert np.array_equal(R.reduced[r].cpu().numpy().view(np.uint64), s.view(np.uint64)), r
        assert int(R.seq[r].item()) == step, r
    for name in ("params", "m", "v", "state", "norms"):
        for r in range(1, W):
            assert _same_bits(getattr(R, name)[r], getattr(R, name)[0]), (name, r)
    # ... and the same bits as impala_clip_adam on the reduced gradient with a separate copy of the state
    norms = ops.clip_adam(shadow["p"], R.reduced[0][:R.n].clone(), shadow["m"], shadow["v"], shadow["state"],
                          R.n_policy, max_norm, lr, B1, B2, EPS)
    torch.cuda.synchronize()
    for name, got in (("p", R.params[0]), ("m", R.m[0]), ("v", R.v[0]), ("state", R.state[0])):
        assert _same_bits(got, shadow[name]), name
    assert _same_bits(R.norms[0], norms)
    return comms


# ------------------------------------------------------------------ producers and consumer, bit for bit
FUSED = [(20, 16, 24, 256, 256, 4), (5, 7, 8, 128, 256, 2), (3, 50, 28, 256, 128, 3)]  # Narrow: fused push
STANDALONE = [(5, 16, 64, 512, 512, 4), (5, 16, 24, 256, 256, 6), (3, 16, 128, 128, 128, 4)]  # c5, A = 6, O = 128

CASES = ([("fused", s, W, ne, False) for s in FUSED for W, ne in ((8, 12), (3, 4))]
         + [("fused", FUSED[0], 8, 4, True), ("fused", FUSED[0], 5, 0, True)]
         + [("standalone", s, W, ne, False) for s in STANDALONE for W, ne in ((8, 12), (3, 4))]
         + [("standalone", STANDALONE[0], 7, 4, True)])


@pytest.mark.parametrize("producer,shape,W,n_extra,reverse", CASES)
def test_exchange_is_bit_exact(lib, producer, shape, W, n_extra, reverse):
    """Three steps (parities 1, 0, 1) of W simulated ranks: the push lands exactly in slot `rank` of every
    buffer with both tags, the consumer's rank-ordered sum and update are bit-identical on every rank and to
    impala_clip_adam, whatever order the producers were enqueued in."""
    net = Net(*shape)
    fused = producer == "fused"
    assert lib.impala_mlp_backward_pair_push_supported(net.M_pi, net.M_vf, net.O, net.H_pi, net.H_vf, net.A) == fused
    R = Ranks(W, net.n_total, n_extra, net.n_pi, net.init_params(W))
    rng = np.random.default_rng(W * 100 + n_extra)
    order = list(reversed(range(W))) if reverse else None
    for it in range(3):
        inputs = [random_inputs(lib, net, rng, n_extra) for _ in range(W)]
        exchange_step(lib, R, net, inputs, fused, max_norm=(0.05, 1e3, 1.0)[it], lr=1e-3, order=order)


# --------------------------------------------------------------------------- against the real reference
def _golden_step_inputs(lib, net, params, shard, hp, B_global, n_extra=4):
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in shard.items()}
    x = d["obs"].reshape(-1, net.O).contiguous()
    logits, values = ops.mlp_forward_pair(x, params, params[net.n_pi:], net.M_pi, net.M_vf, net.O, net.H_pi,
                                          net.H_vf, net.A)
    res = ops.vtrace_loss(logits.view(net.T, net.B, net.A), d["beh_logits"], d["actions"], d["rewards"], d["done"],
                          d["lens"], values.view(net.T + 1, net.B), hp, 1.0 / B_global)
    return dict(x=x, dl=res["dlogits"], dv=res["dv"], extra=res["scalars"][:n_extra], ws=net.workspaces(lib))


@pytest.mark.parametrize("name", ["c3_small_fixed", "c3_small_ragged"])
def test_sharded_updates_match_reference(lib, name):
    """W in {1, 2, 3, 4, 8} (where W divides B) ranks, each on its shard with inv_batch = 1 / B: vtrace_loss,
    the fused push of [gradient | 4 loss scalars], the gather - against the parameters the real reference
    learner.py computed (tolerance of test_engine_updates_match_reference)."""
    g = Golden(name)
    c = g.case
    B = c["B"]
    init = g.init_params()
    for W in (1, 2, 3, 4, 8):
        if B % W:
            continue
        net = Net(c["T"], B // W, c["O"], c["H_pi"], c["H_v"], c["A"])
        p0 = torch.cat([ops.pack_params(init["policy"]), ops.pack_params(init["value_fn"])])
        R = Ranks(W, net.n_total, 4, net.n_pi, p0)
        for u in range(g.updates):
            inputs = [_golden_step_inputs(lib, net, R.params[r], synth.shard_batch(g.batch(u), r, W), g.hp, B)
                      for r in range(W)]
            exchange_step(lib, R, net, inputs, True, g.hp.max_norm, 0.95 * g.hp.lr)
            want = g.params_after(u)
            flat = R.params[0].cpu().numpy()
            for grp, base, H, N2 in (("policy", 0, net.H_pi, net.A), ("value_fn", net.n_pi, net.H_vf, 1)):
                got = ops.unpack_grad(torch.from_numpy(flat[base:]), net.O, H, N2)
                for k in PKEYS:
                    d = np.abs(got[k] - want[grp][k]).max()
                    assert d < 2e-5 * (1 + u), (W, u, grp, k, d)
            sc, ref = R.reduced[0][net.n_total:].cpu().numpy(), g.scalars(u)
            for i, k in enumerate(("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward")):
                assert abs(sc[i] - ref[k]) < 1e-5 * (1 + u) * max(1.0, abs(ref[k])), (W, u, k, sc[i], ref[k])


@pytest.mark.parametrize("W", [8, 3])
def test_many_steps_both_parities(lib, W):
    """Eight consecutive steps, a fresh batch each: every step bit-exact as above, and the parameters within
    2e-5 of a single-rank full-batch run (impala_mlp_backward_pair + impala_clip_adam) of the same steps."""
    T, B, O, H, A = 20, 48, 24, 256, 4
    hp = default_hparams(batch_size=B, max_timesteps=T)
    lr = 0.95 * hp.lr
    net, full = Net(T, B // W, O, H, H, A), Net(T, B, O, H, H, A)
    p0 = net.init_params(11)
    R = Ranks(W, net.n_total, 4, net.n_pi, p0)
    ref = dict(p=p0.clone(), m=torch.zeros_like(p0), v=torch.zeros_like(p0),
               state=torch.zeros(3, dtype=torch.int64, device="cuda"))
    for s in range(8):
        batch = synth.make_batch(200 + s, T, B, O, A, ragged=s % 2 == 1)
        inputs = [_golden_step_inputs(lib, net, R.params[r], synth.shard_batch(batch, r, W), hp, B)
                  for r in range(W)]
        exchange_step(lib, R, net, inputs, True, hp.max_norm, lr)
        one = _golden_step_inputs(lib, full, ref["p"], batch, hp, B)
        g = contribution(lib, full, ref["p"], one, 0)
        ops.clip_adam(ref["p"], g, ref["m"], ref["v"], ref["state"], full.n_pi, hp.max_norm, lr, B1, B2, EPS)
        d = float((R.params[0] - ref["p"]).abs().max())
        assert d < 2e-5, (s, d)
    assert int(R.seq[0].item()) == 8 and int(R.state[0][0].item()) == 8


@pytest.mark.parametrize("producer", ["fused", "standalone"])
def test_one_graph_serves_every_step(lib, producer):
    """One step's producer and consumer launches of all 8 ranks captured once into a CUDA graph and replayed for
    four steps (seq on the device picks parity and tag) equal the same steps launched eagerly, bit for bit."""
    W, n_extra = 8, 12
    net = Net(*(FUSED[0] if producer == "fused" else STANDALONE[0]))
    fused = producer == "fused"
    p0 = net.init_params(5)
    rng = np.random.default_rng(5)
    steps = [[random_inputs(lib, net, rng, n_extra) for _ in range(W)] for _ in range(4)]
    eager = Ranks(W, net.n_total, n_extra, net.n_pi, p0)
    for inputs in steps:  # checked: the graph only runs once the eager steps are known to be right
        exchange_step(lib, eager, net, inputs, fused, 1.0, 1e-3)

    G = Ranks(W, net.n_total, n_extra, net.n_pi, p0)
    static = [random_inputs(lib, net, rng, n_extra) for _ in range(W)]
    local = [torch.zeros(net.n_total + n_extra, dtype=torch.float64, device="cuda") for _ in range(W)]
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream, capture_error_mode="thread_local"):
            for r in range(W):
                if fused:
                    G.push_fused(lib, r, net, static[r])
                else:
                    G.push(lib, r, local[r])
            for r in range(W):
                G.consume(lib, r, 1.0, 1e-3)
    for inputs in steps:
        for r in range(W):
            for k in ("x", "dl", "dv", "extra"):
                static[r][k].copy_(inputs[r][k])
            if not fused:  # the stand-alone producer's source, computed outside the graph
                local[r].copy_(contribution(lib, net, G.params[r], inputs[r], n_extra))
        graph.replay()
        torch.cuda.synchronize()
        G.assert_no_error()
    for name in ("params", "m", "v", "state", "norms", "reduced", "seq", "gather"):
        for r in range(W):
            assert _same_bits(getattr(G, name)[r], getattr(eager, name)[r]), (name, r)
    assert int(G.seq[0].item()) == 4


# --------------------------------------------------------------------------------- clip + Adam at its edges
def adam_ref(p, m, v, g, t, n_policy, max_norm, lr):
    """One float64 clip + Adam step from the kernel's float32 state (p, m, v) after t steps, gradient g
    (float64).  Returns p, m, v, the two norms and per-entry error bounds for p, m and v: four float32 ulps
    of |p| plus 2e-6 of the step size lr / (1 - beta1^t) scaled by the size of the terms of the new moment
    relative to the denominator; 4e-7 (m) and 8e-7 (v) of the terms' magnitudes (float32 rounding of
    g, the coefficient and the two products)."""
    p, m, v = (np.asarray(a, np.float64) for a in (p, m, v))
    norms, coefs = [], []
    for lo, hi in ((0, n_policy), (n_policy, len(g))):
        c, nrm = orc.clip_coef([g[lo:hi]], max_norm)
        norms.append(nrm)
        coefs.append(c)
    with np.errstate(invalid="ignore", over="ignore"):
        gc = g * np.where(np.arange(len(g)) < n_policy, coefs[0], coefs[1])
        ma, mb = B1 * m, (1.0 - B1) * gc
        va, vb = B2 * v, (1.0 - B2) * gc * gc
        m2, v2 = ma + mb, va + vb
        step = lr / (1.0 - B1 ** (t + 1))
        denom = np.sqrt(v2) / math.sqrt(1.0 - B2 ** (t + 1)) + EPS
        p2 = p - step * m2 / denom
        tol_p = (4 * np.spacing(np.abs(p2).astype(np.float32)).astype(np.float64)
                 + 2e-6 * step * (1.0 + (np.abs(ma) + np.abs(mb)) / denom))
    return dict(p=p2, m=m2, v=v2, norms=norms, tol_p=tol_p, tol_m=4e-7 * (np.abs(ma) + np.abs(mb)) + 1e-38,
                tol_v=8e-7 * (va + vb) + 1e-38)


def assert_step(got, ref, what):
    for k in ("p", "m", "v"):
        g, w, tol = got[k], ref[k], ref["tol_" + k]
        nan = np.isnan(w)
        assert np.array_equal(np.isnan(g), nan), (what, k, "NaN positions differ")
        err = np.abs(g[~nan] - w[~nan])
        assert (err <= tol[~nan]).all(), (what, k, float(err.max()), int(np.argmax(err - tol[~nan])))
    for got_n, want_n in zip(got["norms"], ref["norms"]):
        assert (math.isnan(got_n) and math.isnan(want_n)) or got_n == want_n or abs(got_n - want_n) <= 1e-9 * want_n, \
            (what, got_n, want_n)


class Opt:
    """impala_clip_adam and impala_gather_clip_adam at W = 1 (fed by impala_peer_push) side by side on copies of
    the same state: they share the arithmetic order, so they must agree bit for bit."""

    def __init__(self, lib, p0, n_policy):
        self.lib, self.n_policy, n = lib, n_policy, p0.numel()
        self.p, self.m, self.v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
        self.state = torch.zeros(3, dtype=torch.int64, device="cuda")
        self.R = Ranks(1, n, 0, n_policy, p0)

    def set_state(self, m, v, state):
        for dst in ((self.m, self.R.m[0], m), (self.v, self.R.v[0], v), (self.state, self.R.state[0], state)):
            dst[0].copy_(dst[2]), dst[1].copy_(dst[2])

    def host(self):
        return dict(p=self.p.cpu().numpy(), m=self.m.cpu().numpy(), v=self.v.cpu().numpy(),
                    t=int(self.state[0].item()))

    def step(self, g, max_norm, lr):
        norms = ops.clip_adam(self.p, g, self.m, self.v, self.state, self.n_policy, max_norm, lr, B1, B2, EPS)
        self.R.push(self.lib, 0, g)
        self.R.consume(self.lib, 0, max_norm, lr)
        torch.cuda.synchronize()
        self.R.assert_no_error()
        R = self.R
        for a, b, name in ((self.p, R.params[0], "params"), (self.m, R.m[0], "m"), (self.v, R.v[0], "v"),
                           (self.state, R.state[0], "state"), (norms, R.norms[0], "norms")):
            assert _same_bits(a, b), f"impala_gather_clip_adam (W = 1) differs from impala_clip_adam in {name}"
        assert np.array_equal(R.reduced[0].cpu().numpy().view(np.uint64), g.cpu().numpy().view(np.uint64))
        return dict(p=self.p.cpu().numpy(), m=self.m.cpu().numpy(), v=self.v.cpu().numpy(),
                    norms=norms.cpu().numpy().tolist())


def _largest_route_size():
    return _cabi.param_layout(1024, 1024, 32)[1] + _cabi.param_layout(1024, 1024, 1)[1]


SIZES = [1, 31, 8191, 8192, 8193, 16383, 16384, 16385, 14144, 69312, "largest"]


@pytest.mark.parametrize("n_total", SIZES)
def test_clip_adam_sizes_and_groups(lib, n_total):
    """Around the register / strided-loop boundary (2 x 8 x 1024 entries), the c4 and c5 sizes and the largest
    parameter vector the route table allows; empty, one-entry and warp-split groups; two steps each."""
    n = _largest_route_size() if n_total == "largest" else n_total
    rng = np.random.default_rng(n)
    for n_policy in sorted({0, 1, min(n, 17), n - 1, n}):
        p0 = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).cuda()
        opt = Opt(lib, p0, n_policy)
        for it, (scale, max_norm) in enumerate(((1.0, 0.3), (1e-3, 10.0))):
            g = rng.standard_normal(n) * scale
            before = opt.host()
            ref = adam_ref(before["p"], before["m"], before["v"], g, before["t"], n_policy, max_norm, 0.05)
            assert_step(opt.step(torch.from_numpy(g).cuda(), max_norm, 0.05), ref, (n, n_policy, it))
        assert int(opt.state[0].item()) == 2


@pytest.mark.parametrize("regime", ["below", "far_above", "zero_gradient", "one_zero_group"])
def test_clip_regimes(lib, regime):
    n, n_policy, max_norm = 20000, 9000, 1.0
    rng = np.random.default_rng(1)
    p0 = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).cuda()
    opt = Opt(lib, p0, n_policy)
    opt.step(torch.from_numpy(rng.standard_normal(n) * 0.01).cuda(), max_norm, 0.01)  # nonzero m and v
    g = rng.standard_normal(n) * {"below": 1e-3, "far_above": 1e3}.get(regime, 1.0)
    if regime == "zero_gradient":
        g[:] = 0.0
    if regime == "one_zero_group":
        g[:n_policy] = 0.0
    before, state_before = opt.host(), opt.state.clone()
    ref = adam_ref(before["p"], before["m"], before["v"], g, before["t"], n_policy, max_norm, 0.01)
    got = opt.step(torch.from_numpy(g).cuda(), max_norm, 0.01)
    assert_step(got, ref, regime)
    if regime == "below":  # coefficient exactly 1: the same bits as a step that cannot clip
        assert max(ref["norms"]) + 1e-6 < max_norm
        twin = Opt(lib, torch.from_numpy(before["p"]).cuda(), n_policy)
        twin.set_state(torch.from_numpy(before["m"]).cuda(), torch.from_numpy(before["v"]).cuda(), state_before)
        unclipped = twin.step(torch.from_numpy(g).cuda(), 1e30, 0.01)
        for k in ("p", "m", "v"):
            assert np.array_equal(unclipped[k].view(np.int32), got[k].view(np.int32)), k
    if regime == "far_above":
        assert min(ref["norms"]) > 100 * max_norm
    if regime == "zero_gradient":  # momentum only
        assert got["norms"] == [0.0, 0.0]
        np.testing.assert_array_equal(got["m"], (np.float32(B1) * before["m"]).astype(np.float32))
    if regime == "one_zero_group":
        assert got["norms"][0] == 0.0 and got["norms"][1] > 0.0


def test_clip_adam_long_run(lib):
    """3000 steps: the running powers are the only record of the step count."""
    n, n_policy, steps, max_norm, lr = 5000, 1234, 3000, 1.0, 0.01
    gen = torch.Generator(device="cuda").manual_seed(7)
    scale = torch.tensor([(3.0, 0.01, 0.3)[s % 3] for s in range(steps)], dtype=torch.float64, device="cuda")
    grads = torch.randn(steps, n, dtype=torch.float64, device="cuda", generator=gen) * scale[:, None]
    p0 = torch.randn(n, device="cuda", generator=gen)
    opt = Opt(lib, p0, n_policy)
    sampled = {1, 2, 3, 50, 1000, 2998, 2999, 3000}
    for s in range(1, steps + 1):
        if s in sampled:
            before = opt.host()
            g = grads[s - 1].cpu().numpy()
            ref = adam_ref(before["p"], before["m"], before["v"], g, before["t"], n_policy, max_norm, lr)
            assert_step(opt.step(grads[s - 1], max_norm, lr), ref, s)
        else:
            ops.clip_adam(opt.p, grads[s - 1], opt.m, opt.v, opt.state, n_policy, max_norm, lr, B1, B2, EPS)
            opt.R.push(lib, 0, grads[s - 1])
            opt.R.consume(lib, 0, max_norm, lr)
    torch.cuda.synchronize()
    opt.R.assert_no_error()
    st = opt.state.cpu()
    assert int(st[0]) == steps
    p1, p2 = st[1:].view(torch.float64).tolist()
    assert abs(p1 - B1 ** steps) <= 1e-12 * B1 ** steps and abs(p2 - B2 ** steps) <= 1e-12 * B2 ** steps
    assert torch.equal(opt.R.state[0], opt.state) and _same_bits(opt.R.params[0], opt.p)


def test_clip_adam_resumes_from_state(lib):
    """A state written from outside - (t, beta1^t, beta2^t) with nonzero m and v - continues as the oracle's
    Adam does from step t."""
    n, n_policy, t, max_norm, lr = 14144, 6144, 500, 10.0, 0.01
    rng = np.random.default_rng(500)
    p0 = rng.standard_normal(n).astype(np.float32)
    m0 = (rng.standard_normal(n) * 0.01).astype(np.float32)
    v0 = (rng.random(n) * 1e-4).astype(np.float32)
    opt = Opt(lib, torch.from_numpy(p0).cuda(), n_policy)
    state = torch.tensor([t, 0, 0], dtype=torch.int64)
    state[1:] = torch.tensor([B1 ** t, B2 ** t], dtype=torch.float64).view(torch.int64)
    opt.set_state(torch.from_numpy(m0).cuda(), torch.from_numpy(v0).cuda(), state.cuda())
    g = rng.standard_normal(n) * 0.1
    got = opt.step(torch.from_numpy(g).cuda(), max_norm, lr)
    ref = adam_ref(p0, m0, v0, g, t, n_policy, max_norm, lr)
    assert_step(got, ref, "resume")
    # the oracle's Adam (python betas 0.9 / 0.999) continuing from t
    params = [p0[:n_policy].astype(np.float64), p0[n_policy:].astype(np.float64)]
    adam = orc.Adam(params, lr / 0.95)
    adam.t, adam.m, adam.v = t, [m0[:n_policy].astype(np.float64), m0[n_policy:].astype(np.float64)], \
        [v0[:n_policy].astype(np.float64), v0[n_policy:].astype(np.float64)]
    c0, _ = orc.clip_coef([g[:n_policy]], max_norm)
    c1, _ = orc.clip_coef([g[n_policy:]], max_norm)
    adam.step(params, [g[:n_policy] * c0, g[n_policy:] * c1])
    # the oracle's betas are the python floats: 1 - beta1 is 2.4e-7 and 1 - beta2 1.3e-5 (relative) apart from the
    # float32 ones the kernel takes, which moves the denominator, hence the update, by up to 6.5e-6 of itself
    assert (np.abs(got["p"] - np.concatenate(params)) <= ref["tol_p"] + 1e-5 * np.abs(ref["p"] - p0)).all()
    assert (np.abs(got["m"] - np.concatenate(adam.m)) <= 2 * ref["tol_m"]).all()
    assert int(opt.state[0].item()) == t + 1


@pytest.mark.parametrize("kind,where", [("nan", 5), ("nan", 19000), ("nan", 16500), ("inf", 12000), ("inf", 3)])
def test_non_finite_gradients_match_torch(lib, kind, where):
    """A NaN entry makes every parameter, m and v of its group NaN (torch.clamp keeps the NaN coefficient) and
    the norm NaN, the other group is unaffected; an infinite entry clips its group by 0 (that entry NaN).
    Against torch.nn.utils.clip_grad_norm_ per group + torch.optim.Adam in float64 on the CPU."""
    n, n_policy, max_norm, lr = 20000, 9000, 1.0, 0.01
    rng = np.random.default_rng(where)
    p0 = rng.standard_normal(n).astype(np.float32)
    grads = [rng.standard_normal(n) * 0.5, rng.standard_normal(n) * 0.5]
    grads[1][where] = np.nan if kind == "nan" else np.inf
    opt = Opt(lib, torch.from_numpy(p0).cuda(), n_policy)
    tp = [torch.tensor(p0[:n_policy], dtype=torch.float64, requires_grad=True),
          torch.tensor(p0[n_policy:], dtype=torch.float64, requires_grad=True)]
    adam = torch.optim.Adam(tp, lr=lr, betas=(0.9, 0.999), eps=EPS, foreach=False)
    for g in grads:
        tp[0].grad = torch.tensor(g[:n_policy])
        tp[1].grad = torch.tensor(g[n_policy:])
        tn = [float(torch.nn.utils.clip_grad_norm_([t], max_norm)) for t in tp]
        adam.step()
        before = opt.host()
        ref = adam_ref(before["p"], before["m"], before["v"], g, before["t"], n_policy, max_norm, lr)
        got = opt.step(torch.from_numpy(g).cuda(), max_norm, lr)
        assert_step(got, ref, (kind, where))
    bad = int(where >= n_policy)
    sl = [slice(0, n_policy), slice(n_policy, n)]
    assert math.isnan(got["norms"][bad]) if kind == "nan" else math.isinf(got["norms"][bad])
    assert math.isfinite(got["norms"][1 - bad]) and got["norms"][1 - bad] == pytest.approx(tn[1 - bad], rel=1e-9)
    for key, want in (("p", [t.detach().numpy() for t in tp]),
                      ("m", [adam.state[t]["exp_avg"].numpy() for t in tp]),
                      ("v", [adam.state[t]["exp_avg_sq"].numpy() for t in tp])):
        for grp in (0, 1):
            gk, w = got[key][sl[grp]].astype(np.float64), want[grp]
            assert np.array_equal(np.isnan(gk), np.isnan(w)), (key, grp)
            if kind == "nan" and grp == bad:
                assert np.isnan(gk).all(), (key, grp)
            ok = ~np.isnan(w)
            if not ok.any():
                continue
            # torch's betas are the python floats: 1 - beta2 is 1.3e-5 (relative) away from the float32 one
            scale = np.abs(w[ok]).max()
            tol = {"p": 1e-5 * lr + 2e-6 * scale, "m": 2e-6 * scale, "v": 2e-5 * scale}[key]
            assert np.abs(gk[ok] - w[ok]).max() <= tol, (key, grp)
