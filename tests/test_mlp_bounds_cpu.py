"""CPU: the float64 error bound of tests/mlp_bounds.py fails wrong kernels and passes a float32 one.

Every case of every MLP shape list of the GPU tests is rebuilt from that test's own seeded inputs.  Exact float64
results with one defect each - the kind a tiling, tail, masking or precision bug in a kernel produces - must fail
the test's check (the bound together with the precision floor the test uses):

- a 16-row slab omitted (the last 16 rows, every M);
- batch row M-1 omitted, row 0 omitted, the first row of the last 64-row tile omitted, row M-1 counted twice.
  Only at M <= 21504: one row is about 1/M of a gradient entry while the bound grows like sqrt(M); at M = 60001
  a single row moves the entries by 0.03 to 1.7 of their bound, depending on the row's magnitudes, so a single
  lost row is not always resolvable there (a 16-row slab still is, at every M);
- feature O-1 ignored; the last hidden unit dropped (the last one some row activates);
- one ReLU that is not a tie flipped: the pair whose flip moves an entry most relative to its bound, so the
  easiest flip to detect, not a typical one;
- a GEMM operand at TF32 precision: W1 in the forward (3xTF32 without its x * W1_lo term), every operand of the
  forward, and every operand of the backward (dout, W2, DP, x, h);
- b2 missing in the forward (not on raw 0..255 byte rows: their outputs are of order 1e2, and |b2| <= 1/sqrt(H)
  is below float32 resolution there).

A float32 model of a kernel - sequential float32 sums over features and hidden units, the batch in 132 partial
rows of 32-row tiles each summed sequentially in float32, the partials combined in float64 - passes with at least
10x margin.
"""
import numpy as np
import pytest
import torch

import test_gpu_actions_mid as mid
import test_gpu_bwd_blocks as blocks
import test_gpu_mlp_corners as corners
import test_gpu_obs_wide as obs
import test_gpu_parity as parity
import test_gpu_wide_shapes as wide
from mlp_bounds import FWD_ATOL, GRAD_REL, PKEYS, MlpBound, within

ONE_ROW_MAX_M = 21504


def _forward_cases():
    """name -> (inputs, the test's forward floor scaled by max(1, max |out|)?)"""
    for M, O, H, N2 in parity.MLP_SHAPES + wide.WIDE_MLP_SHAPES + mid.SHAPES:
        yield f"{M},{O},{H},{N2}", (lambda M=M, O=O, H=H, N2=N2: parity.forward_case(M, O, H, N2), False)
    for M, O, H, N2 in obs.OBS_SHAPES:
        for kind in obs.INPUTS:
            yield f"obs {M},{O},{H},{N2} {kind}", (
                lambda M=M, O=O, H=H, N2=N2, k=kind: obs.forward_case(M, O, H, N2, k), False)
    for name, case in corners.FORWARD_CASES.items():
        yield f"corner {name}", (lambda case=case: corners.make_case(case)[:2], True)


def _backward_cases():
    """name -> (inputs, the test's backward floor)"""
    for shapes, rel in ((parity.BWD_SHAPES + wide.WIDE_MLP_SHAPES, GRAD_REL), (mid.SHAPES, mid.REL)):
        for M, O, H, N2 in shapes:
            yield f"{M},{O},{H},{N2}", (lambda M=M, O=O, H=H, N2=N2: parity.backward_case(M, O, H, N2), rel)
    for M, O, H, N2 in obs.OBS_SHAPES:
        for kind in obs.INPUTS:
            yield f"obs {M},{O},{H},{N2} {kind}", (
                lambda M=M, O=O, H=H, N2=N2, k=kind: obs.backward_case(M, O, H, N2, k), GRAD_REL)
    for shape in blocks.PAIR_SHAPES:
        for i, net in enumerate(("policy", "value")):
            yield f"pair {shape} {net}", (lambda shape=shape, i=i: blocks.pair_cases(*shape)[i], GRAD_REL)
    for M, O, H, N2 in blocks.SINGLE_SHAPES:
        yield f"single {M},{O},{H},{N2}", (lambda M=M, O=O, H=H, N2=N2: blocks.single_case(M, O, H, N2), GRAD_REL)
    for name, case in corners.BACKWARD_CASES.items():
        yield f"corner {name}", (lambda case=case: corners.make_case(case), GRAD_REL)


FORWARD = dict(_forward_cases())
BACKWARD = dict(_backward_cases())


def _exact(x, w1, b1, w2, b2, dout=None):
    """Forward output and (given dout) the four gradients in float64."""
    pre = x @ w1.T + b1
    h = pre.clamp_min(0.0)
    out = h @ w2.T + b2
    if dout is None:
        return out, None
    dp = (dout @ w2) * (pre > 0)
    return out, (dp.T @ x, dp.sum(0), dout.T @ h, dout.sum(0))


def tf32(a):
    """a rounded to TF32 (10 explicit mantissa bits, to nearest), as float64."""
    bits = a.to(torch.float32).contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32).to(torch.float64)


def _unit_dropped(b):
    """W1 and b1 without the last hidden unit that any row activates (dropping a unit that is dead on every
    row changes nothing)."""
    j = int(torch.nonzero((b.pre > 0).any(dim=0)).max())
    w1, b1 = b.w1.clone(), b.b1.clone()
    w1[j], b1[j] = 0.0, 0.0
    return w1, b1


def _forward_defects(b):
    x0 = b.x.clone()
    x0[:, -1] = 0.0
    yield "feature O-1 ignored", _exact(x0, b.w1, b.b1, b.w2, b.b2)[0]
    yield "last hidden unit dropped", _exact(b.x, *_unit_dropped(b), b.w2, b.b2)[0]
    if not b.raw_bytes:
        yield "b2 missing", b.out - b.b2
    # 3xTF32 with its x * W1_lo term missing: W1 at TF32 precision; and a plain 1xTF32 forward
    yield "W1 at TF32 precision", _exact(b.x, tf32(b.w1), b.b1, b.w2, b.b2)[0]
    h = (tf32(b.x) @ tf32(b.w1).T + b.b1).clamp_min(0.0)
    yield "1xTF32 forward", tf32(h) @ tf32(b.w2).T + b.b2


def _rows(b, rows, sign):
    dp = b.dh[rows] * (b.pre[rows] > 0)
    return tuple(sign * d for d in (dp.T @ b.x[rows], dp.sum(0), b.dout[rows].T @ b.h[rows], b.dout[rows].sum(0)))


def _flip(b):
    """The gradients with the ReLU of one untied pair (m, j) switched.  The pair is the easiest one to detect: the
    untied pair whose flip moves db1[j] or W1[j, k] (k the largest |x[m, k]|) most relative to that entry's
    bound.  So this shows that the check can see a single flipped ReLU, not that it sees a typical one."""
    tied = b.pre.abs() < b.e_pre
    adh = b.dh.abs()
    kstar = b.x.abs().argmax(dim=1)
    score_w = adh * b.x.abs().gather(1, kstar[:, None]) / b.e_grad[0][:, kstar].T
    score = torch.maximum(score_w, adh / b.e_grad[1]).masked_fill(tied, -1.0)
    m, j = divmod(int(score.argmax()), b.H)
    act = 1.0 if b.pre[m, j] > 0 else 0.0
    sign = 1.0 - 2.0 * act  # +1: the unit switches on, -1: off
    d = sign * b.dh[m, j]
    dw1 = torch.zeros_like(b.grad[0])
    db1 = torch.zeros_like(b.grad[1])
    dw2 = torch.zeros_like(b.grad[2])
    dw1[j] = d * b.x[m]
    db1[j] = d
    dw2[:, j] = sign * b.dout[m] * b.pre[m, j]
    return dw1, db1, dw2, torch.zeros_like(b.grad[3])


def _backward_defects(b):
    M = b.M
    add = lambda delta: tuple(g + d for g, d in zip(b.grad, delta))  # noqa: E731
    yield "last 16-row slab omitted", add(_rows(b, slice(max(0, M - 16), M), -1.0))
    if M <= ONE_ROW_MAX_M:
        yield "row M-1 omitted", add(_rows(b, slice(M - 1, M), -1.0))
        yield "row 0 omitted", add(_rows(b, slice(0, 1), -1.0))
        r = 64 * ((M - 1) // 64)
        yield "first row of the last 64-row tile omitted", add(_rows(b, slice(r, r + 1), -1.0))
        yield "row M-1 counted twice", add(_rows(b, slice(M - 1, M), 1.0))
    x0 = b.x.clone()
    x0[:, -1] = 0.0
    yield "feature O-1 ignored", _exact(x0, b.w1, b.b1, b.w2, b.b2, b.dout)[1]
    yield "last hidden unit dropped", _exact(b.x, *_unit_dropped(b), b.w2, b.b2, b.dout)[1]
    yield "one untied ReLU flipped", add(_flip(b))
    # every GEMM operand at TF32 precision, float64 sums
    dout, w2, x, h = tf32(b.dout), tf32(b.w2), tf32(b.x), tf32(b.h)
    dp = tf32((dout @ w2) * (b.pre > 0))
    yield "1xTF32 backward", (dp.T @ x, dp.sum(0), dout.T @ h, dout.sum(0))


@pytest.mark.parametrize("name", list(FORWARD))
def test_bound_fails_wrong_forward(name):
    make, scaled = FORWARD[name]
    x, p = make()
    b = MlpBound(x, p, device="cpu")
    # outputs of raw 0..255 rows are of order 1e2, where |b2| <= 1 / sqrt(H) is below float32 resolution
    b.raw_bytes = x.dtype == np.uint8
    assert within(b.forward_errors(b.out, FWD_ATOL, scaled))
    for defect, out in _forward_defects(b):
        rep = b.forward_errors(out, FWD_ATOL, scaled)
        assert not within(rep), (defect, rep)


@pytest.mark.parametrize("name", list(BACKWARD))
def test_bound_fails_wrong_backward(name):
    make, rel = BACKWARD[name]
    x, p, dout = make()
    b = MlpBound(x, p, dout, device="cpu")
    assert within(b.backward_errors(b.grad, rel))
    caught = {}
    for defect, grad in _backward_defects(b):
        rep = b.backward_errors(grad, rel)
        caught[defect] = max(v for k, v in rep.items() if k not in ("ties", "pad"))
    print(name, {k: round(v, 2) for k, v in caught.items()})
    assert all(v > 1.0 for v in caught.values()), caught


def fp32_model(x, p, dout, act=None, parts=132, rows=32):
    """A kernel in float32 on the CPU: every dot product a sequential float32 sum; the batch in 32-row tiles
    dealt round-robin to `parts` partial rows, each a sequential float32 sum, combined in float64.  `act`: a
    (tied, active) pair of (M, H) masks that overrides the ReLU decision at the tied pairs."""
    f = np.float32
    x = np.asarray(x, f)
    w1, b1, w2, b2 = (np.asarray(p[k], f) for k in PKEYS)
    dout = np.asarray(dout, f)
    M, O = x.shape
    H, N2 = w1.shape[0], w2.shape[0]
    acc = np.zeros((M, H), f)
    for k in range(O):
        acc += x[:, k:k + 1] * w1[:, k]
    pre = acc + b1
    h = np.maximum(pre, f(0))
    acc = np.zeros((M, N2), f)
    for j in range(H):
        acc += h[:, j:j + 1] * w2[:, j]
    out = acc + b2
    dh = np.zeros((M, H), f)
    for n in range(N2):
        dh += dout[:, n:n + 1] * w2[n]
    on = pre > 0
    if act is not None:
        on = np.where(act[0], act[1], on)
    dp = dh * on
    tiles = (M + rows - 1) // rows
    order = [[r for t in range(c, tiles, parts) for r in range(t * rows, min(M, (t + 1) * rows))]
             for c in range(min(parts, tiles))]
    L = max(map(len, order))
    idx = np.array([o + [M] * (L - len(o)) for o in order])  # row M: a zero row
    xz, dpz, hz, dz = (np.concatenate([a, np.zeros((1, a.shape[1]), f)]) for a in (x, dp, h, dout))
    g = [np.zeros((len(order), H, O), f), np.zeros((len(order), H), f), np.zeros((len(order), N2, H), f),
         np.zeros((len(order), N2), f)]
    for i in range(L):
        r = idx[:, i]
        g[0] += dpz[r][:, :, None] * xz[r][:, None, :]
        g[1] += dpz[r]
        g[2] += dz[r][:, :, None] * hz[r][:, None, :]
        g[3] += dz[r]
    return out, [a.astype(np.float64).sum(0) for a in g]


@pytest.mark.parametrize("M,O,H,N2", [(5, 128, 128, 32), (97, 32, 128, 16), (1000, 24, 256, 32), (4097, 24, 256, 4),
                                      (20480, 128, 256, 18), (86016, 24, 256, 1)])
def test_float32_model_passes_with_margin(M, O, H, N2):
    """The float32 model within the bound, and within a tenth of it where it takes the float64 ReLU decision at
    the ties: a tie the model switches the other way moves W1 / b1 by exactly the tie allowance."""
    x, p, dout = parity.backward_case(M, O, H, N2)
    b = MlpBound(x, p, dout, device="cpu")
    out, grad = fp32_model(x, p, dout)
    rep = {**b.forward_errors(out, FWD_ATOL), **b.backward_errors(grad, GRAD_REL)}
    assert within(rep), rep
    tied = (b.pre.abs() < b.e_pre).numpy()
    out, grad = fp32_model(x, p, dout, act=(tied, (b.pre > 0).numpy()))
    rep = {**b.forward_errors(out), **b.backward_errors(grad)}
    print(M, O, H, N2, rep)
    assert all(v <= 0.1 for k, v in rep.items() if k != "ties"), rep
