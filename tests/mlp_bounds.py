"""Float64 reference of the two-layer MLP with an error bound for every output and gradient entry.

The MLP kernels (Narrow, Wide, Obs on the tensor cores in 3xTF32, FP32 on the CUDA cores) compute in float32 with
different summation orders.  A tolerance relative to the largest entry of a tensor hides a wrong kernel in the
entries that are small: a W1 row that misses a few batch rows can stay inside it.  This module gives each entry
its own bound from the magnitudes that enter it, in the style of a running-error analysis with u = 2^-24:

    pre   = x W1^T + b1           e_pre = lam u sqrt(O+1) (|x| |W1|^T + |b1|)
    out   = h W2^T + b2           e_out = lam u sqrt(H+1) ((|h| + e_pre) |W2|^T + |b2|) + e_pre |W2|^T
    dh    = dout W2               e_dh  = lam u sqrt(N2) |dout| |W2|
    DP    = dh [pre > 0]
    dW2   = dout^T h              e_dW2 = lam u sqrt(M+32) |dout|^T (|h| + e_pre) + |dout|^T e_pre
    db2   = sum dout              e_db2 = lam u sqrt(M+32) sum |dout|
    dW1   = DP^T x                e_dW1 = lam u sqrt(M+32) (|DP| + e_dh)^T |x| + e_dh^T |x|
    db1   = sum DP                e_db1 = lam u sqrt(M+32) sum (|DP| + e_dh) + sum e_dh

A pair (m, j) is a ReLU tie when |pre[m, j]| < e_pre[m, j]: float32 may switch that unit either way, so the pair
adds |dh[m, j]| |x[m, :]| to the bound of W1 row j and |dh[m, j]| to that of b1[j], and nothing elsewhere.  An
exact pre-activation (e_pre = 0, e.g. a zero row and a zero bias) is never a tie: it must take torch's
relu'(0) = 0.  An entry passes when |got - want| <= e; an entry with e = 0 must be exact.

The bound sums worst cases, so on its own it is loose about precision: a forward or backward computed at TF32
precision stays inside it at several shapes.  The checks therefore also hold precision floors (FWD_ATOL on the
forward, GRAD_REL on W2, b2 and the W1 / b1 rows of hidden units without a tie), which such a kernel misses by
3x or more (tests/test_mlp_bounds_cpu.py).

The batch sums take sqrt(M + 32) rather than sqrt(M): the tensor-core kernels split each float32 operand into two
TF32 halves (3xTF32), which leaves every product with an error of a few u however short the sum; with sqrt(M)
the narrow backward used half of the bound at M = 1.  No family's err / e grows with the reduction length (the W1
ratios are largest at M <= 5 and below 0.005 from M = 1000 up), so none needs a linear-n term.

LAM = 8 leaves at least 4x headroom on every kernel family.  Worst err / e on one H100 80GB HBM3 (700 W) over the
shape lists of the GPU MLP tests and the engine checks (W1 / b1: over the hidden units without a tie; the entries
of a tie that float32 switches use about all of their allowance, by construction), then the worst share of the
floors:

    family       out     W1      b1      W2      b2      floors
    Narrow       0.019   0.20*   0.030   0.036   0.004   0.15
    Wide, 1 KA   0.010   0.16*   0.023   0.024   0.007   0.031
    Wide, 2 KA   0.003   0.14*   0.037   0.029   0.011   0.053
    Wide, 4 KA   0.003   0.076   0.026   0.031   0.026   0.051
    Obs          0.003   0.065   0.021   0.004   0.036   0.029
    FP32         0.020   0.042   0.032   0.025   0.026   0.11
    engine, pair 0.004   0.11    0.015   0.055   0.011   0.32

    * at M = 1 (Narrow, Wide 1 KA) and M = 5 (Wide 2 KA).

tests/test_mlp_bounds_cpu.py shows the checks still fail kernels that drop a batch row, a 16-row slab, a feature,
a hidden unit or b2, flip one ReLU or compute a GEMM at TF32 precision.
"""
from __future__ import annotations

import math

import numpy as np
import torch

PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")
U = 2.0 ** -24
LAM = 8.0
SHORT = 32  # the batch sums take sqrt(M + SHORT): see above
# Precision floors next to the bound.  The bound sums worst cases (e_pre |W2|^T is linear in H), so on its own it
# admits a kernel that computes a GEMM at TF32 precision (one of the three 3xTF32 terms missing): that stays
# within the bound at several shapes, while it misses these floors by 3x or more.
FWD_ATOL = 1e-5  # forward: absolute, outputs are of order 1
GRAD_REL = 2e-5  # backward: relative to the tensor's largest entry, on W2, b2 and the W1 / b1 rows without a tie


def _dev(device):
    if device is not None:
        return torch.device(device)
    return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def _f64(a, device):
    t = a.detach() if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    return t.to(device=device, dtype=torch.float64)


def _params(params, device):
    seq = [params[k] for k in PKEYS] if isinstance(params, dict) else list(params)
    return [_f64(a, device) for a in seq]


def _worst(got, want, e) -> float:
    """max err / e, with err / 0 = inf for any nonzero err (and 0 / 0 = 0)."""
    err = (_f64(got, want.device).reshape(want.shape) - want).abs()
    if not torch.isfinite(err).all():
        return math.inf
    r = torch.where(e > 0, err / torch.where(e > 0, e, 1.0), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


class MlpBound:
    """Reference values and per-entry bounds of one forward (and, given dout, one backward) on rows x (M, O),
    float32 or uint8 values taken exactly.  `params`: a state_dict with PKEYS or (W1, b1, W2, b2)."""

    def __init__(self, x, params, dout=None, lam: float = LAM, device=None):
        dev = _dev(device)
        x = _f64(x, dev)
        w1, b1, w2, b2 = _params(params, dev)
        M, O = x.shape
        H, N2 = w1.shape[0], w2.shape[0]
        self.M, self.O, self.H, self.N2, self.lam = M, O, H, N2, lam
        c = lam * U
        ax, aw1, aw2 = x.abs(), w1.abs(), w2.abs()
        self.x, self.w1, self.b1, self.w2, self.b2 = x, w1, b1, w2, b2
        self.pre = x @ w1.T + b1
        self.e_pre = c * math.sqrt(O + 1) * (ax @ aw1.T + b1.abs())
        self.h = self.pre.clamp_min(0.0)
        self.out = self.h @ w2.T + b2
        self.e_out = c * math.sqrt(H + 1) * ((self.h + self.e_pre) @ aw2.T + b2.abs()) + self.e_pre @ aw2.T
        self.grad = self.e_grad = None
        self.ties = 0
        if dout is None:
            return
        dout = _f64(dout, dev).reshape(M, N2)
        adout = dout.abs()
        self.dout = dout
        self.dh = dout @ w2
        e_dh = c * math.sqrt(N2) * (adout @ aw2)
        dp = self.dh * (self.pre > 0)
        tied = self.pre.abs() < self.e_pre
        self.ties = int(tied.sum())
        cm = c * math.sqrt(M + SHORT)
        dpe = dp.abs() + e_dh
        tdh = self.dh.abs() * tied
        self.grad = (dp.T @ x, dp.sum(0), dout.T @ self.h, dout.sum(0))
        self.untied = ~tied.any(dim=0)  # hidden units without a tie: their W1 / b1 bounds are rounding only
        self.e_grad = (cm * (dpe.T @ ax) + e_dh.T @ ax + tdh.T @ ax,
                       cm * dpe.sum(0) + e_dh.sum(0) + tdh.sum(0),
                       cm * (adout.T @ (self.h + self.e_pre)) + adout.T @ self.e_pre,
                       cm * adout.sum(0))

    def forward_errors(self, got, atol=None, scaled=False) -> dict:
        """{"out": worst err / e} of the (M, N2) output and, given `atol`, "out abs": max err / atol (with `scaled`,
        atol * max(1, max |out|))."""
        rep = {"out": _worst(got, self.out, self.e_out)}
        if atol is not None:
            err = float((_f64(got, self.out.device).reshape(self.out.shape) - self.out).abs().max())
            floor = atol * (max(1.0, float(self.out.abs().max())) if scaled else 1.0)
            rep["out abs"] = err / floor if math.isfinite(err) else math.inf
        return rep

    def backward_errors(self, got, rel=None) -> dict:
        """Worst err / e per parameter tensor, the same for W1 / b1 over the hidden units without a tie ("W1 untied",
        "b1 untied": a switched tie moves its entries by about its whole allowance, so only these show how much of
        the rounding bound a kernel uses), "pad": largest |entry| outside the four tensors (must be 0) and "ties".
        Given `rel`, also max err / (rel * max |tensor|) of W2 and b2 and of the W1 / b1 entries of the untied units
        (keys ending in " rel").  `got`: the kernel's flat float64 gradient block, or a dict / 4-tuple of the
        tensors."""
        rep = {}
        if torch.is_tensor(got) and got.dim() == 1:
            from torched_impala_b200 import _cabi

            offs, total = _cabi.param_layout(self.O, self.H, self.N2)
            assert got.numel() == total, (got.numel(), total)
            flat = got.detach().to(self.out.device, torch.float64)
            real = torch.zeros(total, dtype=torch.bool, device=flat.device)
            parts = []
            for off, w in zip(offs, self.grad):
                real[off:off + w.numel()] = True
                parts.append(flat[off:off + w.numel()])
            rep["pad"] = float(flat[~real].abs().max()) if (~real).any() else 0.0
            if not torch.isfinite(flat[~real]).all():
                rep["pad"] = math.inf
            got = parts
        elif isinstance(got, dict):
            got = [got[k] for k in PKEYS]
        for k, g, w, e in zip(PKEYS, got, self.grad, self.e_grad):
            rep[k] = _worst(g, w, e)
        for k, g, w, e in zip(("W1 untied", "b1 untied"), got, self.grad, self.e_grad):
            g = _f64(g, w.device).reshape(w.shape)
            rep[k] = _worst(g[self.untied], w[self.untied], e[self.untied])
        if rel is not None:
            for k, g, w in zip(("W1 untied rel", "b1 untied rel", "W2 rel", "b2 rel"), got, self.grad):
                g = _f64(g, w.device).reshape(w.shape)
                d = (g - w).abs()[self.untied] if k.startswith(("W1", "b1")) else (g - w).abs()
                err = float(d.max()) if d.numel() else 0.0
                scale = rel * float(w.abs().max())
                rep[k] = (err / scale if scale > 0 else math.inf * (err > 0)) if math.isfinite(err) else math.inf
        rep["ties"] = self.ties
        return rep


def within(rep: dict) -> bool:
    return all(v <= 1.0 for k, v in rep.items() if k not in ("pad", "ties")) and rep.get("pad", 0.0) == 0.0


def assert_within(rep: dict, what="") -> None:
    print("bound", what, {k: (round(v, 4) if isinstance(v, float) else v) for k, v in rep.items()})
    assert within(rep), (what, rep)


def check_forward(got, x, params, what="", atol=FWD_ATOL, scaled=False, **kw) -> dict:
    """The output within its bound and within `atol` absolute (see FWD_ATOL)."""
    rep = MlpBound(x, params, **kw).forward_errors(got, atol, scaled)
    assert_within(rep, what)
    return rep


def check_backward(got, x, params, dout, what="", rel=GRAD_REL, **kw) -> dict:
    """Every gradient entry within its bound, and W2, b2 and the untied W1 / b1 rows within `rel` of their tensor's
    largest entry (see GRAD_REL)."""
    rep = MlpBound(x, params, dout, **kw).backward_errors(got, rel)
    assert_within(rep, what)
    return rep
