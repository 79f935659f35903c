"""Thin per-kernel wrappers over the C ABI for torch CUDA tensors.

Each function allocates its outputs with torch (device-memory plumbing), launches one
C-ABI call on the current torch stream and returns the outputs.  They exist for the
parity tests and for users who want a single piece of the update (e.g. V-trace only);
the learner itself goes through `engine.LearnerEngine`, which pre-allocates everything.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _cabi

PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _need_cuda(*ts):
    for t in ts:
        if not (torch.is_tensor(t) and t.is_cuda and t.is_contiguous()):
            raise _cabi.ImpalaCudaError("expected contiguous CUDA tensors (there is no CPU fallback)")


def pack_params(state_dict: dict, device="cuda") -> torch.Tensor:
    """state_dict of one reference MLP (models.py:13-18) -> flat float32 parameter block."""
    w1 = np.asarray(state_dict[PKEYS[0]], dtype=np.float32)
    w2 = np.asarray(state_dict[PKEYS[2]], dtype=np.float32)
    H, O = w1.shape
    N2 = w2.shape[0]
    offs, total = _cabi.param_layout(O, H, N2)
    flat = np.zeros(total, np.float32)
    for k, off in zip(PKEYS, offs):
        a = np.asarray(state_dict[k], dtype=np.float32).reshape(-1)
        flat[off:off + a.size] = a
    return torch.from_numpy(flat).to(device)


def unpack_grad(flat, O: int, H: int, N2: int) -> dict:
    offs, _ = _cabi.param_layout(O, H, N2)
    shapes = ((H, O), (H,), (N2, H), (N2,))
    a = flat.detach().cpu().numpy()
    return {k: a[off:off + int(np.prod(s))].reshape(s).copy() for k, off, s in zip(PKEYS, offs, shapes)}


def mlp_forward(x, params, O: int, H: int, N2: int):
    _need_cuda(x, params)
    M = x.numel() // O
    out = torch.empty(M, N2, dtype=torch.float32, device=x.device)
    _cabi.check(_cabi.lib().impala_mlp_forward(_p(x), _p(params), _p(out), M, O, H, N2, _st()),
                "impala_mlp_forward")
    return out


def mlp_backward(x, params, dout, O: int, H: int, N2: int):
    _need_cuda(x, params, dout)
    lib = _cabi.lib()
    M = x.numel() // O
    _, total = _cabi.param_layout(O, H, N2)
    nbytes = lib.impala_mlp_backward_workspace(M, O, H, N2)
    if nbytes < 0:
        _cabi.check(int(nbytes), "impala_mlp_backward_workspace")
    ws = torch.zeros(int(nbytes), dtype=torch.uint8, device=x.device)  # control words start at 0
    grad = torch.empty(total, dtype=torch.float64, device=x.device)
    _cabi.check(lib.impala_mlp_backward(_p(x), _p(params), _p(dout), _p(grad), _p(ws), int(nbytes),
                                        M, O, H, N2, _st()), "impala_mlp_backward")
    return grad


def mlp_forward_u8(x, params, O: int, H: int, N2: int):
    """impala_mlp_forward_u8: byte observations x (uint8, values unscaled), 128 < O <= 1024."""
    _need_cuda(x, params)
    if x.dtype != torch.uint8:
        raise _cabi.ImpalaCudaError(f"mlp_forward_u8 takes uint8 observations, got {x.dtype}")
    M = x.numel() // O
    out = torch.empty(M, N2, dtype=torch.float32, device=x.device)
    _cabi.check(_cabi.lib().impala_mlp_forward_u8(_p(x), _p(params), _p(out), M, O, H, N2, _st()),
                "impala_mlp_forward_u8")
    return out


def mlp_backward_u8(x, params, dout, O: int, H: int, N2: int):
    """impala_mlp_backward_u8 (workspace as for mlp_backward)."""
    _need_cuda(x, params, dout)
    if x.dtype != torch.uint8:
        raise _cabi.ImpalaCudaError(f"mlp_backward_u8 takes uint8 observations, got {x.dtype}")
    lib = _cabi.lib()
    M = x.numel() // O
    _, total = _cabi.param_layout(O, H, N2)
    nbytes = lib.impala_mlp_backward_workspace(M, O, H, N2)
    if nbytes < 0:
        _cabi.check(int(nbytes), "impala_mlp_backward_workspace")
    ws = torch.zeros(int(nbytes), dtype=torch.uint8, device=x.device)
    grad = torch.empty(total, dtype=torch.float64, device=x.device)
    _cabi.check(lib.impala_mlp_backward_u8(_p(x), _p(params), _p(dout), _p(grad), _p(ws), int(nbytes),
                                           M, O, H, N2, _st()), "impala_mlp_backward_u8")
    return grad


def obs_u8_to_f32(x):
    """Exact float32 copy of a uint8 tensor (impala_obs_u8_to_f32)."""
    _need_cuda(x)
    if x.dtype != torch.uint8:
        raise _cabi.ImpalaCudaError(f"obs_u8_to_f32 takes uint8, got {x.dtype}")
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    _cabi.check(_cabi.lib().impala_obs_u8_to_f32(_p(x), _p(out), x.numel(), _st()), "impala_obs_u8_to_f32")
    return out


def obs_unstack(frames, k: int, out_dtype=None):
    """Dense stacked observations (R, B, k F) from frames (R + k - 1, B, F) (impala_obs_unstack): row (t, b) is
    frames t .. t+k-1 of column b, oldest first.  uint8 -> uint8 | float32, float32 -> float32."""
    _need_cuda(frames)
    codes = {torch.uint8: _cabi.OBS_U8, torch.float32: _cabi.OBS_F32}
    out_dtype = frames.dtype if out_dtype is None else out_dtype
    if frames.dim() != 3 or frames.dtype not in codes or out_dtype not in codes:
        raise _cabi.ImpalaCudaError(f"obs_unstack takes (R+k-1, B, F) uint8 / float32 frames, got {tuple(frames.shape)} "
                                    f"{frames.dtype} -> {out_dtype}")
    n, B, F = frames.shape
    R = n - k + 1
    out = torch.empty(max(R, 0), B, k * F, dtype=out_dtype, device=frames.device)
    _cabi.check(_cabi.lib().impala_obs_unstack(_p(frames), codes[frames.dtype], _p(out), codes[out_dtype], R, B, F, k,
                                               _st()), "impala_obs_unstack")
    return out


def batch_compose(store, plan, T: int, B: int, Bf: int, F: int, frames: int, A: int, obs_dtype: str = "float32",
                  out=None, action_dist: str = "categorical", action_heads=(), action_mask: bool = False):
    """The B-column training slab (uint8 bytes, _cabi.batch_layout(T, B, ...)) gathered from `store`, a
    (slabs, slab_bytes) uint8 tensor of Bf-column slabs, by `plan` (B, 2) int32 (slab, column), slab < 0 = an
    empty column (impala_batch_compose; impala_batch_compose_act for action_dist="gaussian" and "multi_discrete",
    whose action_heads give the K int32 actions per step, and for action_mask=True, whose actions end in the legal
    word).  `out`: a uint8 tensor of the slab's size to write into."""
    _need_cuda(store, plan)
    if store.dtype != torch.uint8 or store.dim() != 2 or plan.dtype != torch.int32 or tuple(plan.shape) != (B, 2):
        raise _cabi.ImpalaCudaError(f"batch_compose takes a (slabs, bytes) uint8 store and a ({B}, 2) int32 plan, got "
                                    f"{tuple(store.shape)} {store.dtype}, {tuple(plan.shape)} {plan.dtype}")
    _, total = _cabi.batch_layout(T, B, F * frames, A, obs_dtype, frames, action_dist, action_heads, action_mask)
    if out is None:
        out = torch.empty(total, dtype=torch.uint8, device=store.device)
    _need_cuda(out)
    if out.dtype != torch.uint8 or out.numel() != total:
        raise _cabi.ImpalaCudaError(f"batch_compose writes a slab of {total} bytes, got {out.numel()} {out.dtype}")
    if action_dist != "categorical" or action_mask:
        _cabi.check(_cabi.lib().impala_batch_compose_act(_p(out), _p(store), store.shape[1], _p(plan), T, B, Bf, F,
                                                         frames, A, _cabi.obs_dtype_code(obs_dtype),
                                                         _cabi.act_kind_code(action_dist, action_heads, action_mask),
                                                         _st()),
                    "impala_batch_compose_act")
        return out
    _cabi.check(_cabi.lib().impala_batch_compose(_p(out), _p(store), store.shape[1], _p(plan), T, B, Bf, F, frames, A,
                                                 _cabi.obs_dtype_code(obs_dtype), _st()), "impala_batch_compose")
    return out


def mlp_forward_pair(x, params_pi, params_vf, M_pi: int, M_vf: int, O: int, H_pi: int, H_vf: int, A: int):
    """Policy logits on the first M_pi rows of x and values on the first M_vf rows, one call."""
    _need_cuda(x, params_pi, params_vf)
    logits = torch.empty(M_pi, A, dtype=torch.float32, device=x.device)
    values = torch.empty(M_vf, dtype=torch.float32, device=x.device)
    _cabi.check(_cabi.lib().impala_mlp_forward_pair(_p(x), _p(params_pi), _p(params_vf), _p(logits), _p(values),
                                                    M_pi, M_vf, O, H_pi, H_vf, A, _st()),
                "impala_mlp_forward_pair")
    return logits, values


def mlp_backward_pair(x, params_pi, params_vf, dlogits, dv, O: int, H_pi: int, H_vf: int, A: int):
    _need_cuda(x, params_pi, params_vf, dlogits, dv)
    lib = _cabi.lib()
    M_pi, M_vf = dlogits.numel() // A, dv.numel()
    out, wss = [], []
    for M, H, N2 in ((M_pi, H_pi, A), (M_vf, H_vf, 1)):
        nbytes = lib.impala_mlp_backward_workspace(M, O, H, N2)
        if nbytes < 0:
            _cabi.check(int(nbytes), "impala_mlp_backward_workspace")
        wss.append(torch.zeros(int(nbytes), dtype=torch.uint8, device=x.device))
        out.append(torch.empty(_cabi.param_layout(O, H, N2)[1], dtype=torch.float64, device=x.device))
    _cabi.check(lib.impala_mlp_backward_pair(_p(x), _p(params_pi), _p(params_vf), _p(dlogits), _p(dv),
                                             _p(out[0]), _p(out[1]), _p(wss[0]), wss[0].numel(), _p(wss[1]),
                                             wss[1].numel(), M_pi, M_vf, O, H_pi, H_vf, A, _st()),
                "impala_mlp_backward_pair")
    return out[0], out[1]


def vtrace(cur_logits, beh_logits, actions, rewards, done, lens, v, gamma, rho_bar, c_bar,
           mode="reference"):
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v)
    T, B, A = cur_logits.shape
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=v.device)
    pg = torch.empty(T, B, dtype=torch.float32, device=v.device)
    _cabi.check(_cabi.lib().impala_vtrace(_p(cur_logits), _p(beh_logits), _p(actions), _p(rewards),
                                          _p(done), _p(lens), _p(v), _p(vs), _p(pg), T, B, A,
                                          float(gamma), float(rho_bar), float(c_bar),
                                          _cabi.MODES[mode], _st()), "impala_vtrace")
    return vs, pg


def vtrace_loss(cur_logits, beh_logits, actions, rewards, done, lens, v, hp, inv_batch,
                mode="reference"):
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v)
    T, B, A = cur_logits.shape
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(T, B, A, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    lib = _cabi.lib()
    ws_bytes = int(lib.impala_vtrace_loss_workspace(T, B, A))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    _cabi.check(lib.impala_vtrace_loss(
        _p(cur_logits), _p(beh_logits), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dlogits), _p(dv), _p(scalars), _p(ws), ws_bytes, T, B, A, float(hp.gamma),
        float(hp.rho_bar),
        float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], _st()), "impala_vtrace_loss")
    return dict(vs=vs, pg_adv=pg, dlogits=dlogits, dv=dv, scalars=scalars)


def vtrace_loss_diag(cur_logits, beh_logits, actions, rewards, done, lens, v, hp, inv_batch,
                     mode="reference"):
    """vtrace_loss plus `diag`: the eight float64 off-policy sums of impala_vtrace_loss_diag (see
    engine.diagnostic_values for the logged values derived from them)."""
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v)
    T, B, A = cur_logits.shape
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(T, B, A, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    diag = torch.empty(8, dtype=torch.float64, device=dev)
    lib = _cabi.lib()
    ws_bytes = int(lib.impala_vtrace_loss_diag_workspace(T, B, A))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    _cabi.check(lib.impala_vtrace_loss_diag(
        _p(cur_logits), _p(beh_logits), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dlogits), _p(dv), _p(scalars), _p(diag), _p(ws), ws_bytes, T, B, A, float(hp.gamma),
        float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], _st()), "impala_vtrace_loss_diag")
    return dict(vs=vs, pg_adv=pg, dlogits=dlogits, dv=dv, scalars=scalars, diag=diag)


def clip_adam(params, grad, m, v, step, n_policy, max_norm, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    _need_cuda(params, grad, m, v, step)
    norms = torch.empty(2, dtype=torch.float64, device=params.device)
    _cabi.check(_cabi.lib().impala_clip_adam(_p(params), _p(grad), _p(m), _p(v), _p(step),
                                             int(n_policy), params.numel(), float(max_norm),
                                             float(lr), float(beta1), float(beta2), float(eps),
                                             _p(norms), _st()), "impala_clip_adam")
    return norms


def clip_optim(params, grad, m, v, step, n_policy, max_norm, lr_table, rule="adam", h0=0.9, h1=0.999, eps=1e-8):
    """impala_clip_optim: clip + one Adam ("adam": h0, h1 = beta1, beta2) or RMSprop ("rmsprop": h0, h1 = alpha,
    momentum) step with the learning rate lr_table[min(step[0], len - 1)] (float32 CUDA tensor)."""
    _need_cuda(params, grad, m, v, step, lr_table)
    if lr_table.dtype != torch.float32:
        raise _cabi.ImpalaCudaError(f"lr_table must be float32, got {lr_table.dtype}")
    norms = torch.empty(2, dtype=torch.float64, device=params.device)
    _cabi.check(_cabi.lib().impala_clip_optim(_p(params), _p(grad), _p(m), _p(v), _p(step), int(n_policy),
                                              params.numel(), float(max_norm), _p(lr_table), lr_table.numel(),
                                              _cabi.OPT_RULES[rule], float(h0), float(h1), float(eps), _p(norms),
                                              _st()), "impala_clip_optim")
    return norms


def popart_stats(mu=0.0, nu=1.0, device="cuda"):
    """A float64 PopArt statistics buffer {mu, nu, sigma, mu_loss, sigma_loss} (IMPALA_POPART_STATS) for the
    value statistics (mu, nu); sigma = clamp(sqrt(max(nu - mu^2, 0)), 1e-4, 1e6)."""
    sigma = min(max(max(nu - mu * mu, 0.0) ** 0.5, 1e-4), 1e6)
    return torch.tensor([mu, nu, sigma, mu, sigma], dtype=torch.float64, device=device)


def vtrace_loss_popart(cur_logits, beh_logits, actions, rewards, done, lens, v, hp, inv_batch, popart,
                       mode="reference"):
    """vtrace_loss_diag on the NORMALIZED values v under the PopArt statistics `popart` (float64 CUDA tensor,
    popart_stats' layout): vs and `diag` in reward units, pg_adv, dv, dlogits and the two losses normalized
    (impala_vtrace_loss_popart)."""
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v, popart)
    if popart.dtype != torch.float64 or popart.numel() < 3:
        raise _cabi.ImpalaCudaError("popart must be a float64 tensor of the statistics (popart_stats)")
    T, B, A = cur_logits.shape
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(T, B, A, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    diag = torch.empty(8, dtype=torch.float64, device=dev)
    lib = _cabi.lib()
    ws_bytes = int(lib.impala_vtrace_loss_diag_workspace(T, B, A))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    _cabi.check(lib.impala_vtrace_loss_popart(
        _p(cur_logits), _p(beh_logits), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dlogits), _p(dv), _p(scalars), _p(diag), _p(ws), ws_bytes, T, B, A, float(hp.gamma),
        float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], _p(popart), _st()), "impala_vtrace_loss_popart")
    return dict(vs=vs, pg_adv=pg, dlogits=dlogits, dv=dv, scalars=scalars, diag=diag)


def clip_optim_popart(params, grad, m, v, step, n_policy, max_norm, lr_table, popart, sums_at, w2_off, w2_len,
                      b2_off, beta=3e-4, rule="adam", h0=0.9, h1=0.999, eps=1e-8):
    """impala_clip_optim_popart: clip_optim, then the PopArt statistics update from the eight sums at
    grad[sums_at:sums_at + 8] and the output-preserving rescale of the value head params[w2_off:w2_off + w2_len]
    (W2) and params[b2_off] (b2).  `popart` (float64 CUDA tensor, popart_stats' layout) is updated in place."""
    _need_cuda(params, grad, m, v, step, lr_table, popart)
    if lr_table.dtype != torch.float32:
        raise _cabi.ImpalaCudaError(f"lr_table must be float32, got {lr_table.dtype}")
    if popart.dtype != torch.float64 or popart.numel() < _cabi.POPART_STATS:
        raise _cabi.ImpalaCudaError("popart must be a float64 tensor of the statistics (popart_stats)")
    if grad.numel() < sums_at + 8:
        raise _cabi.ImpalaCudaError(f"grad holds {grad.numel()} entries, the sums end at {sums_at + 8}")
    norms = torch.empty(2, dtype=torch.float64, device=params.device)
    _cabi.check(_cabi.lib().impala_clip_optim_popart(
        _p(params), _p(grad), _p(m), _p(v), _p(step), int(n_policy), params.numel(), float(max_norm), _p(lr_table),
        lr_table.numel(), _cabi.OPT_RULES[rule], float(h0), float(h1), float(eps), _p(norms), _p(popart),
        int(sums_at), int(w2_off), int(w2_len), int(b2_off), float(beta), _st()), "impala_clip_optim_popart")
    return norms


def vtrace_loss_rclip(cur_logits, beh_logits, actions, rewards, done, lens, v, hp, inv_batch, reward_clip,
                      mode="reference", diagnostics=False, popart=None):
    """vtrace_loss (diagnostics=False, popart=None), vtrace_loss_diag (diagnostics=True) or vtrace_loss_popart
    (popart: the statistics tensor) with the reward transform `reward_clip` ("abs_one" | "soft_asymmetric")
    applied to the rewards inside the kernel (impala_vtrace_loss_rclip); scalars[3] stays the raw rewards' mean."""
    code = _cabi.reward_clip_code(reward_clip)
    if not code:
        raise ValueError("vtrace_loss_rclip needs a reward_clip; vtrace_loss is the untransformed kernel")
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v)
    if popart is not None:
        _need_cuda(popart)
        if popart.dtype != torch.float64 or popart.numel() < 3:
            raise _cabi.ImpalaCudaError("popart must be a float64 tensor of the statistics (popart_stats)")
    with_diag = bool(diagnostics) or popart is not None
    T, B, A = cur_logits.shape
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(T, B, A, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    diag = torch.empty(8, dtype=torch.float64, device=dev) if with_diag else None
    lib = _cabi.lib()
    ws_fn = lib.impala_vtrace_loss_diag_workspace if with_diag else lib.impala_vtrace_loss_workspace
    ws_bytes = int(ws_fn(T, B, A))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    _cabi.check(lib.impala_vtrace_loss_rclip(
        _p(cur_logits), _p(beh_logits), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dlogits), _p(dv), _p(scalars), _p(ws), ws_bytes, T, B, A, float(hp.gamma),
        float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], None if diag is None else _p(diag),
        None if popart is None else _p(popart), code, _st()), "impala_vtrace_loss_rclip")
    out = dict(vs=vs, pg_adv=pg, dlogits=dlogits, dv=dv, scalars=scalars)
    if with_diag:
        out["diag"] = diag
    return out


def vtrace_loss_gauss(cur_params, beh_params, actions, rewards, done, lens, v, hp, inv_batch, mode="reference",
                      diagnostics=False, popart=None, reward_clip=None):
    """The V-trace loss kernel for diagonal Gaussian policies (impala_vtrace_loss_gauss): cur_params / beh_params
    (T, B, 2A) float32 policy outputs [mean | log std], actions (T, B, A) float32 samples.  Returns vs, pg_adv,
    dparams (T, B, 2A), dv, scalars and, with diagnostics=True or popart (the statistics tensor), diag."""
    code = _cabi.reward_clip_code(reward_clip)
    _need_cuda(cur_params, beh_params, actions, rewards, done, lens, v)
    if popart is not None:
        _need_cuda(popart)
        if popart.dtype != torch.float64 or popart.numel() < 3:
            raise _cabi.ImpalaCudaError("popart must be a float64 tensor of the statistics (popart_stats)")
    T, B, A2 = cur_params.shape
    if A2 % 2 or actions.dtype != torch.float32 or tuple(actions.shape) != (T, B, A2 // 2):
        raise _cabi.ImpalaCudaError(f"vtrace_loss_gauss takes (T, B, 2A) outputs and (T, B, A) float32 actions, got "
                                    f"{tuple(cur_params.shape)} and {tuple(actions.shape)} {actions.dtype}")
    A = A2 // 2
    with_diag = bool(diagnostics) or popart is not None
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dparams = torch.empty(T, B, 2 * A, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    diag = torch.empty(8, dtype=torch.float64, device=dev) if with_diag else None
    lib = _cabi.lib()
    ws_fn = lib.impala_vtrace_loss_diag_workspace if with_diag else lib.impala_vtrace_loss_workspace
    ws_bytes = int(ws_fn(T, B, A))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    _cabi.check(lib.impala_vtrace_loss_gauss(
        _p(cur_params), _p(beh_params), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dparams), _p(dv), _p(scalars), _p(ws), ws_bytes, T, B, A, float(hp.gamma),
        float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], None if diag is None else _p(diag),
        None if popart is None else _p(popart), code, _st()), "impala_vtrace_loss_gauss")
    out = dict(vs=vs, pg_adv=pg, dparams=dparams, dv=dv, scalars=scalars)
    if with_diag:
        out["diag"] = diag
    return out


def vtrace_loss_md(cur_logits, beh_logits, actions, rewards, done, lens, v, hp, inv_batch, heads, mode="reference",
                   diagnostics=False, popart=None, reward_clip=None):
    """The V-trace loss kernel for multi-discrete policies (impala_vtrace_loss_md): cur_logits / beh_logits (T, B, N)
    float32 with N = sum(heads), actions (T, B, K) int32, one index per head.  Returns vs, pg_adv, dlogits (T, B, N),
    dv, scalars and, with diagnostics=True or popart (the statistics tensor), diag."""
    code = _cabi.reward_clip_code(reward_clip)
    heads = _cabi.check_heads(heads)
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v)
    if popart is not None:
        _need_cuda(popart)
        if popart.dtype != torch.float64 or popart.numel() < 3:
            raise _cabi.ImpalaCudaError("popart must be a float64 tensor of the statistics (popart_stats)")
    T, B, N = cur_logits.shape
    K = len(heads)
    if N != sum(heads) or actions.dtype != torch.int32 or tuple(actions.shape) != (T, B, K):
        raise _cabi.ImpalaCudaError(f"vtrace_loss_md takes (T, B, {sum(heads)}) logits and (T, B, {K}) int32 actions "
                                    f"for heads {heads}, got {tuple(cur_logits.shape)} and {tuple(actions.shape)} "
                                    f"{actions.dtype}")
    with_diag = bool(diagnostics) or popart is not None
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(T, B, N, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    diag = torch.empty(8, dtype=torch.float64, device=dev) if with_diag else None
    lib = _cabi.lib()
    ws_fn = lib.impala_vtrace_loss_diag_workspace if with_diag else lib.impala_vtrace_loss_workspace
    ws_bytes = int(ws_fn(T, B, N))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    h = (C.c_int32 * K)(*heads)
    _cabi.check(lib.impala_vtrace_loss_md(
        _p(cur_logits), _p(beh_logits), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dlogits), _p(dv), _p(scalars), _p(ws), ws_bytes, T, B, N, float(hp.gamma),
        float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], None if diag is None else _p(diag),
        None if popart is None else _p(popart), code, h, K, _st()), "impala_vtrace_loss_md")
    out = dict(vs=vs, pg_adv=pg, dlogits=dlogits, dv=dv, scalars=scalars)
    if with_diag:
        out["diag"] = diag
    return out


def vtrace_loss_mask(cur_logits, beh_logits, actions, rewards, done, lens, v, hp, inv_batch, heads=(),
                     mode="reference", diagnostics=False, popart=None, reward_clip=None):
    """The V-trace loss kernel with invalid-action masks (impala_vtrace_loss_mask): cur_logits / beh_logits (T, B, N)
    float32, N <= 32; actions (T, B, 2) int32 [a, legal] for a categorical policy (heads=()) or (T, B, K + 1)
    [a_0 .. a_{K-1}, legal] for the multi-discrete heads `heads` (sum = N).  Bit j of the legal word: output j is
    legal.  Returns vs, pg_adv, dlogits (T, B, N), dv, scalars and, with diagnostics=True or popart, diag."""
    code = _cabi.reward_clip_code(reward_clip)
    heads = _cabi.check_heads(heads) if len(heads) else ()
    _need_cuda(cur_logits, beh_logits, actions, rewards, done, lens, v)
    if popart is not None:
        _need_cuda(popart)
        if popart.dtype != torch.float64 or popart.numel() < 3:
            raise _cabi.ImpalaCudaError("popart must be a float64 tensor of the statistics (popart_stats)")
    T, B, N = cur_logits.shape
    K = len(heads)
    if (heads and N != sum(heads)) or actions.dtype != torch.int32 or tuple(actions.shape) != (T, B, K + 1 if K else 2):
        raise _cabi.ImpalaCudaError(f"vtrace_loss_mask takes (T, B, N) logits and (T, B, {K + 1 if K else 2}) int32 "
                                    f"actions ending in the legal word for heads {heads}, got {tuple(cur_logits.shape)}"
                                    f" and {tuple(actions.shape)} {actions.dtype}")
    with_diag = bool(diagnostics) or popart is not None
    dev = v.device
    vs = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    pg = torch.empty(T, B, dtype=torch.float32, device=dev)
    dlogits = torch.empty(T, B, N, dtype=torch.float32, device=dev)
    dv = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    scalars = torch.empty(4, dtype=torch.float64, device=dev)
    diag = torch.empty(8, dtype=torch.float64, device=dev) if with_diag else None
    lib = _cabi.lib()
    ws_fn = lib.impala_vtrace_loss_diag_workspace if with_diag else lib.impala_vtrace_loss_workspace
    ws_bytes = int(ws_fn(T, B, N))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    h = (C.c_int32 * K)(*heads) if K else None
    _cabi.check(lib.impala_vtrace_loss_mask(
        _p(cur_logits), _p(beh_logits), _p(actions), _p(rewards), _p(done), _p(lens), _p(v), _p(vs),
        _p(pg), _p(dlogits), _p(dv), _p(scalars), _p(ws), ws_bytes, T, B, N, float(hp.gamma),
        float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c), float(hp.policy_loss_c), float(hp.entropy_c),
        float(inv_batch), _cabi.MODES[mode], None if diag is None else _p(diag),
        None if popart is None else _p(popart), code, h, K, _st()), "impala_vtrace_loss_mask")
    out = dict(vs=vs, pg_adv=pg, dlogits=dlogits, dv=dv, scalars=scalars)
    if with_diag:
        out["diag"] = diag
    return out
