"""ctypes binding of include/impala_b200.h (the C-ABI boundary of the hot path).

There is no CPU fallback anywhere in this package: if `libimpala_b200.so` is
missing, or a call returns non-zero, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import numbers
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# IMPALA_LIB_DIR: a library built elsewhere (build.py honours the same variable)
LIB_PATH = os.path.join(os.environ.get("IMPALA_LIB_DIR", os.path.join(_HERE, "lib")), "libimpala_b200.so")

MODE_REFERENCE = 0
MODE_PAPER = 1
MODES = {"reference": MODE_REFERENCE, "paper": MODE_PAPER}

OBS_F32 = 0
OBS_U8 = 1
OBS_DTYPES = {"float32": OBS_F32, "uint8": OBS_U8}  # batch-slab observation types (impala_batch_layout_obs)
OBS_NORM_MAX_FEATURES = 1024  # observation features of impala_obs_normalize (IMPALA_OBS_NORM_MAX_FEATURES)

OPT_ADAM = 0
OPT_RMSPROP = 1
OPT_RULES = {"adam": OPT_ADAM, "rmsprop": OPT_RMSPROP}  # update rules of impala_clip_optim
POPART_STATS = 5  # float64 {mu, nu, sigma, mu_loss, sigma_loss} (IMPALA_POPART_STATS)
REWARD_CLIP_ABS_ONE = 1
REWARD_CLIP_SOFT_ASYMMETRIC = 2
# reward transforms of impala_vtrace_loss_rclip (IMPALA_REWARD_CLIP_*)
REWARD_CLIPS = {"abs_one": REWARD_CLIP_ABS_ONE, "soft_asymmetric": REWARD_CLIP_SOFT_ASYMMETRIC}


def obs_dtype_code(obs_dtype: str) -> int:
    if obs_dtype not in OBS_DTYPES:
        raise ValueError(f"obs_dtype must be one of {sorted(OBS_DTYPES)}, got {obs_dtype!r}")
    return OBS_DTYPES[obs_dtype]


def reward_clip_code(reward_clip) -> int:
    """The IMPALA_REWARD_CLIP_* code of `reward_clip` ("abs_one" | "soft_asymmetric"), 0 for None (no transform);
    anything else raises ValueError naming the accepted values."""
    if reward_clip is None:
        return 0
    if not isinstance(reward_clip, str) or reward_clip not in REWARD_CLIPS:
        raise ValueError(f"reward_clip must be None or one of {sorted(REWARD_CLIPS)}, got {reward_clip!r}")
    return REWARD_CLIPS[reward_clip]

ACT_CATEGORICAL = 0
ACT_GAUSSIAN = 1
ACT_MULTI_DISCRETE = 0x100  # IMPALA_ACT_MULTI_DISCRETE(K) = ACT_MULTI_DISCRETE | K
ACT_MASKED = 0x200  # IMPALA_ACT_MASKED: OR-ed onto categorical or multi-discrete, one int32 legal word per step
ACT_DISTS = {"categorical": ACT_CATEGORICAL, "gaussian": ACT_GAUSSIAN}  # action distributions (IMPALA_ACT_*)
MAX_GAUSSIAN_DIMS = 16  # action dimensions of impala_vtrace_loss_gauss (2A <= 32 policy outputs)
MAX_HEADS = 16  # heads of impala_vtrace_loss_md (sum n_k <= 32 policy outputs)
MAX_OUTPUTS = 32  # policy outputs of the MLP kernels


def check_heads(action_heads) -> tuple:
    """The head sizes (n_0, .., n_K-1) of a multi-discrete policy as a tuple of ints: 1 <= K <= 16 heads of at least
    two actions each, at most 32 outputs in all; anything else raises ValueError."""
    heads = tuple(action_heads)
    if not all(isinstance(n, numbers.Integral) and not isinstance(n, bool) for n in heads):
        raise ValueError(f"action_heads must be integers, got {heads!r}")
    heads = tuple(int(n) for n in heads)
    if not 1 <= len(heads) <= MAX_HEADS:
        raise ValueError(f"a multi-discrete policy takes 1 to {MAX_HEADS} heads, got {len(heads)}")
    if min(heads) < 2:
        raise ValueError(f"every head of a multi-discrete policy has at least 2 actions, got {heads}")
    if sum(heads) > MAX_OUTPUTS:
        raise ValueError(f"a multi-discrete policy takes at most {MAX_OUTPUTS} outputs in all, got sum{heads} = "
                         f"{sum(heads)}")
    return heads


def act_kind_code(action_dist: str, action_heads=(), action_mask: bool = False) -> int:
    """The IMPALA_ACT_* code of `action_dist`; "multi_discrete" carries its head count (check_heads), action_mask=True
    adds IMPALA_ACT_MASKED (categorical and multi-discrete only)."""
    if not isinstance(action_mask, bool):
        raise ValueError(f"action_mask must be a bool, got {action_mask!r}")
    if action_dist == "multi_discrete":
        code = ACT_MULTI_DISCRETE | len(check_heads(action_heads))
    elif not isinstance(action_dist, str) or action_dist not in ACT_DISTS:
        raise ValueError(f"action_dist must be one of {sorted(ACT_DISTS) + ['multi_discrete']}, got {action_dist!r}")
    else:
        code = ACT_DISTS[action_dist]
    if action_mask and code == ACT_GAUSSIAN:
        raise ValueError("action_mask is for categorical and multi-discrete policies, not action_dist='gaussian'")
    return code | ACT_MASKED if action_mask else code


_ERRORS = {-1: "IMPALA_ERR_BAD_ARG", -2: "IMPALA_ERR_UNSUPPORTED_SHAPE",
           -3: "IMPALA_ERR_WORKSPACE_TOO_SMALL"}

_p = C.c_void_p
_i = C.c_int
_i64 = C.c_int64
_f = C.c_float

# name -> (restype, argtypes); must list every symbol include/impala_b200.h declares
SIGNATURES = {
    "impala_abi_version": (_i, []),
    "impala_compiled_sm": (_i, []),
    "impala_param_layout": (_i, [_i, _i, _i, C.POINTER(_i64), C.POINTER(_i64)]),
    "impala_batch_layout": (_i, [_i, _i, _i, _i, C.POINTER(_i64), C.POINTER(_i64)]),
    "impala_batch_layout_obs": (_i, [_i, _i, _i, _i, _i, C.POINTER(_i64), C.POINTER(_i64)]),
    "impala_ingest": (_i, [_p, _p, _i64, _p]),
    "impala_ingest_shard": (_i, [_p, _p, _i, _i, _i, _i, _i, _i, _p]),
    "impala_ingest_shard_obs": (_i, [_p, _p, _i, _i, _i, _i, _i, _i, _i, _p]),
    "impala_batch_layout_frames": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(_i64), C.POINTER(_i64)]),
    "impala_ingest_shard_frames": (_i, [_p, _p] + [_i] * 8 + [_p]),
    "impala_obs_unstack": (_i, [_p, _i, _p, _i, _i, _i, _i, _i, _p]),
    "impala_batch_compose": (_i, [_p, _p, _i64, _p] + [_i] * 7 + [_p]),
    "impala_obs_u8_to_f32": (_i, [_p, _p, _i64, _p]),
    "impala_obs_normalize_workspace": (_i64, [_i, _i, _i]),
    "impala_obs_normalize": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p, _i64, _p]),
    "impala_obs_norm_update": (_i, [_p, _p, _p, C.c_double, _p, _p, _i64, _i, _i64, _i64, _i, _i64, _i64, _i, _p, _p,
                                    _p, _i64, _i64, _i, _i64, _p, C.c_double, _p]),
    "impala_mlp_forward": (_i, [_p, _p, _p, _i, _i, _i, _i, _p]),
    "impala_mlp_forward_u8": (_i, [_p, _p, _p, _i, _i, _i, _i, _p]),
    "impala_mlp_backward_u8": (_i, [_p, _p, _p, _p, _p, _i64, _i, _i, _i, _i, _p]),
    "impala_launch_count": (C.c_longlong, []),
    "impala_mlp_forward_pair": (_i, [_p] * 5 + [_i] * 6 + [_p]),
    "impala_mlp_backward_workspace": (_i64, [_i, _i, _i, _i]),
    "impala_mlp_backward": (_i, [_p, _p, _p, _p, _p, _i64, _i, _i, _i, _i, _p]),
    "impala_mlp_backward_pair": (_i, [_p] * 8 + [_i64, _p, _i64] + [_i] * 6 + [_p]),
    "impala_mlp_forward_shared": (_i, [_p, _i, _p, _p, _p] + [_i] * 5 + [_p]),
    "impala_mlp_backward_shared": (_i, [_p, _i, _p, _p, _p, _p, _p, _i64] + [_i] * 5 + [_p]),
    "impala_peer_alloc": (_i, [_i64, _p, _p]),
    "impala_peer_open": (_i, [_p, _p]),
    "impala_peer_close": (_i, [_p]),
    "impala_peer_free": (_i, [_p]),
    "impala_peer_push": (_i, [_p, _i64, _p, _p, _i64, _i64, _i, _i, _p]),
    "impala_mlp_backward_pair_push_supported": (_i, [_i] * 6),
    "impala_mlp_backward_pair_push": (_i, [_p] * 6 + [_i64, _p, _i64] + [_i] * 6 + [_p, _i, _p, _p, _i64, _i64, _i, _i, _p]),
    "impala_mlp_backward_pair_push_obs_norm": (_i, [_p] * 6 + [_i64, _p, _i64] + [_i] * 6
                                               + [_p, _i, _p, _p, _i64, _i64, _i, _i, _p]),
    "impala_gather_clip_adam": (_i, [_p] * 4 + [_i64, _i64, _i, _i, _p, _p, _p, _i64, _i64] + [_f] * 5
                                + [_p, _p, C.c_double, _p]),
    "impala_vtrace": (_i, [_p] * 9 + [_i, _i, _i, _f, _f, _f, _i, _p]),
    "impala_vtrace_loss_workspace": (_i64, [_i, _i, _i]),
    "impala_vtrace_loss": (_i, [_p] * 13 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p]),
    "impala_vtrace_loss_diag_workspace": (_i64, [_i, _i, _i]),
    "impala_vtrace_loss_diag": (_i, [_p] * 14 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p]),
    "impala_vtrace_loss_popart": (_i, [_p] * 14 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p, _p]),
    "impala_vtrace_loss_rclip": (_i, [_p] * 13 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p, _p, _i, _p]),
    "impala_vtrace_loss_gauss": (_i, [_p] * 13 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p, _p, _i, _p]),
    "impala_vtrace_loss_md": (_i, [_p] * 13 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p, _p, _i, _p, _i, _p]),
    "impala_vtrace_loss_mask": (_i, [_p] * 13 + [_i64, _i, _i, _i] + [_f] * 7 + [_i, _p, _p, _i, _p, _i, _p]),
    "impala_batch_layout_act": (_i, [_i] * 7 + [C.POINTER(_i64), C.POINTER(_i64)]),
    "impala_ingest_shard_act": (_i, [_p, _p] + [_i] * 9 + [_p]),
    "impala_batch_compose_act": (_i, [_p, _p, _i64, _p] + [_i] * 8 + [_p]),
    "impala_clip_adam": (_i, [_p, _p, _p, _p, _p, _i64, _i64, _f, _f, _f, _f, _f, _p, _p]),
    "impala_clip_optim": (_i, [_p, _p, _p, _p, _p, _i64, _i64, _f, _p, _i64, _i, _f, _f, _f, _p, _p]),
    "impala_gather_clip_optim": (_i, [_p] * 4 + [_i64, _i64, _i, _i, _p, _p, _p, _i64, _i64, _f, _p, _i64, _i]
                                 + [_f] * 3 + [_p, _p, C.c_double, _p]),
    "impala_clip_optim_popart": (_i, [_p, _p, _p, _p, _p, _i64, _i64, _f, _p, _i64, _i, _f, _f, _f, _p, _p]
                                 + [_i64] * 4 + [_f, _p]),
    "impala_gather_clip_optim_popart": (_i, [_p] * 4 + [_i64, _i64, _i, _i, _p, _p, _p, _i64, _i64, _f, _p, _i64, _i]
                                        + [_f] * 3 + [_p, _p, C.c_double, _p] + [_i64] * 4 + [_f, _p]),
    "impala_policy_terms": (_i, [_p, _p, _p, _p, _i, _i, _p]),
    "impala_policy_terms_backward": (_i, [_p, _p, _p, _p, _p, _i, _i, _p]),
    "impala_reduce": (_i, [_p, _p, _i64, _i, _p, _p]),
}

_lib = None


class ImpalaCudaError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImpalaCudaError(
                f"{LIB_PATH} is missing - build it with `python -m torched_impala_b200.build` "
                "(there is no CPU fallback for the learner hot path)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    if rc < 0:
        raise ImpalaCudaError(f"{what}: {_ERRORS.get(rc, rc)}")
    raise ImpalaCudaError(f"{what}: CUDA error {rc}")


def param_layout(O: int, H: int, N2: int):
    offs = (_i64 * 4)()
    total = _i64()
    check(lib().impala_param_layout(O, H, N2, offs, C.byref(total)), "impala_param_layout")
    return list(offs), total.value


def batch_layout(T: int, B: int, O: int, A: int, obs_dtype: str = "float32", frames: int = 1,
                 action_dist: str = "categorical", action_heads=(), action_mask: bool = False):
    """Slab layout for networks of O observation features; frames > 1 stores the O / frames features of
    each stacked frame once (impala_batch_layout_frames); action_dist="gaussian" holds (T, B, 2A) behaviour
    outputs and (T, B, A) float32 actions, "multi_discrete" (T, B, A = sum action_heads) behaviour logits and
    (T, B, K) int32 actions (impala_batch_layout_act); action_mask=True adds the legal word to the actions, (T, B, 2)
    or (T, B, K + 1) int32."""
    offs = (_i64 * 6)()
    total = _i64()
    if action_dist != "categorical" or action_mask:
        if frames < 1 or O % frames:
            raise ValueError(f"{O} observation features do not split into {frames} frames")
        check(lib().impala_batch_layout_act(T, B, O // frames, frames, A, obs_dtype_code(obs_dtype),
                                            act_kind_code(action_dist, action_heads, action_mask), offs,
                                            C.byref(total)),
              "impala_batch_layout_act")
    elif frames == 1:
        check(lib().impala_batch_layout_obs(T, B, O, A, obs_dtype_code(obs_dtype), offs, C.byref(total)),
              "impala_batch_layout_obs")
    else:
        if frames < 1 or O % frames:
            raise ValueError(f"{O} observation features do not split into {frames} frames")
        check(lib().impala_batch_layout_frames(T, B, O // frames, frames, A, obs_dtype_code(obs_dtype), offs,
                                               C.byref(total)), "impala_batch_layout_frames")
    return list(offs), total.value
