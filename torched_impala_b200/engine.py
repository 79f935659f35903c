"""Host-side step engine of the GPU learner: buffers, streams, CUDA graph, peer buffers.

One `LearnerEngine` lives in the learner process of one GPU.  It owns every device
buffer of the update path and enqueues, per learner step, exactly the C-ABI calls of
include/impala_b200.h (PyTorch only provides device memory, streams and
`torch.distributed`):

    impala_ingest              pinned host slab -> device slab (one DMA)        learner.py:104-109,117
    impala_mlp_forward_pair    policy logits (T*B rows) + values ((T+1)*B)      learner.py:112-113
    impala_vtrace_loss         V-trace, 3 losses, dL/dlogits, dL/dv, scalars    learner.py:116-162
      diagnostics=True: impala_vtrace_loss_diag, the same outputs plus eight off-policy sums (ratio
      clipping, KL(behaviour || current), value explained variance) that ride the all-reduce with the scalars
    impala_mlp_backward_pair   parameter gradients of both nets (float64)       learner.py:175
    impala_clip_adam           per-net clip + Adam + step counter               learner.py:176-183
      N > 1 (new; SURVEY 8e): the all-reduce of [grads | scalars] is a PUSH over NVLink peer memory -
      the tail of impala_mlp_backward_pair_push (or impala_peer_push for shapes it does not cover)
      stores this rank's contribution, every value tagged with the step number (LL format), into
      every rank's gather buffer; impala_gather_clip_adam polls its local slots, adds them in rank
      order and applies the update.  IMPALA_ALLREDUCE=nccl: torch.distributed all-reduce between the
      backward and impala_clip_adam instead.
      optimizer="rmsprop" or an lr_lambda (learning-rate schedule): impala_clip_optim /
      impala_gather_clip_optim in place of the two Adam entry points, with the rate of every update read
      from a float32 table in device memory (optim.py) - the captured graphs stay valid for every update.
    popart=True (PopArt value normalization): impala_vtrace_loss_popart in place of the V-trace launch and
      impala_clip_optim_popart / impala_gather_clip_optim_popart in place of the optimizer launch (the default
      Adam as a one-entry table).  The value net outputs normalized values; the statistics (float64 in device
      memory, `popart`) are read by the V-trace kernel and updated, with the value head's output-preserving
      rescale, inside the optimizer launch from the eight V-trace sums that ride `comm`.  No launch is added.
    reward_clip="abs_one" | "soft_asymmetric" (reward clipping): impala_vtrace_loss_rclip in place of whichever
      of the three V-trace launches above the step makes, with the same workspace and outputs.  The kernel
      transforms every reward where it enters V-trace, so the slabs, the replay store and the transport keep raw
      rewards; the logged batch_mean_reward stays raw, the losses, diagnostics and PopArt statistics are in
      clipped-reward units.  No launch is added.
    shared_torso=True (shared-torso actor-critic): ONE network with N + 1 outputs [policy | value] in one parameter
      block in place of the two: impala_mlp_forward_shared / impala_mlp_backward_shared replace the pair entry
      points (and the u8 calls), writing and reading the same logits / values / dlogits / dv buffers, so every
      V-trace launch above runs unchanged.  One clip norm over the whole block (the optimizer's value range is all
      of it, its policy range empty; the norm is logged as norm_policy and norm_value is 0), and PopArt's value
      head is row N of W2 and b2[N].  Data-parallel steps push the
      flat gradient with impala_peer_push.  launches_per_step counts the kernels this route takes (a Wide-plan
      backward adds its reduction launch, where the two networks' paired Narrow backward had none).
    action_dist="gaussian" (continuous actions): A counts action dimensions (at most 16) and the policy has 2A
      outputs [mean | log std] of a diagonal Gaussian.  The slabs hold the behaviour outputs (T, B, 2A) and the
      float32 samples (T, B, A) (impala_batch_layout_act); impala_vtrace_loss_gauss takes the V-trace slot of the
      step with the same flags (diagnostics, PopArt, reward clip) and the same workspace.  No launch is added.
    action_dist="multi_discrete", action_heads=(n_0, .., n_K-1) (a gym MultiDiscrete space): K <= 16 independent
      softmax heads over the A = sum n_k <= 32 policy outputs, head k owning [s_k, s_k + n_k).  The slabs hold the
      behaviour logits (T, B, A) and K int32 indices per step, actions (T, B, K) (impala_batch_layout_act with
      IMPALA_ACT_MULTI_DISCRETE(K)); impala_vtrace_loss_md takes the V-trace slot of the step with the same flags and
      workspace, the head sizes passed by value.  No launch is added.
    action_mask=True (categorical or multi-discrete; invalid-action masking): every step's actions end in one more
      int32, the legal word (bit j: output j is legal), (T, B, 2) or (T, B, K + 1) (impala_batch_layout_act with
      IMPALA_ACT_MASKED); impala_vtrace_loss_mask takes the V-trace slot with the same flags and workspace, pi and mu
      renormalised over the legal entries.  No launch is added.

obs_norm=True (observation normalization): impala_obs_normalize is the step's first launch after any compose. It
replaces the widening / unstacking launch below (one launch more for float32 dense slabs). It writes normalized
float32 rows (T+1, B, O) that every later kernel reads, and the batch's per-feature sums into `comm` after the
logged extras. One launch after the optimizer, impala_obs_norm_update, merges the (rank-summed) sums into float64
running statistics and writes `folded`, the block with its first layers in raw-observation coordinates: what
`state()` returns and the Learner publishes. Byte observations of O > 128 then run the float kernels. Data-parallel:
the sums ride every all-reduce route (the paired backward's fused push, as impala_mlp_backward_pair_push_obs_norm,
impala_peer_push, NCCL); on the peer routes the update kernel adds the ranks' sums in rank order out of the gather
buffer.

obs_dtype="uint8" (byte observations): the slabs hold obs as uint8 (impala_batch_layout_obs).  For
O > 128 the two networks run impala_mlp_{forward,backward}_u8 on the bytes, one after the other as the
pair entry points do at those widths.  For O <= 128 impala_obs_u8_to_f32 widens the obs into a float32
device buffer first (one more launch) and the pair entry points read that.

frames=k > 1 (frame-stacked observations, O = k F): the slabs hold each frame once, obs (T+k, B, F)
(impala_batch_layout_frames), and the step's first launch, impala_obs_unstack, rebuilds the dense (T+1, B, O)
rows into a device buffer the unchanged kernels read: uint8 for the byte kernels (O > 128), the float32 buffer
of the widened path (O <= 128 bytes: it replaces the widening launch), float32 for float32 frames.

With `use_graph=True` the whole launch sequence of a step is captured once per slab into ONE CUDA
graph and replayed (two graphs around the collective in the NCCL scheme).
Ingest is double buffered: two pinned host slabs, two device slabs and
a dedicated copy stream, so the DMA of batch i+1 runs under the kernels of batch i
(`ingest(slot)` / `step(slot)` order themselves with events); the loss scalars come back
through a small ring of pinned buffers (`post_scalars` / `fetch_scalars`) so the host only
ever waits for the previous step.

replay_slabs=R, replay_columns=Br (experience replay, both 0 = off): the host slabs, `fill_host` and the
ingest calls speak the FRESH layout of Bf = B - Br columns, and the DMA of update n lands in slot n mod (R + 2)
of a store of fresh slabs in HBM that keeps the last R fresh batches.  The step's first launch,
impala_batch_compose, gathers the B-column training slab out of the store by the update's plan (replay.py):
its own Bf columns, then Br columns drawn uniformly from the fresh batches of the R updates before it (empty
columns at update 1).  The plan reaches a small device buffer per training slab on the copy stream, ahead of
the event the step waits on, so the captured graphs keep fixed pointers.  R + 2 slots: while update n trains,
the slot that receives update n + 1 is in nobody's pool, so the DMA still runs under the kernels.  The kernels
after the compose launch are unchanged; the logged `batch_mean_reward` scalar is the composed batch's (sum of
all B columns' rewards / B), the mean over the fresh trajectories is the caller's (Learner logs that one).

The keyword options above (obs_dtype, frames, diagnostics, replay_slabs, replay_columns, optimizer, optimizer_kwargs,
popart, popart_beta, reward_clip, action_dist, action_heads, shared_torso, action_mask, obs_norm, obs_norm_eps) are the
fields of `LearnerOptions`.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
import numbers
from typing import NamedTuple

import numpy as np
import torch

from . import _cabi
from .optim import POPART_BETA, check_popart_args, optim_config
from .replay import ReplaySampler, check_replay_args

PKEYS = ("model.0.weight", "model.0.bias", "model.3.weight", "model.3.bias")
SCALAR_NAMES = ("value_fn_loss", "policy_loss", "policy_entropy", "batch_mean_reward")
DIAG_NAMES = ("log_ratio_mean", "rho_clip_fraction", "c_clip_fraction", "kl_behaviour_current",
              "value_explained_variance", "valid_steps")
_BATCH_FIELDS = (("obs", np.float32), ("beh_logits", np.float32), ("actions", np.int32),
                 ("rewards", np.float32), ("done", np.uint8), ("lens", np.int32))
_TORCH_DT = {np.float32: torch.float32, np.int32: torch.int32, np.uint8: torch.uint8}


def diagnostic_values(sums, value_fn_loss: float, global_batch: int) -> dict:
    """The logged off-policy diagnostics from the eight sums of impala_vtrace_loss_diag (all ranks added).

    sum (vs - v)^2 over the valid steps is not summed again: it is 2 B value_fn_loss (the baseline loss
    is 0.5 sum (v - vs)^2 over t <= lens, and its t = lens term is 0).  value_explained_variance =
    1 - Var(vs - v) / Var(vs) (population variances over the valid steps), NaN when n < 2 or Var(vs) <= 0."""
    n, s_lr, n_rho, n_c, s_kl, s_vs, s_vs2, s_err = (float(x) for x in sums)
    nan = float("nan")
    out = {"valid_steps": n}
    if n <= 0:
        out.update(dict.fromkeys(DIAG_NAMES[:5], nan))
        return out
    out.update(log_ratio_mean=s_lr / n, rho_clip_fraction=n_rho / n, c_clip_fraction=n_c / n,
               kl_behaviour_current=s_kl / n)
    var_vs = s_vs2 / n - (s_vs / n) ** 2
    var_err = 2.0 * global_batch * value_fn_loss / n - (s_err / n) ** 2
    out["value_explained_variance"] = 1.0 - var_err / var_vs if n >= 2 and var_vs > 0.0 else nan
    return out


def popart_sigma(mu: float, nu: float) -> float:
    """sigma of the PopArt statistics (mu, nu), as the optimizer kernel forms it."""
    return min(max(max(nu - mu * mu, 0.0) ** 0.5, 1e-4), 1e6)


def check_obs_norm_args(obs_norm, eps, O: int) -> None:
    """The observation-normalization setting, checked before any device work: a bool, a finite eps > 0 and at most
    IMPALA_OBS_NORM_MAX_FEATURES features."""
    if not isinstance(obs_norm, bool):
        raise ValueError(f"obs_norm must be a bool, got {obs_norm!r}")
    if isinstance(eps, bool) or not isinstance(eps, numbers.Real) or not math.isfinite(eps) or not eps > 0:
        raise ValueError(f"obs_norm_eps must be a finite number > 0, got {eps!r}")
    if obs_norm and O > _cabi.OBS_NORM_MAX_FEATURES:
        raise ValueError(f"obs_norm takes at most {_cabi.OBS_NORM_MAX_FEATURES} observation features, got {O}")


def obs_norm_f32(mean, var, eps: float):
    """(mu_f, r_f): the float32 statistics the kernels normalize with, mean and 1 / sqrt(var + eps) rounded."""
    mean, var = np.asarray(mean, np.float64), np.asarray(var, np.float64)
    return mean.astype(np.float32), (1.0 / np.sqrt(var + eps)).astype(np.float32)


def check_shared_torso(shared_torso: bool, H_pi: int, H_v: int, n_policy: int) -> bool:
    """The shared-torso setting, checked before any device work: one hidden layer of H_pi == H_v units and
    n_policy + 1 <= 32 outputs (categorical A <= 31, Gaussian A <= 15)."""
    if not shared_torso:
        return False
    if H_pi != H_v:
        raise ValueError(f"a shared torso has one hidden layer: H_pi ({H_pi}) must equal H_v ({H_v})")
    if n_policy + 1 > 32:
        raise ValueError(f"a shared torso takes at most 31 policy outputs (+ 1 value), got {n_policy}")
    return True


class CheckedOptions(NamedTuple):
    """What `LearnerOptions.check` derives from the options and the shapes."""
    B_fresh: int           # columns of an update that arrive from the host (B without replay)
    N_pi: int              # policy outputs: A, or 2A [mean | log std] for a Gaussian policy (multi-discrete: A)
    obs_code: int          # IMPALA_OBS_*
    act_kind: int          # IMPALA_ACT_* (multi-discrete: IMPALA_ACT_MULTI_DISCRETE(K))
    reward_clip_code: int  # IMPALA_REWARD_CLIP_*, 0 = none


@dataclasses.dataclass(frozen=True)
class LearnerOptions:
    """The learner's feature options (module docstring): `Learner` and `LearnerEngine` keywords, JSON for the worker
    ranks of a data-parallel learner.  The schedule is not one: a lambda is not JSON, its table travels apart."""
    obs_dtype: str = "float32"
    frames: int = 1
    diagnostics: bool = False
    replay_slabs: int = 0
    replay_columns: int = 0
    optimizer: str = "adam"
    optimizer_kwargs: dict = dataclasses.field(default_factory=dict)
    popart: bool = False
    popart_beta: float = POPART_BETA
    reward_clip: str | None = None
    action_dist: str = "categorical"
    # multi_discrete: the head sizes (n_0, .., n_K-1), sum = A, a tuple whatever sequence came in (a JSON list on the
    # worker ranks: Learner._cfg carries it and engine_from_cfg passes it on).  Init-only rather than a field, so that
    # dataclasses.asdict / fields list the options every action distribution has; compared by __eq__ like a field.
    # dataclasses.replace does not carry it: pass action_heads= again.
    action_heads: dataclasses.InitVar[tuple] = ()
    shared_torso: bool = False
    # invalid-action masking (categorical and multi-discrete): every step carries a legal word in its actions.
    # Init-only like action_heads (Learner._cfg carries it, engine_from_cfg passes it when true).
    action_mask: dataclasses.InitVar[bool] = False
    # observation normalization: running per-feature mean and variance of the raw observations, folded into the
    # published weights (module docstring).  Init-only like action_mask (Learner._cfg carries both, engine_from_cfg
    # passes them when obs_norm is true).
    obs_norm: dataclasses.InitVar[bool] = False
    obs_norm_eps: dataclasses.InitVar[float] = 1e-8

    def __post_init__(self, action_heads, action_mask, obs_norm, obs_norm_eps):
        object.__setattr__(self, "optimizer_kwargs", dict(self.optimizer_kwargs or {}))
        # a tuple whatever sequence came in; check() refuses bad entries
        heads = tuple(action_heads) if isinstance(action_heads, (list, tuple)) else action_heads
        object.__setattr__(self, "action_heads", heads)
        object.__setattr__(self, "action_mask", action_mask)
        object.__setattr__(self, "obs_norm", obs_norm)
        object.__setattr__(self, "obs_norm_eps", obs_norm_eps)

    def __eq__(self, other):
        if other.__class__ is not self.__class__:
            return NotImplemented
        return self.action_heads == other.action_heads and self.action_mask is other.action_mask and \
            self.obs_norm is other.obs_norm and self.obs_norm_eps == other.obs_norm_eps and all(
            getattr(self, f.name) == getattr(other, f.name) for f in dataclasses.fields(self))

    def check(self, B: int, O: int, A: int, H_pi: int, H_v: int, world: int = 1) -> CheckedOptions:
        """Refuse options that B columns per update, O features, A actions (Gaussian: action dimensions), hidden
        widths H_pi, H_v and `world` devices cannot take.  optim_config checks the optimizer and its keywords."""
        obs_code = _cabi.obs_dtype_code(self.obs_dtype)
        if self.frames < 1 or O % self.frames:
            raise ValueError(f"{O} observation features do not split into {self.frames} stacked frames")
        if self.action_dist == "multi_discrete":
            if not isinstance(self.action_heads, tuple):
                raise ValueError(f"action_heads must be a sequence of head sizes, got {self.action_heads!r}")
            heads = _cabi.check_heads(self.action_heads)
            if sum(heads) != A:
                raise ValueError(f"the heads {heads} of a multi-discrete policy have {sum(heads)} outputs; the policy "
                                 f"has A = {A}")
        elif self.action_heads != ():
            raise ValueError(f"action_heads is for action_dist='multi_discrete', not {self.action_dist!r}")
        act_kind = _cabi.act_kind_code(self.action_dist, self.action_heads, self.action_mask)
        if self.action_mask and A > _cabi.MAX_OUTPUTS:
            raise ValueError(f"action_mask takes at most {_cabi.MAX_OUTPUTS} policy outputs (one 32-bit legal word), "
                             f"got A = {A}")
        gaussian = act_kind == _cabi.ACT_GAUSSIAN
        if gaussian and not 1 <= A <= _cabi.MAX_GAUSSIAN_DIMS:
            raise ValueError(f"a Gaussian policy takes 1 to {_cabi.MAX_GAUSSIAN_DIMS} action dimensions (2A outputs "
                             f"[mean | log std]), got A = {A}")
        N_pi = 2 * A if gaussian else A
        check_shared_torso(self.shared_torso, H_pi, H_v, N_pi)
        reward_clip_code = _cabi.reward_clip_code(self.reward_clip)
        check_popart_args(self.popart, self.popart_beta)
        check_obs_norm_args(self.obs_norm, self.obs_norm_eps, O)
        B_fresh = check_replay_args(B, self.replay_slabs, self.replay_columns)
        if self.replay_slabs and world > 1:
            raise ValueError(f"experience replay runs on one device, not {world}: the store is not sharded")
        return CheckedOptions(B_fresh, N_pi, obs_code, act_kind, reward_clip_code)


def engine_from_cfg(cfg: dict, world: int, device, process_group=None, lr_table=None) -> LearnerEngine:
    """The engine of one of `world` ranks from a Learner's JSON config (`Learner._cfg`) and learning-rate table:
    rank 0 and every data-parallel worker rank build theirs here, so all of them train with the same options."""
    from .utils import Hyperparameters

    if cfg["B"] % world:
        raise ValueError(f"batch_size {cfg['B']} does not divide over {world} devices")
    return LearnerEngine(cfg["T"], cfg["B"] // world, cfg["O"], cfg["A"], cfg["H_pi"], cfg["H_v"],
                         Hyperparameters(**cfg["hp"]), global_batch=cfg["B"], device=device, mode=cfg["mode"],
                         process_group=process_group, lr_table=lr_table,
                         **{f.name: cfg[f.name] for f in dataclasses.fields(LearnerOptions)},
                         **({"action_heads": tuple(cfg["action_heads"])} if cfg.get("action_heads") else {}),
                         **({"action_mask": True} if cfg.get("action_mask") else {}),
                         **({"obs_norm": True, "obs_norm_eps": cfg["obs_norm_eps"]} if cfg.get("obs_norm") else {}))


def _ptr(t: torch.Tensor) -> C.c_void_p:
    return C.c_void_p(t.data_ptr())


class _NoCtx:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


_NO_CTX = _NoCtx()


class LearnerEngine:
    def __init__(self, T: int, B_local: int, O: int, A: int, H_pi: int, H_v: int, hp,
                 global_batch: int | None = None, device: str | torch.device = "cuda:0",
                 mode: str = "reference", process_group=None, use_graph: bool = True, slabs: int = 2,
                 replay_seed: int = 0, lr_lambda=None, lr_table=None, **options):
        # the options, the update rule and the schedule, checked before any device work; the default rule - Adam at
        # 0.95 * hp.lr - keeps impala_clip_adam with the rate as a launch argument
        o = self.options = LearnerOptions(**options)
        self.optim = optim_config(hp, o.optimizer, o.optimizer_kwargs, lr_lambda, lr_table)
        self.pg = process_group
        self.world = 1
        if process_group is not None:
            import torch.distributed as dist

            self.world = dist.get_world_size(process_group)
        # B_fresh of the B columns of an update arrive from the host (the rest from the replay store)
        self.B_fresh, self.N_pi, self.obs_code, self.act_kind, self.reward_clip_code = o.check(
            B_local, O, A, H_pi, H_v, self.world)
        if not torch.cuda.is_available():
            raise _cabi.ImpalaCudaError("LearnerEngine needs a CUDA device; there is no CPU path")
        self.lib = _cabi.lib()
        # the options the step reads; every rank must agree on diagnostics and PopArt (the length of `comm`)
        self.gaussian = self.act_kind == _cabi.ACT_GAUSSIAN
        # multi-discrete: the head sizes (K = len), passed by value to every impala_vtrace_loss_md call
        self.heads = tuple(int(n) for n in o.action_heads) if o.action_dist == "multi_discrete" else ()
        self.md_heads = (C.c_int32 * len(self.heads))(*self.heads) if self.heads else None
        # action_mask: one more int32 per step in the actions, the legal word (impala_vtrace_loss_mask)
        self.masked = bool(o.action_mask)
        self.shared_torso, self.popart, self.diagnostics = bool(o.shared_torso), bool(o.popart), bool(o.diagnostics)
        self.popart_beta, self.replay_slabs = float(o.popart_beta), int(o.replay_slabs)
        self.frames, self.F = o.frames, O // o.frames
        self.obs_norm, self.obs_norm_eps = bool(o.obs_norm), float(o.obs_norm_eps)
        self.dev = torch.device(device)
        torch.cuda.set_device(self.dev)
        self.T, self.B, self.O, self.A, self.H_pi, self.H_v = T, B_local, O, A, H_pi, H_v
        self.hp = hp
        # logged float64 values after the gradient in `comm`; PopArt forms its statistics from the eight sums
        self.n_extra = 12 if o.diagnostics or o.popart else 4
        self.mode = _cabi.MODES[mode]
        self.global_batch = int(global_batch if global_batch is not None else B_local * self.world)
        self.inv_batch = 1.0 / self.global_batch
        self.use_graph = use_graph
        self.stream = torch.cuda.Stream(device=self.dev)
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.launches_per_step = 0

        # ---- parameter blocks: [policy | value_fn], float32, 128-byte aligned tensors.  Shared torso: one block of
        # N_pi + 1 outputs, n_pi = n_total (n_clip below sets how the optimizer clips it)
        if self.shared_torso:
            self.pi_off, self.n_pi = _cabi.param_layout(O, H_pi, self.N_pi + 1)
            self.vf_off, self.n_vf = None, 0
        else:
            self.pi_off, self.n_pi = _cabi.param_layout(O, H_pi, self.N_pi)
            self.vf_off, self.n_vf = _cabi.param_layout(O, H_v, 1)
        self.n_total = self.n_pi + self.n_vf
        # the optimizer clips [0, n_clip) and [n_clip, n_total) separately.  Shared torso: one range, the whole
        # block, as the value range (PopArt's value head must lie in it); its norm is logged as norm_policy
        self.n_clip = 0 if self.shared_torso else self.n_pi
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.params = torch.zeros(self.n_total, **f32)
        self.adam_m = torch.zeros(self.n_total, **f32)
        self.adam_v = torch.zeros(self.n_total, **f32)
        self.adam_step = torch.zeros(3, dtype=torch.int64, device=self.dev)  # step, beta1^t, beta2^t bits
        # float64 [gradient | 4 loss scalars | (diagnostics: 8 off-policy sums |) (obs_norm: the batch's observation
        # sums, 2 O + 1 |) pad]: the all-reduce payload
        self.obs_sums_at = self.n_total + self.n_extra
        self.n_comm = self.obs_sums_at + (2 * O + 1 if self.obs_norm else 0) + 4
        self.comm = torch.zeros(self.n_comm, dtype=torch.float64, device=self.dev)
        self.norms = torch.zeros(2, dtype=torch.float64, device=self.dev)
        # the schedule (rmsprop or an lr_lambda): update n reads entry min(n - 1, len - 1); the state buffers
        # keep their Adam names, RMSprop's square_avg lives in adam_v and its momentum buffer in adam_m
        self.lr_table = (None if self.optim.lr_table is None
                         else torch.from_numpy(self.optim.lr_table.copy()).to(self.dev))
        if self.popart and self.lr_table is None:  # the default Adam through the table entry point: same bits
            self.lr_table = torch.tensor([self.optim.lr_scalar], dtype=torch.float32, device=self.dev)
        # PopArt statistics {mu, nu, sigma, mu_loss, sigma_loss} (IMPALA_POPART_STATS), a fresh run at mu 0, nu 1
        self.popart_buf = torch.tensor([0.0, 1.0, 1.0, 0.0, 1.0], dtype=torch.float64, device=self.dev)
        # the value head inside `params`: W2 (1 x H_v) and b2 (shared torso: row N_pi of W2 and b2[N_pi])
        if self.shared_torso:
            self.w2_at, self.b2_at = self.pi_off[2] + self.N_pi * H_pi, self.pi_off[3] + self.N_pi
        else:
            self.w2_at, self.b2_at = self.n_pi + self.vf_off[2], self.n_pi + self.vf_off[3]

        # ---- batch slab (device) and pinned staging slabs (host), identical layouts (replay: the host slabs
        # hold the B_fresh columns that cross the host link, the device slabs the B columns trained on)
        train_off, train_bytes = _cabi.batch_layout(T, B_local, O, A, o.obs_dtype, o.frames, o.action_dist,
                                                    o.action_heads, o.action_mask)
        self.slab_off, self.slab_bytes = train_off, train_bytes
        if self.replay_slabs:
            self.slab_off, self.slab_bytes = _cabi.batch_layout(T, self.B_fresh, O, A, o.obs_dtype, o.frames,
                                                                o.action_dist, o.action_heads, o.action_mask)
        self.fields = ((("obs", np.uint8 if o.obs_dtype == "uint8" else np.float32),) + _BATCH_FIELDS[1:])
        if self.gaussian:  # float32 action samples
            self.fields = self.fields[:2] + (("actions", np.float32),) + self.fields[3:]
        self.n_slabs = slabs
        self.d_slabs = [torch.zeros(train_bytes, dtype=torch.uint8, device=self.dev)
                        for _ in range(slabs)]
        self.h_slabs = [torch.zeros(self.slab_bytes, dtype=torch.uint8).pin_memory()
                        for _ in range(slabs)]
        self.shapes = self._shapes(B_local)
        h_shapes = self._shapes(self.B_fresh)
        self.d_views, self.h_views = [], []
        for dslab, hslab in zip(self.d_slabs, self.h_slabs):
            arr = hslab.numpy()
            dv, hv = {}, {}
            for (name, dt), d_off, h_off in zip(self.fields, train_off, self.slab_off):
                item = np.dtype(dt).itemsize
                nd, nh = int(np.prod(self.shapes[name])) * item, int(np.prod(h_shapes[name])) * item
                dv[name] = dslab[d_off:d_off + nd].view(_TORCH_DT[dt]).view(self.shapes[name])
                hv[name] = arr[h_off:h_off + nh].view(dt).reshape(h_shapes[name])
            self.d_views.append(dv)
            self.h_views.append(hv)
        self.d = self.d_views[0]
        self.slab_ready = [torch.cuda.Event() for _ in range(slabs)]  # H2D into slab done
        self.slab_free = [torch.cuda.Event() for _ in range(slabs)]   # last consumer of slab done
        self._slab_used = [False] * slabs
        if self.replay_slabs:
            self.sampler = ReplaySampler(replay_seed, self.replay_slabs, self.B_fresh, o.replay_columns)
            self.store = torch.zeros(self.replay_slabs + 2, self.slab_bytes, dtype=torch.uint8, device=self.dev)
            self.d_plans = [torch.zeros(B_local, 2, dtype=torch.int32, device=self.dev) for _ in range(slabs)]
            self.h_plans = [torch.zeros(B_local, 2, dtype=torch.int32).pin_memory() for _ in range(slabs)]
            self.replay_plan = None  # plan of the last ingested update: (B, 2) int32 (store slot, column)
            self._slab_update = [0] * slabs  # update number held by each training slab
            self._ingested = self._stepped = 0  # updates whose DMA / whose step has been enqueued
            self._update_done = [torch.cuda.Event() for _ in range(3)]  # store reads of update u: index u % 3

        # ---- activations / gradients of the non-MLP part
        self.logits = torch.zeros(T, B_local, self.N_pi, **f32)
        self.values = torch.zeros(T + 1, B_local, **f32)
        self.vs = torch.zeros(T + 1, B_local, **f32)
        self.pg_adv = torch.zeros(T, B_local, **f32)
        self.dlogits = torch.zeros(T, B_local, self.N_pi, **f32)
        self.dv = torch.zeros(T + 1, B_local, **f32)
        self.M_pi, self.M_vf = T * B_local, (T + 1) * B_local
        if self.shared_torso:  # one backward over the (T + 1) B rows; ws_pi is its workspace
            self.ws_pi_bytes = self._ws_bytes(self.M_vf, O, H_pi, self.N_pi + 1)
            self.ws_vf_bytes = 0
        else:
            self.ws_pi_bytes = self._ws_bytes(self.M_pi, O, H_pi, self.N_pi)
            self.ws_vf_bytes = self._ws_bytes(self.M_vf, O, H_v, 1)
        self.ws_pi = torch.zeros(self.ws_pi_bytes, dtype=torch.uint8, device=self.dev)
        self.ws_vf = torch.zeros(self.ws_vf_bytes, dtype=torch.uint8, device=self.dev)
        # byte observations: O > 128 runs the networks on the bytes (impala_mlp_{forward,backward}_u8); narrower
        # observations are widened once per step into this float32 copy for the float kernels
        self.obs_u8_native = o.obs_dtype == "uint8" and O > 128 and not self.obs_norm
        self.obs_f32 = (torch.zeros((T + 1) * B_local * O, **f32)
                        if o.obs_dtype == "uint8" and not self.obs_u8_native and not self.obs_norm else None)
        # frames > 1: the dense rows the kernels read, rebuilt from the slab's frames once per step
        self.obs_dense = None
        if o.frames > 1 and not self.obs_norm:
            self.obs_dense = self.obs_f32 if self.obs_f32 is not None else torch.zeros(
                (T + 1) * B_local * O, dtype=torch.uint8 if self.obs_u8_native else torch.float32, device=self.dev)
        # obs_norm: impala_obs_normalize writes the normalized float32 rows every later kernel reads (in place of the
        # widening / unstacking launch), impala_obs_norm_update the statistics and the folded block after the optimizer
        self.obs_normed = self.folded = None
        # (W1 offset, b1 offset, H) of each network in `params`
        self.w1_nets = ((self.pi_off[0], self.pi_off[1], H_pi),) if self.shared_torso else (
            (self.pi_off[0], self.pi_off[1], H_pi), (self.n_pi + self.vf_off[0], self.n_pi + self.vf_off[1], H_v))
        if self.obs_norm:
            self.obs_normed = torch.zeros((T + 1) * B_local * O, **f32)
            self.folded = torch.zeros(self.n_total, **f32)
            # [count | mean (O) | var (O)] float64 and the kernels' float32 [mu_f (O) | r_f (O)]; fresh: 0, 0, 1
            self.obs_stats = torch.zeros(1 + 2 * O, dtype=torch.float64, device=self.dev)
            self.obs_norm_dev = torch.zeros(2 * O, **f32)
            self._set_obs_stats(0.0, np.zeros(O), np.ones(O))
            n = int(self.lib.impala_obs_normalize_workspace(T, B_local, O))
            _cabi.check(min(n, 0), "impala_obs_normalize_workspace")
            self.obs_norm_ws = torch.zeros(n, dtype=torch.uint8, device=self.dev)  # counters zeroed once
            self.obs_norm_ctl = torch.zeros(2, dtype=torch.int32, device=self.dev)
        ws_fn = (self.lib.impala_vtrace_loss_diag_workspace if self.n_extra == 12
                 else self.lib.impala_vtrace_loss_workspace)
        self.ws_vt_bytes = int(ws_fn(T, B_local, A))
        self.ws_vt = torch.zeros(self.ws_vt_bytes, dtype=torch.uint8, device=self.dev)  # zeroed once
        # ring of 4 tickets: [4 scalars | 2 norms | peer error | pad (| 8 off-policy sums) (| 5 PopArt statistics |
        # pad)]
        self.h_scalars = torch.zeros(4, 24 if o.popart else 16 if o.diagnostics else 8,
                                     dtype=torch.float64).pin_memory()
        self._scalar_events = [torch.cuda.Event() for _ in range(4)]
        self._ticket = 0

        self._loop_thread = None  # thread whose current stream IS self.stream for a whole update loop (loop_stream)
        self._graph_main = {}  # slab slot -> captured step
        self._graph_opt = None
        self._main_launches = 0
        self.steps_done = 0
        self.peer = None
        if self.world > 1:
            self._setup_peer_allreduce()

    # ------------------------------------------------------------------ parameters
    # ------------------------------------------------------------------------ multi-GPU plumbing
    def _setup_peer_allreduce(self) -> None:
        """Allocate this rank's gather buffer (LL elements, 16 bytes per float64) and map every peer's
        (CUDA IPC over NVLink) for the push-model all-reduce.  IMPALA_ALLREDUCE=nccl - or a failed mapping on ANY rank -
        keeps the torch.distributed all-reduce between the backward and the optimizer instead."""
        import os
        import warnings

        import torch.distributed as dist

        rank, world = dist.get_rank(self.pg), self.world
        ok, err, mine = os.environ.get("IMPALA_ALLREDUCE", "peer") != "nccl" and world <= 8, "", {}
        lib = self.lib
        if ok:
            try:
                for name, nbytes in (("gather", self.gather_bytes(world)),):
                    ptr, handle = C.c_void_p(), (C.c_char * 64)()
                    _cabi.check(lib.impala_peer_alloc(nbytes, C.byref(ptr), handle), "impala_peer_alloc")
                    mine[name] = (ptr.value, bytes(handle.raw))
            except Exception as e:  # noqa: BLE001 - reported below, all ranks fall back together
                ok, err = False, repr(e)
        handles = [None] * world
        dist.all_gather_object(handles, {k: v[1] for k, v in mine.items()} if ok else None, group=self.pg)
        ok = ok and all(h is not None for h in handles)
        ptrs = {"gather": []}
        opened = []
        if ok:
            try:
                for r, h in enumerate(handles):
                    for name in ("gather",):
                        if r == rank:
                            ptrs[name].append(mine[name][0])
                        else:
                            ptr = C.c_void_p()
                            _cabi.check(lib.impala_peer_open(h[name], C.byref(ptr)), f"impala_peer_open(rank {r})")
                            opened.append(ptr.value)
                            ptrs[name].append(ptr.value)
            except Exception as e:  # noqa: BLE001
                ok, err = False, repr(e)
        agree = torch.tensor([1 if ok else 0], device=self.dev)
        dist.all_reduce(agree, op=dist.ReduceOp.MIN, group=self.pg)
        if int(agree.item()) == 0:
            if os.environ.get("IMPALA_ALLREDUCE", "peer") != "nccl" and rank == 0:
                warnings.warn(f"peer-memory all-reduce unavailable ({err or 'a rank could not map its peers'}); "
                              "using the NCCL all-reduce between backward and optimizer")
            return
        self._use_peers(mine["gather"][0], ptrs["gather"], rank, world, opened=opened)
        torch.cuda.synchronize(self.dev)
        dist.barrier(group=self.pg)

    def gather_bytes(self, world: int) -> int:
        """Bytes of one rank's gather buffer for `world` ranks: 2 parities x `world` slots of n_comm LL elements
        (16 bytes per float64)."""
        return 2 * 16 * world * self.n_comm

    def _use_peers(self, gather_ptr: int, gather_ptrs, rank: int, world: int, timeout_s: float | None = None,
                   opened=()) -> None:
        """Make the step exchange `comm` by the push over peer memory as rank `rank` of `world`: gather_ptr is this
        rank's zero-filled gather buffer (gather_bytes(world) bytes, 16-byte aligned), gather_ptrs every rank's as
        this process addresses it.  _setup_peer_allreduce calls it with the mapped IPC buffers; any device addresses
        serve (several simulated ranks on one device, each with its own buffer).  timeout_s=None: the
        IMPALA_PEER_TIMEOUT_S environment variable, 600 s by default."""
        import os

        if not 1 <= world <= 8 or not 0 <= rank < world or len(gather_ptrs) != world:
            raise ValueError(f"rank {rank} of {world} with {len(gather_ptrs)} gather buffers (1 to 8 ranks)")
        if self.replay_slabs and world > 1:
            raise ValueError(f"experience replay runs on one device, not {world}: the store is not sharded")
        i64 = dict(dtype=torch.int64, device=self.dev)
        # the fused push is the paired backward's; a shared torso pushes `comm` after its backward
        fused = not self.shared_torso and bool(self.lib.impala_mlp_backward_pair_push_supported(
            self.M_pi, self.M_vf, self.O, self.H_pi, self.H_v, self.N_pi))
        if os.environ.get("IMPALA_PUSH_FUSED", "1") == "0":
            fused = False
        if timeout_s is None:
            timeout_s = float(os.environ.get("IMPALA_PEER_TIMEOUT_S", "600"))
        slot = self.n_comm                              # LL elements per rank slot: [gradient | scalars | pad]
        self.world = world
        self.peer = dict(gather=int(gather_ptr), opened=list(opened),
                         gather_ptrs=torch.tensor([int(p) for p in gather_ptrs], **i64),
                         seq=torch.zeros(1, **i64), rank=rank, slot=slot, buf=world * slot, fused=fused,
                         err=torch.zeros(1, dtype=torch.int32, device=self.dev), timeout_s=float(timeout_s))

    def _shapes(self, B: int) -> dict:
        """Shapes of the six batch tensors in a slab of B columns."""
        T, A = self.T, self.A
        K = (len(self.heads) or 1) + 1 if self.masked else len(self.heads)  # the indices, then the legal word
        return {"obs": (T + self.frames, B, self.F), "beh_logits": (T, B, self.N_pi),
                "actions": (T, B, A) if self.gaussian else (T, B, K) if self.heads or self.masked else (T, B),
                "rewards": (T, B), "done": (T, B), "lens": (B,)}

    def _ws_bytes(self, M, O, H, N2):
        n = self.lib.impala_mlp_backward_workspace(M, O, H, N2)
        if n < 0:
            _cabi.check(int(n), f"impala_mlp_backward_workspace(M={M},O={O},H={H},N2={N2})")
        return int(n)

    def _segments(self):
        """(group, key, flat offset, shape) of every parameter tensor in `self.params`.  Shared torso: the
        policy view (W1, b1, W2[:N], b2[:N]) and the value view (W1, b1, W2[N:], b2[N:]) of the one block; the
        two views share W1 and b1."""
        O, N = self.O, self.N_pi
        if self.shared_torso:
            H, o = self.H_pi, self.pi_off
            for key, off, shp in zip(PKEYS, o, ((H, O), (H,), (N, H), (N,))):
                yield "policy", key, off, shp
            for key, off, shp in zip(PKEYS, (o[0], o[1], o[2] + N * H, o[3] + N), ((H, O), (H,), (1, H), (1,))):
                yield "value_fn", key, off, shp
            return
        shp_pi = ((self.H_pi, O), (self.H_pi,), (N, self.H_pi), (N,))
        shp_vf = ((self.H_v, O), (self.H_v,), (1, self.H_v), (1,))
        for key, off, shp in zip(PKEYS, self.pi_off, shp_pi):
            yield "policy", key, off, shp
        for key, off, shp in zip(PKEYS, self.vf_off, shp_vf):
            yield "value_fn", key, self.n_pi + off, shp

    def load_state(self, state: dict, popart: dict | None = None, obs_norm: dict | None = None) -> None:
        """state = {"policy": state_dict, "value_fn": state_dict} (any float dtype, CPU).

        With PopArt the value function is taken FOLDED, in reward units (what `state()` returns): popart =
        {"mu": mu, "nu": nu} sets the statistics and unfolds W2 / sigma, (b2 - mu) / sigma (in float64) into the
        normalized head; popart=None starts from mu = 0, nu = 1, where the folded head is the normalized one.

        Shared torso: the torso (W1, b1) and the policy head come from "policy", the value head (W2 of one row,
        b2 of one entry) from "value_fn"; the value function's first layer is ignored, so a two-network state
        loads with the policy's torso.  load_state(state()) restores the block exactly.

        With obs_norm the first layers are taken FOLDED into raw-observation coordinates too (what `state()` returns):
        obs_norm = {"count", "mean", "var"} sets the statistics, and W1 = W1' / r_f, b1 = b1' + W1' mu_f (float64, with
        the float32 mu_f, r_f the kernels use, obs_norm_f32) unfolds each network's first layer; obs_norm=None starts
        from count 0, mean 0, var 1."""
        if popart is not None and not self.popart:
            raise ValueError("PopArt statistics given to an engine built with popart=False")
        if obs_norm is not None and not self.obs_norm:
            raise ValueError("observation statistics given to an engine built with obs_norm=False")
        mu, nu = (0.0, 1.0) if popart is None else (float(popart["mu"]), float(popart["nu"]))
        sigma = popart_sigma(mu, nu)
        flat = torch.zeros(self.n_total, dtype=torch.float32)
        for grp, key, off, shp in self._segments():
            if self.shared_torso and grp == "value_fn" and key in PKEYS[:2]:
                continue
            t = torch.as_tensor(np.asarray(state[grp][key]) if not torch.is_tensor(state[grp][key])
                                else state[grp][key].detach().cpu())
            if tuple(t.shape) != tuple(shp):
                raise ValueError(f"{grp}.{key}: expected {shp}, got {tuple(t.shape)}")
            if self.popart and grp == "value_fn" and key in PKEYS[2:]:
                t = t.to(torch.float64)
                t = t / sigma if key == PKEYS[2] else (t - mu) / sigma
            flat[off:off + t.numel()] = t.reshape(-1).to(torch.float32)
        if self.obs_norm:
            self.folded.copy_(flat)
            O = self.O
            count, mean, var = ((0.0, np.zeros(O), np.ones(O)) if obs_norm is None else
                                (float(obs_norm["count"]), np.asarray(obs_norm["mean"], np.float64).reshape(-1),
                                 np.asarray(obs_norm["var"], np.float64).reshape(-1)))
            if mean.shape != (O,) or var.shape != (O,) or not count >= 0 or not (var >= 0).all():
                raise ValueError(f"obs_norm statistics need a count >= 0 and mean, var of {O} features (var >= 0)")
            mu_f, r_f = (x.astype(np.float64) for x in obs_norm_f32(mean, var, self.obs_norm_eps))
            for grp, (w1, b1, H) in zip(("policy", "value_fn"), self.w1_nets):
                W = np.asarray(torch.as_tensor(state[grp][PKEYS[0]]).detach().cpu().to(torch.float64))
                b = np.asarray(torch.as_tensor(state[grp][PKEYS[1]]).detach().cpu().to(torch.float64))
                flat[w1:w1 + H * O] = torch.from_numpy((W / r_f).reshape(-1))
                flat[b1:b1 + H] = torch.from_numpy(b + W @ mu_f)
            self._set_obs_stats(count, mean, var)
        self.params.copy_(flat)
        if self.popart:
            self.popart_buf.copy_(torch.tensor([mu, nu, sigma, mu, sigma], dtype=torch.float64))
        torch.cuda.synchronize(self.dev)

    def _set_obs_stats(self, count: float, mean, var) -> None:
        mu_f, r_f = obs_norm_f32(mean, var, self.obs_norm_eps)
        self.obs_stats.copy_(torch.from_numpy(np.concatenate([[count], mean, var]).astype(np.float64)))
        self.obs_norm_dev.copy_(torch.from_numpy(np.concatenate([mu_f, r_f])))

    def obs_norm_stats(self) -> dict:
        """The current observation statistics {"count": float, "mean", "var": float64 arrays of O} (waits for the
        stream); var is 1 where nothing has been counted."""
        self.stream.synchronize()
        st = self.obs_stats.cpu().numpy()
        return {"count": float(st[0]), "mean": st[1:1 + self.O].copy(), "var": st[1 + self.O:].copy()}

    def popart_stats(self) -> dict:
        """The current PopArt statistics {"mu", "nu", "sigma"} (float; waits for the stream)."""
        self.stream.synchronize()
        mu, nu, sigma = self.popart_buf[:3].tolist()
        return {"mu": mu, "nu": nu, "sigma": sigma}

    def state(self, dtype=torch.float64) -> dict:
        """Reference-format state_dicts (CPU, float64 like reference models.py:6).  obs_norm: the first layers folded
        into raw-observation coordinates (the block impala_obs_norm_update wrote), which is what actors run."""
        self.stream.synchronize()
        flat = (self.folded if self.obs_norm else self.params).detach().cpu()
        out = {"policy": {}, "value_fn": {}}
        mu, _, sigma = self.popart_buf[:3].tolist() if self.popart else (0.0, 1.0, 1.0)
        for grp, key, off, shp in self._segments():
            n = int(np.prod(shp))
            t = flat[off:off + n].reshape(shp)
            if self.popart and grp == "value_fn" and key in PKEYS[2:]:  # folded: the value in reward units
                t = t.to(torch.float64) * sigma + (mu if key == PKEYS[3] else 0.0)
            out[grp][key] = t.to(dtype).clone()
        return out

    def normalized_state(self, dtype=torch.float64) -> dict:
        """Like `state()`, but the networks as the engine holds them (the value function normalized under PopArt, the
        first layers reading normalized observations under obs_norm)."""
        self.stream.synchronize()
        flat = self.params.detach().cpu()
        out = {"policy": {}, "value_fn": {}}
        for grp, key, off, shp in self._segments():
            n = int(np.prod(shp))
            out[grp][key] = flat[off:off + n].reshape(shp).to(dtype).clone()
        return out

    def grads(self) -> dict:
        """Last step's pre-clip gradient (float64), reference state_dict layout."""
        self.stream.synchronize()
        flat = self.comm[: self.n_total].detach().cpu()
        out = {"policy": {}, "value_fn": {}}
        for grp, key, off, shp in self._segments():
            n = int(np.prod(shp))
            out[grp][key] = flat[off:off + n].reshape(shp).numpy().copy()
        return out

    # ---------------------------------------------------------------------- ingest
    def host_batch(self, slot: int = 0) -> dict:
        """Writable numpy views of pinned staging slab `slot` (fill these, then ingest)."""
        return self.h_views[slot]

    def fill_host(self, batch: dict, slot: int = 0) -> None:
        for name, _ in self.fields:
            if name == "obs" and self.options.obs_dtype == "uint8" and np.asarray(batch["obs"]).dtype != np.uint8:
                raise ValueError("a uint8-observation engine takes uint8 obs arrays")
            np.copyto(self.h_views[slot][name], batch[name])

    def ingest(self, slot: int = 0) -> None:
        """Async H2D of pinned slab `slot` into device slab `slot` on the copy stream."""
        cs = self.copy_stream
        if self._slab_used[slot]:
            cs.wait_event(self.slab_free[slot])  # the step that last read this slab is done
        _cabi.check(self.lib.impala_ingest(self._ingest_target(slot),
                                           C.c_void_p(self.h_slabs[slot].data_ptr()),
                                           self.slab_bytes, C.c_void_p(cs.cuda_stream)),
                    "impala_ingest")
        self.slab_ready[slot].record(cs)

    def _ingest_target(self, slot: int) -> C.c_void_p:
        """Device address the DMA for training slab `slot` writes: the slab itself, or with replay the store
        slot of the update being ingested, after the update's plan has been queued on the copy stream."""
        if not self.replay_slabs:
            return _ptr(self.d_slabs[slot])
        n, cs = self._ingested + 1, self.copy_stream
        if self._stepped < n - 2:
            raise RuntimeError(f"replay: update {n} ingested before the step of update {n - 2} was enqueued; its "
                               "store slot may still be read (at most two updates in flight)")
        if n > 2:  # the store slot last held update n - R - 2, which update n - 2 may have sampled
            cs.wait_event(self._update_done[(n - 2) % 3])
        self.slab_ready[slot].synchronize()  # the pinned plan buffer's previous copy has left the host
        plan = self.sampler.plan(n)
        self.h_plans[slot].numpy()[...] = plan
        _cabi.check(self.lib.impala_ingest(_ptr(self.d_plans[slot]), C.c_void_p(self.h_plans[slot].data_ptr()),
                                           plan.nbytes, C.c_void_p(cs.cuda_stream)), "impala_ingest(plan)")
        self.replay_plan, self._ingested, self._slab_update[slot] = plan, n, n
        return C.c_void_p(self.store.data_ptr() + (n % self.sampler.slots) * self.slab_bytes)

    def register_host(self, address: int, nbytes: int) -> None:
        """Page-lock caller-owned host memory (e.g. a shared-memory trajectory ring) for DMA."""
        rc = torch.cuda.cudart().cudaHostRegister(address, nbytes, 0)
        if int(rc) != 0:
            raise _cabi.ImpalaCudaError(f"cudaHostRegister failed: {rc}")

    def ingest_from(self, host_address: int, slot: int = 0) -> None:
        """Like `ingest`, but the source slab is caller-owned (registered) host memory in the
        same batch layout - the DMA reads the actors' shared-memory slab directly."""
        cs = self.copy_stream
        if self._slab_used[slot]:
            cs.wait_event(self.slab_free[slot])
        _cabi.check(self.lib.impala_ingest(self._ingest_target(slot), C.c_void_p(host_address),
                                           self.slab_bytes, C.c_void_p(cs.cuda_stream)), "impala_ingest")
        self.slab_ready[slot].record(cs)

    def ingest_shard_from(self, host_address: int, b0: int, B_total: int, slot: int = 0) -> None:
        """Data-parallel ingest: columns [b0, b0 + B_local) of a caller-owned (registered) host slab
        laid out for B_total columns -> device slab `slot` (impala_ingest_shard)."""
        if self.replay_slabs:
            raise ValueError("experience replay runs on one device: there is no sharded ingest into the store")
        cs = self.copy_stream
        if self._slab_used[slot]:
            cs.wait_event(self.slab_free[slot])
        if self.gaussian or self.heads or self.masked:
            _cabi.check(self.lib.impala_ingest_shard_act(_ptr(self.d_slabs[slot]), C.c_void_p(host_address), self.T,
                                                         B_total, self.F, self.frames, self.A, self.obs_code,
                                                         self.act_kind, b0, self.B, C.c_void_p(cs.cuda_stream)),
                        "impala_ingest_shard_act")
        else:
            _cabi.check(self.lib.impala_ingest_shard_frames(_ptr(self.d_slabs[slot]), C.c_void_p(host_address),
                                                            self.T, B_total, self.F, self.frames, self.A,
                                                            self.obs_code, b0, self.B, C.c_void_p(cs.cuda_stream)),
                        "impala_ingest_shard_frames")
        self.slab_ready[slot].record(cs)

    def load_device_batch(self, batch: dict, slot: int = 0) -> None:
        """Convenience for kernel-only timing: put a batch in HBM and wait for it."""
        self.fill_host(batch, slot)
        self.ingest(slot)
        self.copy_stream.synchronize()

    # ------------------------------------------------------------------------ step
    def _enqueue_main(self, slot: int = 0) -> int:
        lib, hp, st = self.lib, self.hp, C.c_void_p(torch.cuda.current_stream().cuda_stream)
        launched = lib.impala_launch_count()
        d = self.d_views[slot]
        T, B, O, A = self.T, self.B, self.O, self.N_pi  # A: the policy's outputs from here on
        if self.replay_slabs and (self.gaussian or self.heads or self.masked):
            _cabi.check(lib.impala_batch_compose_act(_ptr(self.d_slabs[slot]), _ptr(self.store), self.slab_bytes,
                                                     _ptr(self.d_plans[slot]), T, B, self.B_fresh, self.F, self.frames,
                                                     self.A, self.obs_code, self.act_kind, st),
                        "impala_batch_compose_act")
        elif self.replay_slabs:  # the training slab out of the store, by the plan ingest left in d_plans[slot]
            _cabi.check(lib.impala_batch_compose(_ptr(self.d_slabs[slot]), _ptr(self.store), self.slab_bytes,
                                                 _ptr(self.d_plans[slot]), T, B, self.B_fresh, self.F, self.frames, A,
                                                 self.obs_code, st), "impala_batch_compose")
        p_pi = C.c_void_p(self.params.data_ptr())
        p_vf = C.c_void_p(self.params.data_ptr() + 4 * self.n_pi)
        # this rank's [gradient | scalars] goes to `comm` (final at N = 1, reduced in place by NCCL,
        # source of impala_peer_push); the fused push variant of the backward sends the gradient
        # straight to the peers and only the scalars pass through `comm`
        gbase = self.comm.data_ptr()
        g_pi = C.c_void_p(gbase)
        g_vf = C.c_void_p(gbase + 8 * self.n_pi)
        scal = C.c_void_p(gbase + 8 * self.n_total)
        obs = _ptr(d["obs"])
        if self.obs_norm:  # normalized float32 rows (any slab form) and the batch's sums into `comm`
            _cabi.check(lib.impala_obs_normalize(obs, self.obs_code, T, B, self.F, self.frames, _ptr(d["lens"]),
                                                 _ptr(self.obs_norm_dev), _ptr(self.obs_normed),
                                                 C.c_void_p(gbase + 8 * self.obs_sums_at), _ptr(self.obs_norm_ws),
                                                 self.obs_norm_ws.numel(), st), "impala_obs_normalize")
            obs = _ptr(self.obs_normed)
        elif self.obs_dense is not None:  # frames: one unstacking launch (widening bytes for O <= 128)
            out_code = _cabi.OBS_U8 if self.obs_dense.dtype == torch.uint8 else _cabi.OBS_F32
            _cabi.check(lib.impala_obs_unstack(obs, self.obs_code, _ptr(self.obs_dense), out_code, T + 1, B, self.F,
                                               self.frames, st), "impala_obs_unstack")
            obs = _ptr(self.obs_dense)
        elif self.obs_f32 is not None:  # byte observations, O <= 128: one widening launch, then the float path
            _cabi.check(lib.impala_obs_u8_to_f32(obs, _ptr(self.obs_f32), self.obs_f32.numel(), st),
                        "impala_obs_u8_to_f32")
            obs = _ptr(self.obs_f32)
        x_code = _cabi.OBS_U8 if self.obs_u8_native else _cabi.OBS_F32
        if self.shared_torso:  # one network, its two heads written into logits and values
            _cabi.check(lib.impala_mlp_forward_shared(obs, x_code, p_pi, _ptr(self.logits), _ptr(self.values),
                                                      self.M_pi, self.M_vf, O, self.H_pi, A, st),
                        "impala_mlp_forward_shared")
        elif self.obs_u8_native:
            # the pair entry point runs the two networks one after the other at these widths: same launches
            for p, out, M, H, N2 in ((p_pi, self.logits, self.M_pi, self.H_pi, A),
                                     (p_vf, self.values, self.M_vf, self.H_v, 1)):
                _cabi.check(lib.impala_mlp_forward_u8(obs, p, _ptr(out), M, O, H, N2, st), "impala_mlp_forward_u8")
        else:
            _cabi.check(lib.impala_mlp_forward_pair(obs, p_pi, p_vf, _ptr(self.logits), _ptr(self.values),
                                                    self.M_pi, self.M_vf, O, self.H_pi, self.H_v, A, st),
                        "impala_mlp_forward_pair")
        vt_in = (_ptr(self.logits), _ptr(d["beh_logits"]), _ptr(d["actions"]),
                 _ptr(d["rewards"]), _ptr(d["done"]), _ptr(d["lens"]), _ptr(self.values),
                 _ptr(self.vs), _ptr(self.pg_adv), _ptr(self.dlogits), _ptr(self.dv), scal)
        vt_hp = (T, B, A, float(hp.gamma), float(hp.rho_bar), float(hp.c_bar), float(hp.v_loss_c),
                 float(hp.policy_loss_c), float(hp.entropy_c), float(self.inv_batch), self.mode, st)
        if self.gaussian:  # the same flags through the Gaussian policy terms; A = action dimensions
            sums = C.c_void_p(gbase + 8 * (self.n_total + 4)) if self.n_extra == 12 else None
            _cabi.check(lib.impala_vtrace_loss_gauss(*vt_in, _ptr(self.ws_vt), self.ws_vt_bytes, T, B, self.A,
                                                     *vt_hp[3:-1], sums, _ptr(self.popart_buf) if self.popart else None,
                                                     self.reward_clip_code, st), "impala_vtrace_loss_gauss")
        elif self.masked:  # the same flags with the legal words (categorical, or the heads of a multi-discrete policy)
            sums = C.c_void_p(gbase + 8 * (self.n_total + 4)) if self.n_extra == 12 else None
            _cabi.check(lib.impala_vtrace_loss_mask(*vt_in, _ptr(self.ws_vt), self.ws_vt_bytes, *vt_hp[:-1], sums,
                                                    _ptr(self.popart_buf) if self.popart else None,
                                                    self.reward_clip_code, self.md_heads, len(self.heads), st),
                        "impala_vtrace_loss_mask")
        elif self.heads:  # the same flags through the multi-discrete policy terms; A = sum of the heads
            sums = C.c_void_p(gbase + 8 * (self.n_total + 4)) if self.n_extra == 12 else None
            _cabi.check(lib.impala_vtrace_loss_md(*vt_in, _ptr(self.ws_vt), self.ws_vt_bytes, *vt_hp[:-1], sums,
                                                  _ptr(self.popart_buf) if self.popart else None,
                                                  self.reward_clip_code, self.md_heads, len(self.heads), st),
                        "impala_vtrace_loss_md")
        elif self.reward_clip_code:  # the same kernel as below with the reward transform
            sums = C.c_void_p(gbase + 8 * (self.n_total + 4)) if self.n_extra == 12 else None
            _cabi.check(lib.impala_vtrace_loss_rclip(*vt_in, _ptr(self.ws_vt), self.ws_vt_bytes, *vt_hp[:-1], sums,
                                                     _ptr(self.popart_buf) if self.popart else None,
                                                     self.reward_clip_code, st), "impala_vtrace_loss_rclip")
        elif self.popart:  # normalized values under the device statistics; the eight sums after the four scalars
            _cabi.check(lib.impala_vtrace_loss_popart(*vt_in, C.c_void_p(gbase + 8 * (self.n_total + 4)),
                                                      _ptr(self.ws_vt), self.ws_vt_bytes, *vt_hp[:-1],
                                                      _ptr(self.popart_buf), st), "impala_vtrace_loss_popart")
        elif self.diagnostics:  # the eight sums land right after the four scalars
            _cabi.check(lib.impala_vtrace_loss_diag(*vt_in, C.c_void_p(gbase + 8 * (self.n_total + 4)),
                                                    _ptr(self.ws_vt), self.ws_vt_bytes, *vt_hp),
                        "impala_vtrace_loss_diag")
        else:
            _cabi.check(lib.impala_vtrace_loss(*vt_in, _ptr(self.ws_vt), self.ws_vt_bytes, *vt_hp),
                        "impala_vtrace_loss")
        pr = self.peer
        if pr and pr["fused"]:  # obs_norm: the observation sums follow the logged extras in `comm` and are pushed too
            push = lib.impala_mlp_backward_pair_push_obs_norm if self.obs_norm else lib.impala_mlp_backward_pair_push
            _cabi.check(push(
                obs, p_pi, p_vf, _ptr(self.dlogits), _ptr(self.dv), _ptr(self.ws_pi), self.ws_pi_bytes,
                _ptr(self.ws_vf), self.ws_vf_bytes, self.M_pi, self.M_vf, O, self.H_pi, self.H_v, A, scal, self.n_extra,
                _ptr(pr["gather_ptrs"]), _ptr(pr["seq"]), pr["slot"], pr["buf"], pr["rank"], self.world, st),
                "impala_mlp_backward_pair_push")
        else:
            if self.shared_torso:  # dz from dlogits (rows < T B) and dv: the gradient of the whole block
                _cabi.check(lib.impala_mlp_backward_shared(obs, x_code, p_pi, _ptr(self.dlogits), _ptr(self.dv), g_pi,
                                                           _ptr(self.ws_pi), self.ws_pi_bytes, self.M_pi, self.M_vf, O,
                                                           self.H_pi, A, st), "impala_mlp_backward_shared")
            elif self.obs_u8_native:
                for p, dout, g, ws, nbytes, M, H, N2 in (
                        (p_pi, self.dlogits, g_pi, self.ws_pi, self.ws_pi_bytes, self.M_pi, self.H_pi, A),
                        (p_vf, self.dv, g_vf, self.ws_vf, self.ws_vf_bytes, self.M_vf, self.H_v, 1)):
                    _cabi.check(lib.impala_mlp_backward_u8(obs, p, _ptr(dout), g, _ptr(ws), nbytes, M, O, H, N2, st),
                                "impala_mlp_backward_u8")
            else:
                _cabi.check(lib.impala_mlp_backward_pair(
                    obs, p_pi, p_vf, _ptr(self.dlogits), _ptr(self.dv), g_pi, g_vf, _ptr(self.ws_pi),
                    self.ws_pi_bytes, _ptr(self.ws_vf), self.ws_vf_bytes, self.M_pi, self.M_vf, O, self.H_pi,
                    self.H_v, A, st), "impala_mlp_backward_pair")
            if pr:  # stand-alone producer: all of comm -> every rank's gather buffer
                _cabi.check(lib.impala_peer_push(_ptr(self.comm), self.n_comm, _ptr(pr["gather_ptrs"]),
                                                 _ptr(pr["seq"]), pr["slot"], pr["buf"], pr["rank"], self.world, st),
                            "impala_peer_push")
        return int(lib.impala_launch_count() - launched)  # kernels actually launched / captured

    def lr_of(self, n: int) -> float:
        """The learning rate update n (1-based) uses (host-side, no device read)."""
        return self.optim.lr_of(n)

    def _enqueue_opt(self) -> int:
        n = self._enqueue_rule()
        if self.obs_norm:
            n += self._enqueue_obs_norm_update()
        return n

    def _enqueue_obs_norm_update(self) -> int:
        """The statistics merge and the folded block, one launch behind the optimizer."""
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        nets = [x for net in self.w1_nets for x in net] + [0, 0, 0] * (2 - len(self.w1_nets))
        pr = self.peer
        peer = ((C.c_void_p(pr["gather"]), _ptr(pr["seq"]), pr["slot"], pr["buf"], self.world, self.obs_sums_at,
                 _ptr(pr["err"]), pr["timeout_s"]) if pr else (None, None, 0, 0, 1, 0, None, 0.0))
        _cabi.check(self.lib.impala_obs_norm_update(
            _ptr(self.obs_stats), _ptr(self.obs_norm_dev), C.c_void_p(self.comm.data_ptr() + 8 * self.obs_sums_at),
            self.obs_norm_eps, _ptr(self.params), _ptr(self.folded), self.n_total, self.O, *nets,
            _ptr(self.obs_norm_ctl), *peer, st), "impala_obs_norm_update")
        return 1

    def _enqueue_rule(self) -> int:
        hp, st = self.hp, C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if self.lr_table is not None:
            return self._enqueue_optim(st)
        if self.peer:
            pr = self.peer
            _cabi.check(self.lib.impala_gather_clip_adam(
                _ptr(self.params), _ptr(self.comm), C.c_void_p(pr["gather"]), _ptr(pr["seq"]),
                pr["slot"], pr["buf"], self.world, self.n_extra, _ptr(self.adam_m), _ptr(self.adam_v), _ptr(self.adam_step),
                self.n_clip, self.n_total, float(hp.max_norm), float(0.95 * hp.lr), 0.9, 0.999, 1e-8,
                _ptr(self.norms), _ptr(pr["err"]), pr["timeout_s"], st), "impala_gather_clip_adam")
            return 1
        _cabi.check(self.lib.impala_clip_adam(
            _ptr(self.params), _ptr(self.comm), _ptr(self.adam_m), _ptr(self.adam_v),
            _ptr(self.adam_step), self.n_clip, self.n_total, float(hp.max_norm),
            float(0.95 * hp.lr),  # LambdaLR(lambda e: 0.95): constant factor, learner.py:42
            0.9, 0.999, 1e-8, _ptr(self.norms), st), "impala_clip_adam")
        return 1

    def _enqueue_optim(self, st) -> int:
        """The chosen rule with the scheduled rate, on the same buffers and paths as _enqueue_opt."""
        o, hp = self.optim, self.hp
        rule = (_ptr(self.lr_table), self.lr_table.numel(), o.rule_code, o.h0, o.h1, o.eps)
        if self.popart:
            return self._enqueue_popart(st, rule)
        if self.peer:
            pr = self.peer
            _cabi.check(self.lib.impala_gather_clip_optim(
                _ptr(self.params), _ptr(self.comm), C.c_void_p(pr["gather"]), _ptr(pr["seq"]),
                pr["slot"], pr["buf"], self.world, self.n_extra, _ptr(self.adam_m), _ptr(self.adam_v), _ptr(self.adam_step),
                self.n_clip, self.n_total, float(hp.max_norm), *rule, _ptr(self.norms), _ptr(pr["err"]), pr["timeout_s"],
                st), "impala_gather_clip_optim")
            return 1
        _cabi.check(self.lib.impala_clip_optim(
            _ptr(self.params), _ptr(self.comm), _ptr(self.adam_m), _ptr(self.adam_v), _ptr(self.adam_step), self.n_clip,
            self.n_total, float(hp.max_norm), *rule, _ptr(self.norms), st), "impala_clip_optim")
        return 1

    def _enqueue_popart(self, st, rule) -> int:
        """_enqueue_optim with the PopArt statistics update and value-head rescale in the same launch."""
        hp = self.hp
        pop = (_ptr(self.popart_buf), self.n_total + 4, self.w2_at, self.H_v, self.b2_at, float(self.popart_beta))
        if self.peer:
            pr = self.peer
            _cabi.check(self.lib.impala_gather_clip_optim_popart(
                _ptr(self.params), _ptr(self.comm), C.c_void_p(pr["gather"]), _ptr(pr["seq"]),
                pr["slot"], pr["buf"], self.world, self.n_extra, _ptr(self.adam_m), _ptr(self.adam_v), _ptr(self.adam_step),
                self.n_clip, self.n_total, float(hp.max_norm), *rule, _ptr(self.norms), _ptr(pr["err"]), pr["timeout_s"],
                *pop, st), "impala_gather_clip_optim_popart")
            return 1
        _cabi.check(self.lib.impala_clip_optim_popart(
            _ptr(self.params), _ptr(self.comm), _ptr(self.adam_m), _ptr(self.adam_v), _ptr(self.adam_step), self.n_clip,
            self.n_total, float(hp.max_norm), *rule, _ptr(self.norms), *pop, st), "impala_clip_optim_popart")
        return 1

    def _capture(self, slot: int):
        # thread_local: other host threads of the learner process (weight publisher, evaluation) keep
        # making CUDA calls while this thread captures
        with torch.cuda.stream(self.stream):
            g1 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g1, stream=self.stream, capture_error_mode="thread_local"):
                self._main_launches = self._enqueue_main(slot)
                if self._one_graph():  # no library collective in between: the optimizer joins the graph
                    self._enqueue_opt()
            self._graph_main[slot] = g1
            if not self._one_graph() and self._graph_opt is None:
                g2 = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g2, stream=self.stream, capture_error_mode="thread_local"):
                    self._enqueue_opt()
                self._graph_opt = g2

    def _one_graph(self) -> bool:
        """Single GPU, or the all-reduce is the push over peer memory (no library call in between)."""
        return self.world == 1 or self.peer is not None

    def loop_stream(self, on: bool = True) -> None:
        """Make `self.stream` the calling thread's current stream for the duration of an update loop, so
        that step / post_scalars do not pay a stream-context switch per call (about 5 us each - the
        learner loop is host-bound at small batches).  loop_stream(False) restores the default stream."""
        import threading

        torch.cuda.set_stream(self.stream if on else torch.cuda.default_stream(self.dev))
        self._loop_thread = threading.get_ident() if on else None

    def _on_stream(self):
        import threading

        if self._loop_thread is not None and self._loop_thread == threading.get_ident():
            return _NO_CTX
        return torch.cuda.stream(self.stream)

    def step(self, slot: int = 0) -> None:
        """One learner update on the batch in device slab `slot` (async on `self.stream`)."""
        with self._on_stream():
            self.stream.wait_event(self.slab_ready[slot])
            if self.use_graph and self.steps_done >= 1:
                if slot not in self._graph_main:
                    self._capture(slot)
                self._graph_main[slot].replay()
                n = self._main_launches
                fused_opt = self._one_graph()
            else:
                n = self._enqueue_main(slot)  # first step eager: fills the launch-config caches
                fused_opt = False
            self.slab_free[slot].record(self.stream)
            self._slab_used[slot] = True
            if self.replay_slabs:  # the store reads of this update are enqueued: ingest of update u + 2 waits here
                u = self._slab_update[slot]
                self._update_done[u % 3].record(self.stream)
                self._stepped = max(self._stepped, u)
            if self.world > 1 and not self.peer:
                import torch.distributed as dist

                dist.all_reduce(self.comm, op=dist.ReduceOp.SUM, group=self.pg)
            if fused_opt:
                n += 1 + self.obs_norm
            elif self.use_graph and self._graph_opt is not None:
                self._graph_opt.replay()
                n += 1 + self.obs_norm
            else:
                n += self._enqueue_opt()
        self.launches_per_step = n
        self.steps_done += 1

    def forward_backward_only(self) -> None:
        """Everything up to (not including) the collective and the optimizer - for tests."""
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(self.slab_ready[0])
            self._enqueue_main(0)

    def read_scalars(self) -> dict:
        """D2H of the step's logged numbers (learner.py:217-240); waits for the step."""
        return self.fetch_scalars(self.post_scalars())

    def post_scalars(self) -> int:
        """Enqueue the D2H of the current step's scalars; returns a ticket for fetch_scalars."""
        k = self._ticket % 4
        self._ticket += 1
        with self._on_stream():
            self.h_scalars[k, :4].copy_(self.comm[self.n_total:self.n_total + 4], non_blocking=True)
            self.h_scalars[k, 4:6].copy_(self.norms, non_blocking=True)
            if self.peer:
                self.h_scalars[k, 6:7].copy_(self.peer["err"].to(torch.float64), non_blocking=True)
            if self.n_extra == 12:
                self.h_scalars[k, 8:16].copy_(self.comm[self.n_total + 4:self.n_total + 12], non_blocking=True)
            if self.popart:  # the statistics after the update and the (mu, sigma) its loss used
                self.h_scalars[k, 16:21].copy_(self.popart_buf, non_blocking=True)
            self._scalar_events[k].record(self.stream)
        return k

    def fetch_scalars(self, ticket: int) -> dict:
        self._scalar_events[ticket].synchronize()
        s = self.h_scalars[ticket].tolist()
        if self.peer and s[6] != 0.0:
            raise _cabi.ImpalaCudaError(
                f"data-parallel learner: a peer rank did not deliver its gradient within {self.peer['timeout_s']:.0f} s "
                "(IMPALA_PEER_TIMEOUT_S); parameters were left untouched on this rank")
        hp = self.hp
        out = dict(zip(SCALAR_NAMES, s[:4]))
        out["total_loss"] = (hp.v_loss_c * out["value_fn_loss"] + hp.policy_loss_c * out["policy_loss"]
                             - hp.entropy_c * out["policy_entropy"])  # learner.py:154-159
        out["norm_policy"], out["norm_value"] = (s[5], 0.0) if self.shared_torso else (s[4], s[5])
        if self.popart:
            out["popart_mu"], out["popart_sigma"] = s[16], s[18]
        if self.diagnostics:
            # explained variance in reward units: the logged value loss is the normalized one of sigma_loss
            vl = out["value_fn_loss"] * (s[20] ** 2 if self.popart else 1.0)
            out.update(diagnostic_values(s[8:16], vl, self.global_batch))
        return out

    def synchronize(self) -> None:
        self.copy_stream.synchronize()
        self.stream.synchronize()
