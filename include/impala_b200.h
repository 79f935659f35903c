/*
 * impala_b200.h - C ABI of the GPU-native (H100, sm_90a) IMPALA learner hot path.
 *
 * Every entry point replaces a stretch of the reference learner's update
 * (threewisemonkeys-as/torched_impala, learner.py) that the reference executes as
 * per-trajectory ATen calls on the CPU.  The reference has no FFI of its own (it
 * is pure Python); these are the functions its `Learner._learn` would bind through
 * ctypes (see INTEGRATION.md for the stub).  Conventions:
 *
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless the
 *     parameter name starts with `host_`;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - nothing allocates, frees or synchronises; every call only enqueues work and
 *     is CUDA-graph capturable; the caller owns all buffers;
 *   - return value: 0 = ok, >0 = cudaError_t of the failed launch,
 *     <0 = IMPALA_ERR_* (argument / unsupported-shape errors).  No exceptions.
 *
 * Batch layout in HBM (time-major, dense, zero padded; `lens[b]` valid steps):
 *   obs (T+1,B,O) f32 (or u8, impala_batch_layout_obs) | beh_logits (T,B,A) f32 | actions (T,B) i32 |
 *   rewards (T,B) f32 | done (T,B) u8 | lens (B) i32
 * Parameter block of one MLP (Linear(O,H) -> ReLU -> Linear(H,N2)), f32, every
 * tensor starting on a 32-float boundary:  W1 (H,O) | b1 (H) | W2 (N2,H) | b2 (N2)
 * (row-major = torch nn.Linear.weight layout, reference models.py:13-18,41-46).
 */
#ifndef IMPALA_B200_H
#define IMPALA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IMPALA_OK 0
#define IMPALA_ERR_BAD_ARG (-1)
#define IMPALA_ERR_UNSUPPORTED_SHAPE (-2)
#define IMPALA_ERR_WORKSPACE_TOO_SMALL (-3)

#define IMPALA_MODE_REFERENCE 0 /* learner.py:126,130 as written (v[:1], double v[i+1] subtraction) */
#define IMPALA_MODE_PAPER 1     /* Espeholt et al. 2018 recurrence; not parity-checked */

#define IMPALA_PARAM_ALIGN 32 /* floats */

/* Version / build info: returns the sm arch the library was compiled for (90). */
int impala_abi_version(void);
int impala_compiled_sm(void);

/* Number of kernels this library has launched (or recorded into a capturing stream) since it was
 * loaded.  Callers difference it around a call sequence to know how many launches the sequence
 * is - e.g. the paired entry points are one launch where the tensor-core path covers both
 * networks and up to four otherwise. */
long long impala_launch_count(void);

/* Parameter-block layout of one MLP.  offsets[4] = float offsets of W1,b1,W2,b2;
 * *total = padded float count of the block (multiple of IMPALA_PARAM_ALIGN). */
int impala_param_layout(int O, int H, int N2, int64_t offsets[4], int64_t* total);

/* Byte offsets of the six batch tensors inside one contiguous slab (each 256-byte
 * aligned) and the slab size; the same layout is used for the pinned host slab and
 * the device slab so that ingest is ONE cudaMemcpyAsync.
 * order: obs, beh_logits, actions, rewards, done, lens.
 * Replaces the five torch.stack calls at learner.py:104-109,117. */
int impala_batch_layout(int T, int B, int O, int A, int64_t offsets[6], int64_t* total_bytes);

/* Observation element types of a batch slab.  IMPALA_OBS_U8: byte observations (Atari RAM, MinAtar
 * planes), values 0..255 entering the network as they are - a quarter of the slab bytes of float32. */
#define IMPALA_OBS_F32 0
#define IMPALA_OBS_U8 1

/* impala_batch_layout with the obs tensor of type obs_dtype ((T+1)*B*O bytes for IMPALA_OBS_U8);
 * every other tensor as above.  impala_batch_layout is its IMPALA_OBS_F32 case.  An unknown obs_dtype
 * returns IMPALA_ERR_BAD_ARG. */
int impala_batch_layout_obs(int T, int B, int O, int A, int obs_dtype, int64_t offsets[6], int64_t* total_bytes);

/* Frame-stacked observations stored once per frame.  With `frames` = k stacked frames of F values
 * each (the network sees O = k F features), the obs tensor of the slab is  frames (T+k, B, F)  of
 * type obs_dtype: observation row (t, b) is frames[t .. t+k-1, b, :] concatenated, oldest first (the
 * gym FrameStack order, flattened); frames s >= lens[b] + k are zero.  Every other tensor as in
 * impala_batch_layout_obs, whose layout is the frames = 1 case (F = O).  Bad arguments (frames < 1
 * included) return IMPALA_ERR_BAD_ARG. */
int impala_batch_layout_frames(int T, int B, int F, int frames, int A, int obs_dtype, int64_t offsets[6],
                               int64_t* total_bytes);

/* Action distributions of a batch slab and of the V-trace loss kernels.
 *   IMPALA_ACT_CATEGORICAL: A actions; beh_logits (T,B,A) f32, actions (T,B) i32 (indices).
 *   IMPALA_ACT_GAUSSIAN: diagonal Gaussian over A action dimensions; the behaviour record is the actor's
 *     policy output [m | s] (means, then log standard deviations), beh_logits (T,B,2A) f32, and the action the
 *     unsquashed sample m + e^s eps, actions (T,B,A) f32.
 *   IMPALA_ACT_MULTI_DISCRETE(K): K independent categorical heads (a gym MultiDiscrete space), 1 <= K <= 16, of
 *     n_k >= 2 actions each; A = N = sum_k n_k policy outputs, head k owning [s_k, s_k + n_k) with s_k = sum_{i<k} n_i.
 *     beh_logits (T,B,N) f32, actions (T,B,K) i32 (one index per head).  K = 1 is the categorical layout.
 *   IMPALA_ACT_MASKED, OR-ed onto IMPALA_ACT_CATEGORICAL or IMPALA_ACT_MULTI_DISCRETE(K): invalid-action masking.
 *     Each step carries one 32-bit legal word, as one more int32 column of the actions: (T,B,2) [a, legal] and
 *     (T,B,K+1) [a_0 .. a_{K-1}, legal].  Bit j set: policy output j is legal (A, N <= 32).
 *       - Bits >= A are ignored.  A head with no legal bit (categorical: the whole row) is all-legal, so padded
 *         steps and the empty columns of replay (every byte 0) need no special case.
 *       - pi and mu are the softmaxes of the current and behaviour logits renormalised over the legal entries
 *         (within each head); log pi(a), the ratio, V-trace, vs, pg_adv, the entropy -sum_{j legal} p_j log p_j
 *         and KL(mu || pi) come from them, and dz_j = 0 exactly at an illegal j.
 *       - The logit values at illegal entries, current or behaviour, reach no output (raw logits, -inf, -1e30 or
 *         NaN give identical results).
 *       - A taken action must be legal: that is the caller's responsibility, like an in-range index.
 *       - With every legal bit set, every output is bitwise that of the unmasked kernel with the same flags.
 *     IMPALA_ACT_GAUSSIAN | IMPALA_ACT_MASKED is refused (IMPALA_ERR_BAD_ARG). */
#define IMPALA_ACT_CATEGORICAL 0
#define IMPALA_ACT_GAUSSIAN 1
#define IMPALA_ACT_MULTI_DISCRETE(K) (0x100 | (K))
#define IMPALA_ACT_MASKED 0x200

/* impala_batch_layout_frames for the action distribution act_kind: IMPALA_ACT_CATEGORICAL is exactly
 * impala_batch_layout_frames, IMPALA_ACT_GAUSSIAN widens beh_logits to (T,B,2A) f32 and actions to (T,B,A) f32,
 * IMPALA_ACT_MULTI_DISCRETE(K) widens actions to (T,B,K) i32, IMPALA_ACT_MASKED adds one i32 column (the legal word)
 * to the actions of either.  An unknown act_kind, K outside 1..16, A < 2K, a masked Gaussian or a masked kind with
 * A > 32 returns IMPALA_ERR_BAD_ARG. */
int impala_batch_layout_act(int T, int B, int F, int frames, int A, int obs_dtype, int act_kind, int64_t offsets[6],
                            int64_t* total_bytes);

/* Host slab -> device slab, async on `stream` (host memory should be pinned). */
int impala_ingest(void* dev_slab, const void* host_slab, int64_t bytes, void* stream);

/* Data-parallel ingest: copy columns [b0, b0 + B_local) of a host slab laid out by
 * impala_batch_layout(T, B, O, A) into a device slab laid out by impala_batch_layout(T, B_local, O, A)
 * (strided 2-D DMAs; the host slab should be page-locked).  Every rank of a data-parallel learner
 * pulls its own shard of the actors' shared-memory slab over its own PCIe link. */
int impala_ingest_shard(void* dev_slab, const void* host_slab, int T, int B, int O, int A, int b0,
                        int B_local, void* stream);
/* The same for slabs laid out by impala_batch_layout_obs(..., obs_dtype) (obs rows of O bytes for
 * IMPALA_OBS_U8); impala_ingest_shard is its IMPALA_OBS_F32 case. */
int impala_ingest_shard_obs(void* dev_slab, const void* host_slab, int T, int B, int O, int A, int obs_dtype,
                            int b0, int B_local, void* stream);
/* The same for slabs laid out by impala_batch_layout_frames (T+frames frame rows of F values);
 * impala_ingest_shard_obs is its frames = 1 case. */
int impala_ingest_shard_frames(void* dev_slab, const void* host_slab, int T, int B, int F, int frames, int A,
                               int obs_dtype, int b0, int B_local, void* stream);
/* The same for slabs laid out by impala_batch_layout_act; impala_ingest_shard_frames is its
 * IMPALA_ACT_CATEGORICAL case. */
int impala_ingest_shard_act(void* dev_slab, const void* host_slab, int T, int B, int F, int frames, int A,
                            int obs_dtype, int act_kind, int b0, int B_local, void* stream);

/* Dense observation rows from frames (pure data movement, one launch):
 *   out[(t B + b) k F + j F + f] = frames[((t + j) B + b) F + f]   for t < R, b < B, j < k, f < F.
 * in_dtype -> out_dtype: IMPALA_OBS_U8 -> IMPALA_OBS_U8, IMPALA_OBS_U8 -> IMPALA_OBS_F32 (exact) or
 * IMPALA_OBS_F32 -> IMPALA_OBS_F32; any other pair, a NULL pointer or R, B, F, k < 1 returns
 * IMPALA_ERR_BAD_ARG.  16-byte loads and stores when F is a multiple of 16 bytes of frame data and both
 * pointers are 16-byte aligned, element copies otherwise. */
int impala_obs_unstack(const void* frames, int in_dtype, void* out, int out_dtype, int R, int B, int F, int k,
                       void* stream);

/* Experience replay: build the dense B-column training slab (impala_batch_layout_frames(T, B, ...)) out of a
 * store of Bf-column slabs (impala_batch_layout_frames(T, Bf, ...) each, store_slab_bytes apart, the fresh
 * batches of past updates).  For every one of the six tensors, column j of the training slab is column
 * plan[2j+1] of store slab plan[2j]; a negative slab index gives the empty trajectory (every byte zero,
 * lens = 0).  Pure data movement on bytes, one launch: any obs_dtype, dense and frame slabs.  plan is a device
 * array of B int32 pairs, 8-byte aligned.  16-byte loads and stores for the tensors whose bytes per (row,
 * column) are a multiple of 16 when both slabs and store_slab_bytes are 16-byte aligned, 4-byte words or single
 * bytes otherwise.  Bf <= 0, Bf >= B, store_slab_bytes smaller than the Bf-column slab, a NULL pointer or
 * arguments impala_batch_layout_frames refuses return IMPALA_ERR_BAD_ARG.  The plan's entries are not
 * checked: slab indices and columns < Bf are the caller's to keep in range. */
int impala_batch_compose(void* dst_slab, const void* store, int64_t store_slab_bytes, const int32_t* plan, int T,
                         int B, int Bf, int F, int frames, int A, int obs_dtype, void* stream);
/* The same for slabs laid out by impala_batch_layout_act; impala_batch_compose is its IMPALA_ACT_CATEGORICAL
 * case.  An unknown act_kind returns IMPALA_ERR_BAD_ARG. */
int impala_batch_compose_act(void* dst_slab, const void* store, int64_t store_slab_bytes, const int32_t* plan, int T,
                             int B, int Bf, int F, int frames, int A, int obs_dtype, int act_kind, void* stream);

/* out[i] = (float)x[i] for i < n: exact widening of byte observations, for the MLP shapes that read
 * float32 rows only (O <= 128). */
int impala_obs_u8_to_f32(const uint8_t* x, float* out, int64_t n, void* stream);

/* out[m, :] = relu(x[m, :] W1^T + b1) W2^T + b2 for m < M.
 * Replaces MlpPolicy.forward / MlpValueFn.forward in eval mode
 * (models.py:23-25, :51-52) as called at learner.py:112-113 on the flattened
 * (T*B, O) / ((T+1)*B, O) batch.  x row-major (M,O); out row-major (M,N2).
 * Shapes: O <= 128 with N2 <= 32 (tensor cores or FP32 kernels), and 128 < O <= 1024 with O % 4 == 0,
 * H = 128 k <= 1024, N2 <= 32 (tensor cores only: refused under IMPALA_MLP_TC=0 / IMPALA_MLP_TCW=0);
 * anything else returns IMPALA_ERR_UNSUPPORTED_SHAPE. */
int impala_mlp_forward(const float* x, const float* params, float* out, int M, int O, int H,
                       int N2, void* stream);

/* Both networks of one learner step in one launch: logits = policy(x[0..M_pi)), values =
 * value_fn(x[0..M_vf)) on the SAME observation rows (learner.py:112-113: `self.policy(obs[:-1])`
 * and `self.value_fn(obs)`; M_pi = T*B, M_vf = (T+1)*B).  Results are identical to two
 * impala_mlp_forward calls; where the tensor-core path covers both shapes the SMs are split
 * between the two tile lists so the step pays one prologue and one launch. */
int impala_mlp_forward_pair(const float* x, const float* params_pi, const float* params_vf,
                            float* logits, float* values, int M_pi, int M_vf, int O, int H_pi,
                            int H_vf, int A, void* stream);

/* Bytes of scratch impala_mlp_backward needs for these dimensions.  The caller zero-fills
 * it ONCE after allocation; every call leaves its control words zeroed again (the tensor-core
 * kernel meets at a self-re-arming grid barrier before its in-kernel reduction; on a workspace
 * that was never zeroed it traps - a launch failure, not a hang).  For O > 128 it holds DP^T (H x M
 * floats, the bulk of it) and two bounded sets of partial gradient rows.  Shape limits as
 * impala_mlp_forward; IMPALA_ERR_UNSUPPORTED_SHAPE (-2) outside them. */
int64_t impala_mlp_backward_workspace(int M, int O, int H, int N2);

/* Gradient of sum_m <dout[m,:], mlp(x[m,:])> w.r.t. the parameter block, written
 * (not accumulated) as float64 into grad[0 .. total) in parameter-block layout
 * (pad entries = 0).  Hidden activations are recomputed from x, nothing is saved
 * by the forward.  Replaces the MLP part of loss.backward() at learner.py:175. */
int impala_mlp_backward(const float* x, const float* params, const float* dout, double* grad,
                        void* workspace, int64_t workspace_bytes, int M, int O, int H, int N2,
                        void* stream);

/* impala_mlp_forward / impala_mlp_backward on byte observations (x row-major (M,O) uint8, 4-byte
 * aligned; values 0..255 enter the network unscaled).  Results are identical to the float entry points
 * on the same values converted to float32; the workspace is sized by impala_mlp_backward_workspace.
 * Shapes: 128 < O <= 1024 under the limits of impala_mlp_forward (K-streamed tensor-core kernels that
 * read the bytes directly).  O <= 128 returns IMPALA_ERR_UNSUPPORTED_SHAPE: callers widen those rows
 * once with impala_obs_u8_to_f32 and call the float entry points. */
int impala_mlp_forward_u8(const uint8_t* x, const float* params, float* out, int M, int O, int H, int N2,
                          void* stream);
int impala_mlp_backward_u8(const uint8_t* x, const float* params, const float* dout, double* grad,
                           void* workspace, int64_t workspace_bytes, int M, int O, int H, int N2, void* stream);

/* The MLP part of the single loss.backward() at learner.py:175 for both networks in one launch:
 * same results as impala_mlp_backward(policy; dout = dlogits) followed by
 * impala_mlp_backward(value_fn; dout = dv), each with its own workspace (sized by
 * impala_mlp_backward_workspace, zero-filled once). */
int impala_mlp_backward_pair(const float* x, const float* params_pi, const float* params_vf,
                             const float* dlogits, const float* dv, double* grad_pi, double* grad_vf,
                             void* workspace_pi, int64_t workspace_pi_bytes, void* workspace_vf,
                             int64_t workspace_vf_bytes, int M_pi, int M_vf, int O, int H_pi,
                             int H_vf, int A, void* stream);

/* Shared-torso actor-critic: ONE network with N2 = N + 1 outputs [policy | value] on M = (T+1)*B rows,
 * its outputs split into two buffers so the V-trace kernels read and write them where they do for two
 * networks.  Head a (the policy) is columns [0, N) of the first M_a = T*B rows, in logits (M_a, N); head b
 * (the value) is column N of all M rows, in values (M).  The forward does not write rows >= M_a of head a;
 * the backward reads dz from dlogits (M_a, N) and dv (M), rows >= M_a of head a as 0.  Results are bitwise
 * equal to impala_mlp_forward / impala_mlp_backward with N2 = N + 1 on the interleaved (M, N + 1) layout.
 * x_dtype: IMPALA_OBS_F32, or IMPALA_OBS_U8 for byte rows (O > 128 only, as impala_mlp_forward_u8).  The
 * workspace is sized by impala_mlp_backward_workspace(M, O, H, N + 1).  N < 1, N + 1 > 32, M_a > M, an
 * unknown x_dtype or a NULL pointer returns IMPALA_ERR_BAD_ARG; shapes as impala_mlp_forward. */
int impala_mlp_forward_shared(const void* x, int x_dtype, const float* params, float* logits, float* values,
                              int M_a, int M, int O, int H, int N, void* stream);
int impala_mlp_backward_shared(const void* x, int x_dtype, const float* params, const float* dlogits,
                               const float* dv, double* grad, void* workspace, int64_t workspace_bytes, int M_a,
                               int M, int O, int H, int N, void* stream);

/* V-trace only (learner.py:116-135): from current/behaviour logits, actions,
 * rewards, done, lens and the value estimates v (T+1,B) produce
 * vs (T+1,B) [the reference's `vt` after :131] and pg_adv (T,B).
 * Padded positions are written as 0. */
int impala_vtrace(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                  const float* rewards, const uint8_t* done, const int32_t* lens, const float* v,
                  float* vs, float* pg_adv, int T, int B, int A, float gamma, float rho_bar,
                  float c_bar, int mode, void* stream);

/* Bytes of scratch impala_vtrace_loss needs.  The caller zero-fills it ONCE after
 * allocation; every call leaves it zeroed where it must be (self-re-arming counter). */
int64_t impala_vtrace_loss_workspace(int T, int B, int A);

/* V-trace + the three losses + their closed-form backward in one kernel
 * (learner.py:116-162 and the non-MLP part of :175; helper functions :298-321).
 *   dlogits (T,B,A), dv (T+1,B): d total_loss / d logits, d total_loss / d v
 *   scalars[0..4) (float64, overwritten): value_fn_loss, policy_loss, policy_entropy (each
 *     sum_b(..)*inv_batch as logged at learner.py:160-162) and batch_mean_reward (:108);
 *     per-CTA sums are combined in a fixed order by the last CTA to finish, so the four
 *     numbers are bitwise reproducible.
 *   vs / pg_adv may be NULL when the caller does not need them.
 *   inv_batch = 1 / GLOBAL batch size (all ranks), so shard results add up. */
int impala_vtrace_loss(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                       const float* rewards, const uint8_t* done, const int32_t* lens,
                       const float* v, float* vs, float* pg_adv, float* dlogits, float* dv,
                       double* scalars, void* workspace, int64_t workspace_bytes, int T, int B,
                       int A, float gamma, float rho_bar, float c_bar, float v_loss_c,
                       float policy_loss_c, float entropy_c, float inv_batch, int mode,
                       void* stream);

/* Workspace of impala_vtrace_loss_diag (same zero-once rule; larger than impala_vtrace_loss's). */
int64_t impala_vtrace_loss_diag_workspace(int T, int B, int A);

/* impala_vtrace_loss (bit-identical vs, pg_adv, dlogits, dv and scalars) plus the off-policy
 * diagnostics of the batch: diag[0..8) (float64, overwritten) are sums over the valid steps
 * (t < lens[b]), NOT scaled by inv_batch, so they add across ranks:
 *   [0] n, the number of valid steps       [1] sum log pi(a_t) - log mu(a_t)  (natural log)
 *   [2] #{ratio_t > rho_bar}               [3] #{ratio_t > c_bar}
 *   [4] sum KL(mu_t || pi_t)               [5] sum vs_t
 *   [6] sum vs_t^2                         [7] sum (vs_t - v_t)
 * pi = softmax(cur_logits), mu = softmax(beh_logits), ratio_t = pi(a_t) / mu(a_t), vs_t the value
 * written to vs.  Combined in a fixed order like the scalars (bitwise reproducible). */
int impala_vtrace_loss_diag(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                            const float* rewards, const uint8_t* done, const int32_t* lens,
                            const float* v, float* vs, float* pg_adv, float* dlogits, float* dv,
                            double* scalars, double* diag, void* workspace, int64_t workspace_bytes,
                            int T, int B, int A, float gamma, float rho_bar, float c_bar,
                            float v_loss_c, float policy_loss_c, float entropy_c, float inv_batch,
                            int mode, void* stream);

/* impala_vtrace_loss_diag with PopArt value normalization (van Hasselt et al. 2016, single task).
 * popart: float64 device statistics {mu, nu, sigma, ...} (the layout impala_clip_optim_popart keeps),
 * read once; v holds the NORMALIZED value output n, the value in reward units is sigma n + mu.
 *   V-trace runs on sigma n + mu for every value read (v[:1] of IMPALA_MODE_REFERENCE included), so vs is
 *   in reward units; pg_adv = rho (r + gamma vs' - v) / sigma, the normalized advantage the policy gradient
 *   and policy loss use; the value loss is 0.5 sum ((v - vs) / sigma)^2, so dv = v_loss_c (v - vs) / (sigma B)
 *   (B = 1 / inv_batch); entropy and reward are unchanged; scalars[0..1] are the normalized losses.
 *   diag[0..8) are impala_vtrace_loss_diag's sums, in reward units.
 * Workspace: impala_vtrace_loss_diag_workspace.  At mu = 0, sigma = 1 every output is bit-identical to
 * impala_vtrace_loss_diag.  Returns IMPALA_ERR_BAD_ARG for a NULL popart and whatever that entry refuses. */
int impala_vtrace_loss_popart(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                              const float* rewards, const uint8_t* done, const int32_t* lens,
                              const float* v, float* vs, float* pg_adv, float* dlogits, float* dv,
                              double* scalars, double* diag, void* workspace, int64_t workspace_bytes,
                              int T, int B, int A, float gamma, float rho_bar, float c_bar,
                              float v_loss_c, float policy_loss_c, float entropy_c, float inv_batch,
                              int mode, const double* popart, void* stream);

#define IMPALA_REWARD_CLIP_ABS_ONE 1         /* r -> clip(r, -1, 1) (Atari) */
#define IMPALA_REWARD_CLIP_SOFT_ASYMMETRIC 2 /* r -> 5 tanh(r / 5) for r >= 0, 1.5 tanh(r / 5) for r < 0 (DMLab) */

/* impala_vtrace_loss (diag == NULL), impala_vtrace_loss_diag (diag, popart == NULL) or
 * impala_vtrace_loss_popart (diag and popart) with the reward transform `reward_clip` (IMPALA_REWARD_CLIP_*)
 * applied to every reward where it enters the recurrence (delta of either mode) and pg_adv.
 *   scalars[3] (batch_mean_reward) stays the mean of the RAW rewards; everything formed from vs - the losses,
 *   diag[0..8) and so the PopArt statistics the optimizer forms from them - is in clipped-reward units.
 *   NaN rewards stay NaN (compare-and-select, as torch.clamp); +-inf saturates.  With rewards already clipped
 *   on the host (abs_one) the outputs other than scalars[3] are bit-identical to the selected entry point's.
 * Workspace: that of the selected entry point.  Returns IMPALA_ERR_BAD_ARG for a popart without diag, a
 * reward_clip outside IMPALA_REWARD_CLIP_* and whatever the selected entry point refuses. */
int impala_vtrace_loss_rclip(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                             const float* rewards, const uint8_t* done, const int32_t* lens,
                             const float* v, float* vs, float* pg_adv, float* dlogits, float* dv,
                             double* scalars, void* workspace, int64_t workspace_bytes, int T, int B,
                             int A, float gamma, float rho_bar, float c_bar, float v_loss_c,
                             float policy_loss_c, float entropy_c, float inv_batch, int mode,
                             double* diag, const double* popart, int reward_clip, void* stream);

/* The V-trace loss kernel of impala_vtrace_loss_rclip for diagonal Gaussian policies (IMPALA_ACT_GAUSSIAN) over
 * A <= 16 action dimensions.  cur_params / beh_params (T,B,2A): the current and the behaviour policy outputs
 * [m | s], sigma = e^s; actions (T,B,A) f32: the unsquashed samples; dparams (T,B,2A): d total_loss / d params.
 *   log pi(a) = sum_k [-((a_k - m_k) / sigma_k)^2 / 2 - s_k - log(2 pi) / 2]  (torch Normal.log_prob summed), the
 *   same for mu with the behaviour outputs; ratio, clipping, V-trace, vs and pg_adv as for categorical policies.
 *   policy_loss = sum -log pi(a) pg_adv, policy_entropy = sum_k (s_k + (1 + log(2 pi)) / 2), each sum_b .. inv_batch.
 *   d/dm_k = -policy_loss_c pg_adv (a_k - m_k) / sigma_k^2 inv_batch,
 *   d/ds_k = (policy_loss_c pg_adv (1 - ((a_k - m_k) / sigma_k)^2) - entropy_c) inv_batch; zero at padded steps.
 *   diag[4] = sum KL(mu || pi) = sum_k [s_k - sb_k + (sigma_b,k^2 + (mb_k - m_k)^2) / (2 sigma_k^2) - 1/2].
 * diag == NULL: the loss sums only (workspace impala_vtrace_loss_workspace); diag: the eight off-policy sums as
 * impala_vtrace_loss_diag (workspace impala_vtrace_loss_diag_workspace); popart (needs diag): PopArt as
 * impala_vtrace_loss_popart; reward_clip: 0 (none) or IMPALA_REWARD_CLIP_*.  A > 16 returns
 * IMPALA_ERR_UNSUPPORTED_SHAPE; a popart without diag, an unknown reward_clip and what impala_vtrace_loss refuses
 * return IMPALA_ERR_BAD_ARG. */
int impala_vtrace_loss_gauss(const float* cur_params, const float* beh_params, const float* actions,
                             const float* rewards, const uint8_t* done, const int32_t* lens, const float* v,
                             float* vs, float* pg_adv, float* dparams, float* dv, double* scalars, void* workspace,
                             int64_t workspace_bytes, int T, int B, int A, float gamma, float rho_bar, float c_bar,
                             float v_loss_c, float policy_loss_c, float entropy_c, float inv_batch, int mode,
                             double* diag, const double* popart, int reward_clip, void* stream);

/* The V-trace loss kernel of impala_vtrace_loss_rclip for multi-discrete policies (IMPALA_ACT_MULTI_DISCRETE(K)):
 * K <= 16 independent softmax heads over A = N = sum_k n_k <= 32 policy outputs, host_heads[k] = n_k >= 2 (read at
 * call time and passed to the kernel by value, so a captured graph keeps them).  cur_logits / beh_logits / dlogits
 * (T,B,N); actions (T,B,K) i32, a_k in [0, n_k).  With p the softmax within a head (z[s_k : s_k + n_k]):
 *   log pi(a) = sum_k log p_k(a_k), the same for mu with the behaviour logits; ratio, clipping, V-trace, vs and
 *   pg_adv as for categorical policies.  policy_loss = sum -log pi(a) pg_adv, policy_entropy = sum_k H_k, each
 *   sum_b .. inv_batch.  For j in head k:
 *   dz_j = inv_batch [policy_loss_c pg_adv (p_j - [j = s_k + a_k]) + entropy_c p_j (log p_j + H_k)]; zero at padded
 *   steps.  diag[4] = sum KL(mu || pi) = sum_k KL_k.  K = 1 is impala_vtrace_loss_rclip's categorical policy.
 * diag, popart, reward_clip and the workspace as impala_vtrace_loss_gauss (impala_vtrace_loss[_diag]_workspace(T, B,
 * N)).  K > 16 or N > 32 returns IMPALA_ERR_UNSUPPORTED_SHAPE; a NULL host_heads, K < 1, an n_k < 2, sum_k n_k != A,
 * a popart without diag, an unknown reward_clip and what impala_vtrace_loss refuses return IMPALA_ERR_BAD_ARG. */
int impala_vtrace_loss_md(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                          const float* rewards, const uint8_t* done, const int32_t* lens, const float* v, float* vs,
                          float* pg_adv, float* dlogits, float* dv, double* scalars, void* workspace,
                          int64_t workspace_bytes, int T, int B, int A, float gamma, float rho_bar, float c_bar,
                          float v_loss_c, float policy_loss_c, float entropy_c, float inv_batch, int mode,
                          double* diag, const double* popart, int reward_clip, const int32_t* host_heads, int K,
                          void* stream);

/* Invalid-action masking (IMPALA_ACT_MASKED, see above) in the V-trace loss kernel of impala_vtrace_loss_rclip.  The
 * arguments are those of impala_vtrace_loss_md, with actions in the widened layout: host_heads == NULL selects one
 * categorical softmax over the A <= 32 outputs, actions (T,B,2) [a, legal]; otherwise the K heads of
 * impala_vtrace_loss_md, actions (T,B,K+1) [a_0 .. a_{K-1}, legal].  actions must be 8-byte aligned (host_heads ==
 * NULL).  diag, popart, reward_clip and the workspace (impala_vtrace_loss[_diag]_workspace(T, B, A)) as
 * impala_vtrace_loss_md; A > 32 returns IMPALA_ERR_UNSUPPORTED_SHAPE, the rest what impala_vtrace_loss_md refuses. */
int impala_vtrace_loss_mask(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                            const float* rewards, const uint8_t* done, const int32_t* lens, const float* v, float* vs,
                            float* pg_adv, float* dlogits, float* dv, double* scalars, void* workspace,
                            int64_t workspace_bytes, int T, int B, int A, float gamma, float rho_bar, float c_bar,
                            float v_loss_c, float policy_loss_c, float entropy_c, float inv_batch, int mode,
                            double* diag, const double* popart, int reward_clip, const int32_t* host_heads, int K,
                            void* stream);

/* Per-group gradient clipping + Adam in one launch (learner.py:176-183).
 *   params/m/v: f32 [n_total]; grad: f64 [n_total] (the possibly all-reduced sum);
 *   group 0 = [0, n_policy) (policy net), group 1 = [n_policy, n_total) (value net);
 *   each group is scaled by min(1, max_norm / (||g||_2 + 1e-6)) as
 *   torch.nn.utils.clip_grad_norm_ does - a NaN norm (a NaN entry in the group) scales by NaN,
 *   so every parameter, m and v of that group becomes NaN, as in torch; an infinite entry gives
 *   coefficient 0 - then one Adam step (no weight decay) with
 *   bias correction from the device-side optimizer state (updated by the kernel):
 *   state = int64[3] {step count, beta1^step, beta2^step as float64 bits}; all zero = fresh.
 *   norms_out (f64[2], may be NULL) receives the two pre-clip norms. */
int impala_clip_adam(float* params, const double* grad, float* m, float* v, int64_t* state,
                     int64_t n_policy, int64_t n_total, float max_norm, float lr, float beta1,
                     float beta2, float eps, double* norms_out, void* stream);

/* Update rules of impala_clip_optim / impala_gather_clip_optim. */
#define IMPALA_OPT_ADAM 0    /* torch.optim.Adam, no weight decay:  h0 = beta1, h1 = beta2 */
#define IMPALA_OPT_RMSPROP 1 /* torch.optim.RMSprop, not centered, no weight decay:  h0 = alpha, h1 = momentum */

/* impala_clip_adam with a choice of update rule and a learning-rate SCHEDULE read from device memory:
 * the update after n completed ones (n = state[0]) uses lr_table[min(n, n_lr - 1)] - torch's
 * LambdaLR(lambda) with lr_table[e] = lr * lambda(e).  The table is only read, so one captured CUDA graph
 * serves every update of a schedule.  Clipping, norms_out and the float32 state are as in impala_clip_adam.
 *   IMPALA_OPT_ADAM     m = exp_avg, v = exp_avg_sq, state = {step, beta1^step, beta2^step bits}: a table of
 *                       one constant lr gives the bits of impala_clip_adam with that lr.
 *   IMPALA_OPT_RMSPROP  per entry, on the clipped gradient g:  v = alpha v + (1 - alpha) g^2,
 *                       avg = sqrt(v) + eps (eps OUTSIDE the root, as torch);  momentum > 0:  m = momentum m +
 *                       g / avg, param -= lr m;  momentum = 0:  param -= lr g / avg and m is neither read nor
 *                       written.  v = square_avg, m = momentum_buffer (both start at 0); state[0] counts the
 *                       steps, state[1] and state[2] are left as they are.
 * Returns IMPALA_ERR_BAD_ARG before any launch for the arguments impala_clip_adam refuses, a NULL lr_table,
 * n_lr < 1, an unknown rule, eps < 0, and for RMSprop alpha outside [0, 1) or momentum < 0 (NaN included). */
int impala_clip_optim(float* params, const double* grad, float* m, float* v, int64_t* state,
                      int64_t n_policy, int64_t n_total, float max_norm, const float* lr_table, int64_t n_lr,
                      int rule, float h0, float h1, float eps, double* norms_out, void* stream);

/* Node-local buffers that the other ranks (one process per GPU) map into their address space
 * for the push-model all-reduce below: impala_peer_alloc = cudaMalloc + zero-fill on the current
 * device and its 64-byte CUDA IPC handle (to be sent to the peers, e.g. through
 * torch.distributed); impala_peer_open maps a peer's handle on the current device with peer
 * access enabled. */
int impala_peer_alloc(int64_t bytes, void** dev_ptr, void* handle64);
int impala_peer_open(const void* handle64, void** dev_ptr);
int impala_peer_close(void* dev_ptr);
int impala_peer_free(void* dev_ptr);

/* Data-parallel learners on one NVLink node (one process per GPU): the gradient all-reduce
 * without a collective library call, as a PUSH over peer-mapped memory in LL format.  Replaces the
 * DistributedDataParallel-style all-reduce a multi-GPU port of learner.py:175-183 would place
 * between loss.backward() and optimizer.step().
 *
 * Every rank owns a gather buffer  G[2 parities][world slots][slot_stride]  of 16-byte LL elements
 * (parities buf_stride elements apart, zero-filled once) mapped by all ranks; peer_gather[r] is
 * THIS process's device pointer to rank r's buffer (own entry included), the array itself in
 * device memory.  An LL element carries one float64 as [lo32 | step32 | hi32 | step32]: each
 * 8-byte half is tagged with the step it belongs to, so data and "ready" travel in the same
 * posted NVLink write - no fence, no flag, no acknowledgement.  `seq` is a device int64
 * (zero-filled once) counting completed optimizer calls; step s = *seq + 1 uses parity s & 1.
 *   producer  stores this rank's [gradient (n_total) | n_extra logged scalars] of step s into slot
 *             `rank` of EVERY rank's buffer: impala_mlp_backward_pair_push does it in the tail of
 *             the paired tensor-core backward kernel (no extra launch); impala_peer_push is the
 *             stand-alone producer for shapes that kernel does not cover (after
 *             impala_mlp_backward[_pair]).
 *   consumer  impala_gather_clip_adam polls the `world` LOCAL slots of each entry until they carry
 *             step s, adds them in rank order (bit-identical sums on every rank), writes them to
 *             `reduced` ([n_total + n_extra], local), applies impala_clip_adam's update and
 *             advances *seq.
 * The parity buffers replace a "slot consumed" message (a slot is rewritten two steps later, after
 * the values of the step in between proved that every peer has finished reading it).  Every rank
 * must make the same sequence of calls.  A rank that never delivers does not kill the others:
 * after timeout_s (<= 0: 600 s) the consumer sets *err = 1 (device int, may be NULL), leaves
 * parameters / optimizer state / seq untouched and returns normally. */
int impala_peer_push(const double* local, int64_t n, void* const* peer_gather, const long long* seq,
                     int64_t slot_stride, int64_t buf_stride, int rank, int world, void* stream);
/* 1 when impala_mlp_backward_pair_push covers these shapes (tensor-core paired backward). */
int impala_mlp_backward_pair_push_supported(int M_pi, int M_vf, int O, int H_pi, int H_vf, int A);
/* impala_mlp_backward_pair whose reduction tail pushes [grad_pi | grad_vf | extra[0..n_extra)] to
 * the peers; `extra` = this rank's local scalars (device, read by the kernel). */
int impala_mlp_backward_pair_push(const float* x, const float* params_pi, const float* params_vf,
                                  const float* dlogits, const float* dv, void* workspace_pi,
                                  int64_t workspace_pi_bytes, void* workspace_vf,
                                  int64_t workspace_vf_bytes, int M_pi, int M_vf, int O, int H_pi,
                                  int H_vf, int A, const double* extra, int n_extra,
                                  void* const* peer_gather, const long long* seq, int64_t slot_stride,
                                  int64_t buf_stride, int rank, int world, void* stream);
/* impala_mlp_backward_pair_push for an observation-normalizing engine: `extra` holds the n_extra (<= 32) logged
 * extras followed by impala_obs_normalize's 2 O + 1 sums, and all n_extra + 2 O + 1 of them are pushed (the slot
 * must hold them).  O > IMPALA_OBS_NORM_MAX_FEATURES returns IMPALA_ERR_BAD_ARG. */
int impala_mlp_backward_pair_push_obs_norm(const float* x, const float* params_pi, const float* params_vf,
                                           const float* dlogits, const float* dv, void* workspace_pi,
                                           int64_t workspace_pi_bytes, void* workspace_vf, int64_t workspace_vf_bytes,
                                           int M_pi, int M_vf, int O, int H_pi, int H_vf, int A, const double* extra,
                                           int n_extra, void* const* peer_gather, const long long* seq,
                                           int64_t slot_stride, int64_t buf_stride, int rank, int world, void* stream);
int impala_gather_clip_adam(float* params, double* reduced, const void* gather, long long* seq,
                            int64_t slot_stride, int64_t buf_stride, int world, int n_extra, float* m,
                            float* v, int64_t* state, int64_t n_policy, int64_t n_total,
                            float max_norm, float lr, float beta1, float beta2, float eps,
                            double* norms_out, int* err, double timeout_s, void* stream);
/* impala_gather_clip_adam whose update is impala_clip_optim's (rule, h0, h1, eps, learning-rate table);
 * refuses what either of the two refuses.  The table entry is read before the wait on the backward. */
int impala_gather_clip_optim(float* params, double* reduced, const void* gather, long long* seq,
                             int64_t slot_stride, int64_t buf_stride, int world, int n_extra, float* m,
                             float* v, int64_t* state, int64_t n_policy, int64_t n_total, float max_norm,
                             const float* lr_table, int64_t n_lr, int rule, float h0, float h1, float eps,
                             double* norms_out, int* err, double timeout_s, void* stream);

/* Size of the PopArt statistics, float64 {mu, nu, sigma, mu_loss, sigma_loss}: the running mean and second
 * moment of the value targets and sigma = clamp(sqrt(max(nu - mu^2, 0)), 1e-4, 1e6), then the (mu, sigma)
 * the loss of the last update used.  A fresh run starts at {0, 1, 1, 0, 1}. */
#define IMPALA_POPART_STATS 5

/* impala_clip_optim (resp. impala_gather_clip_optim) followed, in the same launch, by the PopArt step:
 *   n = grad[sums_at], S1 = grad[sums_at + 5], S2 = grad[sums_at + 6] (impala_vtrace_loss_popart's diag
 *   sums; the gather variant reads them from `reduced`, added in rank order, so sums_at + 8 <= n_total +
 *   n_extra), then with b = beta:
 *     mu' = (1 - b) mu + b S1 / n,  nu' = (1 - b) nu + b S2 / n,  sigma' = clamp(sqrt(max(nu' - mu'^2, 0)), 1e-4, 1e6)
 *   (n = 0 leaves mu, nu, sigma as they are), and, after the optimizer step, the value head is rescaled so that
 *   sigma' n + mu' is the output sigma n + mu of the updated head:
 *     params[w2_off, w2_off + w2_len) *= sigma / sigma',  params[b2_off] = (sigma b2 + mu - mu') / sigma'.
 *   The optimizer state (m, v) is not touched.  popart[3], popart[4] receive the (mu, sigma) the update's
 *   loss used.  A timed-out gather leaves the statistics untouched, like the parameters.
 * Returns IMPALA_ERR_BAD_ARG before any launch for what impala_clip_optim / impala_gather_clip_optim refuse,
 * a NULL popart, beta outside (0, 1] (NaN included), sums_at < n_total, w2_len < 1, a W2 block or b2 outside
 * [n_policy, n_total), or b2 inside the W2 block. */
int impala_clip_optim_popart(float* params, const double* grad, float* m, float* v, int64_t* state,
                             int64_t n_policy, int64_t n_total, float max_norm, const float* lr_table, int64_t n_lr,
                             int rule, float h0, float h1, float eps, double* norms_out, double* popart,
                             int64_t sums_at, int64_t w2_off, int64_t w2_len, int64_t b2_off, float beta,
                             void* stream);
int impala_gather_clip_optim_popart(float* params, double* reduced, const void* gather, long long* seq,
                                    int64_t slot_stride, int64_t buf_stride, int world, int n_extra, float* m,
                                    float* v, int64_t* state, int64_t n_policy, int64_t n_total, float max_norm,
                                    const float* lr_table, int64_t n_lr, int rule, float h0, float h1, float eps,
                                    double* norms_out, int* err, double timeout_s, double* popart, int64_t sums_at,
                                    int64_t w2_off, int64_t w2_len, int64_t b2_off, float beta, void* stream);

/* ---- Observation normalization (obs_norm): running per-feature statistics of the raw observations.
 * Statistics, float64 [count | mean (O) | var (O)]: a fresh run is {0, 0.., 1..}.  The kernels read them as
 * norm, float32 [mu_f (O) | r_f (O)] with mu_f = (float)mean, r_f = (float)(1 / sqrt(var + eps)).
 * Sums of a batch, float64 [sum x (O) | sum x^2 (O) | rows]: over the valid rows t < lens[b] (t < T) only. */
#define IMPALA_OBS_NORM_MAX_FEATURES 1024

/* Bytes of the workspace of impala_obs_normalize for T steps, B columns and O features (O up to
 * IMPALA_OBS_NORM_MAX_FEATURES, else IMPALA_ERR_BAD_ARG).  Its first bytes are counters the caller zeroes ONCE;
 * every launch leaves them zeroed. */
int64_t impala_obs_normalize_workspace(int T, int B, int O);

/* The step's first launch with obs_norm on, in place of impala_obs_unstack / impala_obs_u8_to_f32: reads the
 * slab's observations - dense (T+1, B, F) when k = 1, frames (T+k, B, F) otherwise (impala_batch_layout_frames),
 * float32 or uint8 (in_dtype) - and writes
 *   out (T+1, B, O = k F) float32:  out[r, o] = (x[r, o] - mu_f[o]) * r_f[o]  (float32, every row),
 *   sums (2 O + 1) float64:          the batch's sums over its valid rows.
 * The sums are deterministic: per feature, the rows are split into at most 1024 chunks of a size fixed by
 * (T+1) B alone; eight row lanes each add every eighth row of a chunk in row order, the chunk's partial adds the
 * lanes in order, eight lanes add every eighth chunk's partial in order and the total adds those in order.  No
 * float atomics: the same batch gives the same bits.  O > IMPALA_OBS_NORM_MAX_FEATURES returns
 * IMPALA_ERR_UNSUPPORTED_SHAPE, a short workspace IMPALA_ERR_WORKSPACE_TOO_SMALL. */
int impala_obs_normalize(const void* obs, int in_dtype, int T, int B, int F, int k, const int32_t* lens,
                         const float* norm, float* out, double* sums, void* workspace, int64_t workspace_bytes,
                         void* stream);

/* One launch after the optimizer: merges the batch (sums, summed over the ranks) into the statistics with
 * Chan's parallel merge in float64,
 *   n = n_a + n_b,  d = mean_b - mean_a,  mean = mean_a + d n_b / n,
 *   var = (var_a n_a + max(S2 - S1 mean_b, 0) + d^2 n_a n_b / n) / n     (n_b = 0 leaves them),
 * rewrites norm from them and writes `folded`: params with the W1 block(s) and b1 of each network folded into
 * raw-observation coordinates, W1' = W1 diag(r_f) (float32), b1' = b1 - W1' mu_f (float64 sum), every other entry
 * copied.  Network 0 is (w1_off0, b1_off0, H0); H1 = 0 means one network (shared torso).  ctl: two uint32 the
 * caller zeroes once (every launch leaves them zeroed).
 * gather != NULL (data-parallel, peer route): the sums are entries [sums_at, sums_at + 2 O + 1) of every rank's
 * slot of this rank's gather buffer for the step *seq (the gather optimizer has advanced it), added in rank order;
 * *err != 0 (the optimizer timed out) leaves everything untouched.  A timeout here sets *err and leaves the
 * statistics untouched; `folded` is then incomplete (the host raises on *err, as for the optimizer). */
int impala_obs_norm_update(double* stats, float* norm, const double* sums, double eps, const float* params,
                           float* folded, int64_t n_total, int O, int64_t w1_off0, int64_t b1_off0, int H0,
                           int64_t w1_off1, int64_t b1_off1, int H1, unsigned* ctl, const void* gather,
                           const long long* seq, int64_t slot_stride, int64_t buf_stride, int world, int64_t sums_at,
                           int* err, double timeout_s, void* stream);

/* Pieces of the reference's module-level loss helpers (learner.py:298-321) for callers that use
 * them individually instead of impala_vtrace_loss.  logits (M,A) f32 row-major, actions (M) i32.
 *   log_prob[m]    = log_softmax(logits[m])[actions[m]]           action_log_probs        (:298-303)
 *   neg_entropy[m] = sum_k p_k log p_k                            compute_entropy_loss    (:310-314)
 * backward: dlogits from the upstream gradients of the two outputs (either may be NULL = 0). */
int impala_policy_terms(const float* logits, const int32_t* actions, float* log_prob,
                        float* neg_entropy, int M, int A, void* stream);
int impala_policy_terms_backward(const float* logits, const int32_t* actions,
                                 const float* grad_log_prob, const float* grad_neg_entropy,
                                 float* dlogits, int M, int A, void* stream);

/* Float64 scalar reductions of f32 vectors: mode 0 = sum a, 1 = 0.5 sum a^2 (compute_baseline_loss,
 * learner.py:306-307), 2 = sum a*b (the sum in compute_policy_gradient_loss, :317-321). */
int impala_reduce(const float* a, const float* b, int64_t n, int mode, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* IMPALA_B200_H */
