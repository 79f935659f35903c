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
 *   obs (T+1,B,O) f32 | beh_logits (T,B,A) f32 | actions (T,B) i32 |
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

/* Host slab -> device slab, async on `stream` (host memory should be pinned). */
int impala_ingest(void* dev_slab, const void* host_slab, int64_t bytes, void* stream);

/* Data-parallel ingest: copy columns [b0, b0 + B_local) of a host slab laid out by
 * impala_batch_layout(T, B, O, A) into a device slab laid out by impala_batch_layout(T, B_local, O, A)
 * (strided 2-D DMAs; the host slab should be page-locked).  Every rank of a data-parallel learner
 * pulls its own shard of the actors' shared-memory slab over its own PCIe link. */
int impala_ingest_shard(void* dev_slab, const void* host_slab, int T, int B, int O, int A, int b0,
                        int B_local, void* stream);

/* out[m, :] = relu(x[m, :] W1^T + b1) W2^T + b2 for m < M.
 * Replaces MlpPolicy.forward / MlpValueFn.forward in eval mode
 * (models.py:23-25, :51-52) as called at learner.py:112-113 on the flattened
 * (T*B, O) / ((T+1)*B, O) batch.  x row-major (M,O); out row-major (M,N2). */
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
 * that was never zeroed it traps - a launch failure, not a hang). */
int64_t impala_mlp_backward_workspace(int M, int O, int H, int N2);

/* Gradient of sum_m <dout[m,:], mlp(x[m,:])> w.r.t. the parameter block, written
 * (not accumulated) as float64 into grad[0 .. total) in parameter-block layout
 * (pad entries = 0).  Hidden activations are recomputed from x, nothing is saved
 * by the forward.  Replaces the MLP part of loss.backward() at learner.py:175. */
int impala_mlp_backward(const float* x, const float* params, const float* dout, double* grad,
                        void* workspace, int64_t workspace_bytes, int M, int O, int H, int N2,
                        void* stream);

/* The MLP part of the single loss.backward() at learner.py:175 for both networks in one launch:
 * same results as impala_mlp_backward(policy; dout = dlogits) followed by
 * impala_mlp_backward(value_fn; dout = dv), each with its own workspace (sized by
 * impala_mlp_backward_workspace, zero-filled once). */
int impala_mlp_backward_pair(const float* x, const float* params_pi, const float* params_vf,
                             const float* dlogits, const float* dv, double* grad_pi, double* grad_vf,
                             void* workspace_pi, int64_t workspace_pi_bytes, void* workspace_vf,
                             int64_t workspace_vf_bytes, int M_pi, int M_vf, int O, int H_pi,
                             int H_vf, int A, void* stream);

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

/* Per-group gradient clipping + Adam in one launch (learner.py:176-183).
 *   params/m/v: f32 [n_total]; grad: f64 [n_total] (the possibly all-reduced sum);
 *   group 0 = [0, n_policy) (policy net), group 1 = [n_policy, n_total) (value net);
 *   each group is scaled by min(1, max_norm / (||g||_2 + 1e-6)) as
 *   torch.nn.utils.clip_grad_norm_ does, then one Adam step (no weight decay) with
 *   bias correction from the device-side optimizer state (updated by the kernel):
 *   state = int64[3] {step count, beta1^step, beta2^step as float64 bits}; all zero = fresh.
 *   norms_out (f64[2], may be NULL) receives the two pre-clip norms. */
int impala_clip_adam(float* params, const double* grad, float* m, float* v, int64_t* state,
                     int64_t n_policy, int64_t n_total, float max_norm, float lr, float beta1,
                     float beta2, float eps, double* norms_out, void* stream);

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
int impala_gather_clip_adam(float* params, double* reduced, const void* gather, long long* seq,
                            int64_t slot_stride, int64_t buf_stride, int world, int n_extra, float* m,
                            float* v, int64_t* state, int64_t n_policy, int64_t n_total,
                            float max_norm, float lr, float beta1, float beta2, float eps,
                            double* norms_out, int* err, double timeout_s, void* stream);

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
