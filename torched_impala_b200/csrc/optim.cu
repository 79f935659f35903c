// Per-group gradient clipping + Adam (or RMSprop) + step counter in ONE launch
// (reference learner.py:176-183: two clip_grad_norm_ calls, Adam.step, LambdaLR.step).
//
// The parameter vector is tiny (14 144 floats at H=256, 69 312 at H=512) but the two clip
// norms need every gradient entry before any parameter can move.  One thread-block
// cluster of 8 CTAs (8 x 1024 threads, co-scheduled by hardware) does both phases in a
// single launch: each CTA reduces the squares of its slice in float64, the 8 partial pairs
// are exchanged through distributed shared memory, one cluster barrier later every CTA
// holds the same two norms and applies the update to its slice.  The gradient arrives as float64
// (sum of per-CTA float32 partials, possibly all-reduced over ranks) and the norms are reduced
// in float64; optimizer state stays float32 in HBM and the per-element update runs in float32.
//
// Both kernels are written once, as a body templated on the update rule (AdamRule, RmspropRule)
// and on where the learning rate comes from (LrScalar: a launch argument; LrTable: a device table
// indexed by the step counter, so one captured CUDA graph serves a whole learning-rate schedule).
// impala_clip_adam / impala_gather_clip_adam are the <AdamRule, LrScalar> instantiations.
//
// The body's third parameter is the value normalization (NoPopart, Popart): with Popart one thread of CTA 0
// forms the new value statistics from the eight V-trace sums before the norm exchange's cluster barrier, the
// other CTAs read them through distributed shared memory, and phase 2 rescales the value head's entries right
// after their update, so the PopArt step needs no launch of its own.
#include <cooperative_groups.h>
#include <math.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kAdamThreads = 1024;
constexpr int kAdamCluster = 8;

// ---- learning-rate sources: the rate of the update after `t` completed ones (t = state[0])
struct LrScalar {
    float lr;
    __device__ __forceinline__ float at(int64_t) const { return lr; }
};

// LambdaLR as a table: update n (1-based) uses table[n - 1]; steps past the end keep the last entry.
// The table is only read, so the rate changes from one replay of a captured graph to the next.
struct LrTable {
    const float* __restrict__ table;
    int64_t n;
    __device__ __forceinline__ float at(int64_t t) const { return table[t <= 0 ? 0 : (t < n ? t : n - 1)]; }
};

// ---- update rules.  Each rule sees the clipped float32 gradient g of one entry with its float32 state
// (p, m, v) and writes what it changes; k0 / k1 are the two per-step constants `prepare` left for every
// thread (thread 64 runs `prepare` once, before the update; `finish` advances the state at the very end).

// torch.optim.Adam (no weight decay).  state = int64[3] {step count, beta1^t, beta2^t as float64 bits}
// (all-zero state = fresh optimizer): running powers replace two float64 pow() calls per step.
struct AdamRule {
    float b1, b2, eps;
    __device__ __forceinline__ bool reads_m() const { return true; }
    __device__ __forceinline__ void prepare(const int64_t* __restrict__ state, float lr, float* s_k,
                                            double* s_pow) const {
        const double p1 = state[0] == 0 ? 1.0 : __longlong_as_double(state[1]);
        const double p2 = state[0] == 0 ? 1.0 : __longlong_as_double(state[2]);
        s_pow[0] = p1 * (double)b1, s_pow[1] = p2 * (double)b2;
        s_k[0] = (float)((double)lr / (1.0 - s_pow[0]));  // step_size = lr / (1 - beta1^t)
        s_k[1] = (float)(1.0 / sqrt(1.0 - s_pow[1]));     // 1 / sqrt(1 - beta2^t)
    }
    __device__ __forceinline__ void apply(int64_t i, float g, float p, float mi, float vi, float step_size,
                                          float inv_bc2_sqrt, float* __restrict__ params, float* __restrict__ m,
                                          float* __restrict__ v) const {
        mi = fmaf(b1, mi, (1.f - b1) * g);
        vi = fmaf(b2, vi, (1.f - b2) * g * g);
        const float denom = fmaf(sqrtf(vi), inv_bc2_sqrt, eps);
        params[i] = p - step_size * mi / denom;
        m[i] = mi;
        v[i] = vi;
    }
    __device__ __forceinline__ void finish(int64_t* __restrict__ state, const double* s_pow) const {
        state[0] += 1;
        state[1] = __double_as_longlong(s_pow[0]);
        state[2] = __double_as_longlong(s_pow[1]);
    }
};

// torch.optim.RMSprop (not centered, no weight decay): square_avg in v, the momentum buffer in m (neither read
// nor written when momentum = 0), eps added outside the square root as torch does.  Only state[0] is used.
struct RmspropRule {
    float alpha, momentum, eps;
    __device__ __forceinline__ bool reads_m() const { return momentum > 0.f; }
    __device__ __forceinline__ void prepare(const int64_t* __restrict__, float lr, float* s_k, double*) const {
        s_k[0] = lr;
        s_k[1] = 0.f;
    }
    __device__ __forceinline__ void apply(int64_t i, float g, float p, float mi, float vi, float lr, float,
                                          float* __restrict__ params, float* __restrict__ m,
                                          float* __restrict__ v) const {
        vi = fmaf(alpha, vi, (1.f - alpha) * g * g);
        const float avg = sqrtf(vi) + eps;
        if (momentum > 0.f) {
            mi = fmaf(momentum, mi, g / avg);
            params[i] = p - lr * mi;
            m[i] = mi;
        } else {
            params[i] = p - lr * (g / avg);
        }
        v[i] = vi;
    }
    __device__ __forceinline__ void finish(int64_t* __restrict__ state, const double*) const { state[0] += 1; }
};

// ---- value normalization.  NoPopart: the plain kernels (every member compiles to nothing).
struct NoPopart {
    static constexpr bool kOn = false;
    static constexpr int kShared = 1;
    __device__ __forceinline__ void form(const double*, double*) const {}
    __device__ __forceinline__ void rescale(int64_t, float*, const double*) const {}
    __device__ __forceinline__ void finish(const double*) const {}
};

// PopArt (van Hasselt et al. 2016), single task: stats = float64 {mu, nu, sigma, mu_loss, sigma_loss} in device
// memory, the first three the running statistics, the last two those the update's loss used (written with the
// new ones, so a logged copy of the five is self-consistent).  `form` (one thread) turns the sums of the batch
// (sums[0] = n, [5] = sum vs, [6] = sum vs^2, impala_vtrace_loss_diag's layout) into
//   s = {mu', nu', sigma', sigma / sigma', (mu - mu') / sigma', mu, sigma}
// and `rescale` keeps the unnormalized value output sigma n + mu of the updated head: W2 <- W2 sigma / sigma',
// b2 <- (sigma b2 + mu - mu') / sigma'.  n = 0 keeps the statistics (and the rescale is the identity).
struct Popart {
    static constexpr bool kOn = true;
    static constexpr int kShared = 7;
    double* __restrict__ stats;
    int64_t sums_at, w2_off, w2_len, b2_off;
    float beta;
    __device__ __forceinline__ void form(const double* sums, double* s) const {
        const double mu = stats[0], nu = stats[1], sg = stats[2], n = sums[0];
        double mu1 = mu, nu1 = nu, sg1 = sg;
        if (n > 0.0) {
            const double b = (double)beta;
            mu1 = (1.0 - b) * mu + b * (sums[5] / n);
            nu1 = (1.0 - b) * nu + b * (sums[6] / n);
            sg1 = fmin(fmax(sqrt(fmax(nu1 - mu1 * mu1, 0.0)), 1e-4), 1e6);
        }
        s[0] = mu1, s[1] = nu1, s[2] = sg1, s[3] = sg / sg1, s[4] = (mu - mu1) / sg1, s[5] = mu, s[6] = sg;
    }
    __device__ __forceinline__ void rescale(int64_t i, float* __restrict__ params, const double* s) const {
        if (i >= w2_off && i < w2_off + w2_len) params[i] = (float)((double)params[i] * s[3]);
        else if (i == b2_off) params[i] = (float)fma((double)params[i], s[3], s[4]);
    }
    __device__ __forceinline__ void finish(const double* s) const {
        stats[0] = s[0], stats[1] = s[1], stats[2] = s[2], stats[3] = s[5], stats[4] = s[6];
    }
};

// torch.nn.utils.clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1; a NaN norm gives a NaN
// coefficient (torch.clamp propagates NaN, fmin would return the 1)
__device__ __forceinline__ float clip_coef(double norm, float max_norm) {
    return isnan(norm) ? (float)norm : (float)fmin(1.0, (double)max_norm / (norm + 1e-6));
}

template <class Rule, class Lr, class Pop = NoPopart>
__device__ __forceinline__ void clip_update(float* __restrict__ params, const double* __restrict__ grad,
                                            float* __restrict__ m, float* __restrict__ v,
                                            int64_t* __restrict__ state, int64_t n_policy, int64_t n_total,
                                            float max_norm, Lr lr, Rule rule, double* __restrict__ norms_out,
                                            Pop pop = Pop{}) {
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ double s_pop[Pop::kShared];  // Popart: the statistics CTA 0 forms (read by the peers)
    __shared__ double s_warp[2][kAdamThreads / 32];
    __shared__ double s_cta[2];   // this CTA's partial sums of squares (read by the peers)
    __shared__ float s_coef[2];
    __shared__ float s_bias[2];   // the rule's two per-step constants
    __shared__ double s_pow[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t first = (int64_t)cluster.block_rank() * kAdamThreads + tid;
    const int64_t stride = (int64_t)kAdamCluster * kAdamThreads;

    // phase 1: this thread's gradient entries (kept in registers when there are at most two, the
    // benchmark sizes) and the float32 state they will update - all loads issued up front
    constexpr int kKeep = 2;
    double gk[kKeep];
    float pk[kKeep], mk[kKeep], vk[kKeep];
    double ss0 = 0.0, ss1 = 0.0;
#pragma unroll
    for (int k = 0; k < kKeep; ++k) {  // optimizer state: not touched by the backward, loaded before the wait
        const int64_t i = first + k * stride;
        pk[k] = i < n_total ? params[i] : 0.f;
        mk[k] = i < n_total && rule.reads_m() ? m[i] : 0.f;
        vk[k] = i < n_total ? v[i] : 0.f;
    }
    pdl_wait();  // the gradient comes from the backward kernel
#pragma unroll
    for (int k = 0; k < kKeep; ++k) {
        const int64_t i = first + k * stride;
        gk[k] = i < n_total ? grad[i] : 0.0;
    }
#pragma unroll
    for (int k = 0; k < kKeep; ++k) {
        const int64_t i = first + k * stride;
        if (i < n_policy) ss0 += gk[k] * gk[k];
        else ss1 += gk[k] * gk[k];
    }
    for (int64_t i = first + kKeep * stride; i < n_total; i += stride) {
        const double g = grad[i];
        if (i < n_policy) ss0 += g * g;
        else ss1 += g * g;
    }
    ss0 = warp_sum_f64(ss0);
    ss1 = warp_sum_f64(ss1);
    if (lane == 0) s_warp[0][warp] = ss0, s_warp[1][warp] = ss1;
    if (tid == 64)  // learning rate and bias corrections (nobody writes state before the end)
        rule.prepare(state, lr.at(state[0]), s_bias, s_pow);
    if constexpr (Pop::kOn) {
        if (cluster.block_rank() == 0 && tid == 96) pop.form(grad + pop.sums_at, s_pop);
    }
    __syncthreads();
    if (tid < 2) {
        double s = 0.0;
        for (int i = 0; i < kAdamThreads / 32; ++i) s += s_warp[tid][i];
        s_cta[tid] = s;
    }
    cluster.sync();  // all 8 partial pairs (and CTA 0's statistics) are in place
    if (tid < 2) {
        double s = 0.0;
        for (int r = 0; r < kAdamCluster; ++r) s += *cluster.map_shared_rank(&s_cta[tid], r);
        const double norm = sqrt(s);
        s_coef[tid] = clip_coef(norm, max_norm);
        if (norms_out && cluster.block_rank() == 0) norms_out[tid] = norm;
    }
    __syncthreads();
    // phase 2: the update in float32 arithmetic (the state is float32; one step's rounding is ~1e-7)
    const float k0 = s_bias[0], k1 = s_bias[1];
    const float c0 = s_coef[0], c1 = s_coef[1];
    const double* pop_s = Pop::kOn ? cluster.map_shared_rank(s_pop, 0) : s_pop;
    auto update = [&](int64_t i, float g, float p, float mi, float vi) {
        rule.apply(i, g * (i < n_policy ? c0 : c1), p, mi, vi, k0, k1, params, m, v);
        pop.rescale(i, params, pop_s);  // the value head, right after its update
    };
#pragma unroll
    for (int k = 0; k < kKeep; ++k) {
        const int64_t i = first + k * stride;
        if (i < n_total) update(i, (float)gk[k], pk[k], mk[k], vk[k]);
    }
    for (int64_t i = first + kKeep * stride; i < n_total; i += stride)
        update(i, (float)grad[i], params[i], rule.reads_m() ? m[i] : 0.f, v[i]);
    cluster.sync();  // peers finished reading this CTA's shared memory; every CTA has read state
    if (cluster.block_rank() == 0 && tid == 64) {
        rule.finish(state, s_pow);
        pop.finish(s_pop);
    }
}

__global__ void __cluster_dims__(kAdamCluster, 1, 1) __launch_bounds__(kAdamThreads)
clip_adam_kernel(float* __restrict__ params, const double* __restrict__ grad, float* __restrict__ m,
                 float* __restrict__ v, int64_t* __restrict__ state, int64_t n_policy,
                 int64_t n_total, float max_norm, float lr, float beta1, float beta2, float eps,
                 double* __restrict__ norms_out) {
    clip_update(params, grad, m, v, state, n_policy, n_total, max_norm, LrScalar{lr}, AdamRule{beta1, beta2, eps},
                norms_out);
}

// Rule = AdamRule: h0, h1 = beta1, beta2.  Rule = RmspropRule: h0, h1 = alpha, momentum.
template <class Rule>
__global__ void __cluster_dims__(kAdamCluster, 1, 1) __launch_bounds__(kAdamThreads)
clip_optim_kernel(float* __restrict__ params, const double* __restrict__ grad, float* __restrict__ m,
                  float* __restrict__ v, int64_t* __restrict__ state, int64_t n_policy, int64_t n_total,
                  float max_norm, const float* __restrict__ lr_table, int64_t n_lr, float h0, float h1, float eps,
                  double* __restrict__ norms_out) {
    clip_update(params, grad, m, v, state, n_policy, n_total, max_norm, LrTable{lr_table, n_lr}, Rule{h0, h1, eps},
                norms_out);
}

template <class Rule>
__global__ void __cluster_dims__(kAdamCluster, 1, 1) __launch_bounds__(kAdamThreads)
clip_optim_popart_kernel(float* __restrict__ params, const double* __restrict__ grad, float* __restrict__ m,
                         float* __restrict__ v, int64_t* __restrict__ state, int64_t n_policy, int64_t n_total,
                         float max_norm, const float* __restrict__ lr_table, int64_t n_lr, float h0, float h1,
                         float eps, double* __restrict__ norms_out, Popart pop) {
    clip_update(params, grad, m, v, state, n_policy, n_total, max_norm, LrTable{lr_table, n_lr}, Rule{h0, h1, eps},
                norms_out, pop);
}


// ---------------------------------------------------------------------------------------------
// Data-parallel learners: one-shot all-reduce over NVLink peer memory - PUSH, LL format.
//
// Every rank owns a gather buffer  G[2 parities][world slots][slot_stride]  of 16-byte LL elements
// (common.cuh) that the other ranks of the node have mapped (CUDA IPC).  The producer of a rank's
// float64 [gradient | extra scalars] contribution - the reduction tail of the paired tensor-core
// backward kernel (mlp_bwd_tc.cu), or peer_push_kernel below for shapes that kernel does not cover
// - STORES every value, tagged with the step number, into slot `rank` of every rank's buffer:
// posted NVLink writes, nobody waits for a round trip, no fence, no flag.  The optimizer kernel of
// each rank polls the `world` slots of its OWN buffer (local memory) until each element carries
// the current step, adds them in rank order - every rank forms bit-identical sums, so the
// replicas cannot drift - and runs the clip norms and the update on the sum.  The data path costs one
// NVLink one-way latency.
//
// The buffers are double-buffered by step parity, which makes an "I have read your slot" message
// unnecessary: a rank overwrites parity s & 1 in the backward of step s + 2, i.e. after its
// optimizer kernel of step s + 1 consumed every peer's step-(s + 1) values - and a peer sends
// those only from a backward that runs after its optimizer kernel of step s (the one that read
// the slots) has finished.  The step number lives in device memory (`seq`, advanced by the
// optimizer kernel), so producer and consumer derive parity and tag themselves and ONE captured
// CUDA graph serves every step.
//
// A rank that never delivers (its host is stuck) does not kill the others' CUDA contexts: after
// `timeout_ns` of polling the optimizer kernel sets an error word, leaves parameters, optimizer
// state and `seq` untouched and exits normally; the host raises when it reads the word.
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

constexpr int kPushThreads = 256;  // remote stores are credit-limited per SM: spread the message over many CTAs

// Stand-alone producer: local[0, n) -> slot `rank` of every rank's gather buffer.
__global__ void __launch_bounds__(kPushThreads)
peer_push_kernel(const double* __restrict__ local, int64_t n, PushArgs p) {
    pdl_wait();  // `local` comes from the backward kernel
    const long long step = *p.seq + 1;
    const int64_t off = (step & 1) * p.buf_stride + (int64_t)p.rank * p.slot_stride;
    for (int64_t i = (int64_t)blockIdx.x * kPushThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kPushThreads) {
        const double v = local[i];
#pragma unroll 8
        for (int r = 0; r < p.world; ++r) ll_store(p.gather[r] + off + i, v, (unsigned)step);
    }
}

// Consumer: poll the local slots, add them in rank order, clip + update.
template <class Rule, class Lr, class Pop = NoPopart>
__device__ __forceinline__ void gather_clip_update(float* __restrict__ params, double* __restrict__ reduced,
                                                   const ulonglong2* __restrict__ gather, long long* __restrict__ seq,
                                                   int64_t slot_stride, int64_t buf_stride, int world, int n_extra,
                                                   float* __restrict__ m, float* __restrict__ v,
                                                   int64_t* __restrict__ state, int64_t n_policy, int64_t n_total,
                                                   float max_norm, Lr lr, Rule rule, double* __restrict__ norms_out,
                                                   int* __restrict__ err, unsigned long long timeout_ns,
                                                   Pop pop = Pop{}) {
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ double s_pop[Pop::kShared];  // Popart: the statistics CTA 0 forms from the summed extras
    __shared__ double s_warp[2][kAdamThreads / 32];
    __shared__ double s_cta[2];
    __shared__ int s_abort;     // a thread of this CTA gave up waiting (read by the peers of the cluster)
    __shared__ int s_any_abort;
    __shared__ float s_coef[2];
    __shared__ float s_bias[2];
    __shared__ double s_pow[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int crank = (int)cluster.block_rank();
    const int64_t first = (int64_t)crank * kAdamThreads + tid;
    const int64_t stride = (int64_t)kAdamCluster * kAdamThreads;

    // optimizer state that does not depend on the peers: issued before anything else
    constexpr int kKeep = 2, kMaxWorld = 8, kPoll = 2;  // one NVLink node
    float pk[kKeep], mk[kKeep], vk[kKeep];
#pragma unroll
    for (int k = 0; k < kKeep; ++k) {
        const int64_t i = first + k * stride;
        pk[k] = i < n_total ? params[i] : 0.f;
        mk[k] = i < n_total && rule.reads_m() ? m[i] : 0.f;
        vk[k] = i < n_total ? v[i] : 0.f;
    }
    if (tid == 0) s_abort = 0;
    if (tid == 64)  // learning rate and bias corrections (nobody writes state before the end)
        rule.prepare(state, lr.at(state[0]), s_bias, s_pow);
    pdl_wait();  // orders this kernel behind the local backward (its successors rely on that)
    const long long step64 = *seq + 1;
    const unsigned step = (unsigned)step64;
    __syncthreads();

    // rank-ordered sum of entry i: the loads of kPoll ranks are issued together, then each is re-polled
    // until it carries this step's tag (local memory: the peers' values arrive by themselves).  kPoll = 2:
    // more 16-byte words in flight at the three inlined call sites exceed the 64 registers a 1024-thread
    // CTA allows (all eight spilled 232 bytes to local memory, four still 12).
    const ulonglong2* gb = gather + (step64 & 1) * buf_stride;
    const unsigned long long t_start = global_ns();
    bool ok = true;
    auto gsum = [&](int64_t i) {
        double s = 0.0;
#pragma unroll
        for (int r0 = 0; r0 < kMaxWorld; r0 += kPoll) {
            ulonglong2 w[kPoll];
#pragma unroll
            for (int r = 0; r < kPoll; ++r)
                if (r0 + r < world) w[r] = ll_load(gb + (r0 + r) * slot_stride + i);
#pragma unroll
            for (int r = 0; r < kPoll; ++r) {
                if (r0 + r < world) {
                    unsigned spins = 0;
                    while (!ll_ready(w[r], step)) {
                        if ((++spins & 255u) == 0 && global_ns() - t_start > timeout_ns) {
                            ok = false;
                            break;
                        }
                        if (spins > 16) __nanosleep(20);
                        w[r] = ll_load(gb + (r0 + r) * slot_stride + i);
                    }
                    s += ll_value(w[r]);
                }
            }
        }
        return s;
    };
    double gk[kKeep];
    double ss0 = 0.0, ss1 = 0.0;
#pragma unroll
    for (int k = 0; k < kKeep; ++k) {
        const int64_t i = first + k * stride;
        gk[k] = i < n_total ? gsum(i) : 0.0;
        if (i < n_total) reduced[i] = gk[k];
        if (i < n_policy) ss0 += gk[k] * gk[k];
        else ss1 += gk[k] * gk[k];
    }
    for (int64_t i = first + kKeep * stride; i < n_total; i += stride) {
        const double g = gsum(i);
        reduced[i] = g;
        if (i < n_policy) ss0 += g * g;
        else ss1 += g * g;
    }
    if (crank == 0 && tid < n_extra) reduced[n_total + tid] = gsum(n_total + tid);  // logged scalars
    if (!ok) s_abort = 1;
    ss0 = warp_sum_f64(ss0);
    ss1 = warp_sum_f64(ss1);
    if (lane == 0) s_warp[0][warp] = ss0, s_warp[1][warp] = ss1;
    __syncthreads();
    if constexpr (Pop::kOn) {  // the rank-ordered sums of all ranks' V-trace sums are in `reduced` now
        if (crank == 0 && tid == 96) pop.form(reduced + pop.sums_at, s_pop);
    }
    if (tid < 2) {
        double s = 0.0;
        for (int i = 0; i < kAdamThreads / 32; ++i) s += s_warp[tid][i];
        s_cta[tid] = s;
    }
    cluster.sync();  // all 8 partial pairs (and abort flags, CTA 0's statistics) are in place
    if (tid == 0) {
        int ab = 0;
        for (int r = 0; r < kAdamCluster; ++r) ab |= *cluster.map_shared_rank(&s_abort, r);
        s_any_abort = ab;
    }
    if (tid < 2) {
        double s = 0.0;
        for (int r = 0; r < kAdamCluster; ++r) s += *cluster.map_shared_rank(&s_cta[tid], r);
        const double norm = sqrt(s);
        s_coef[tid] = clip_coef(norm, max_norm);
        if (norms_out && crank == 0) norms_out[tid] = norm;
    }
    __syncthreads();
    if (!s_any_abort) {
        const float k0 = s_bias[0], k1 = s_bias[1];
        const float c0 = s_coef[0], c1 = s_coef[1];
        const double* pop_s = Pop::kOn ? cluster.map_shared_rank(s_pop, 0) : s_pop;
        auto update = [&](int64_t i, float g, float p, float mi, float vi) {
            rule.apply(i, g * (i < n_policy ? c0 : c1), p, mi, vi, k0, k1, params, m, v);
            pop.rescale(i, params, pop_s);
        };
#pragma unroll
        for (int k = 0; k < kKeep; ++k) {
            const int64_t i = first + k * stride;
            if (i < n_total) update(i, (float)gk[k], pk[k], mk[k], vk[k]);
        }
        for (int64_t i = first + kKeep * stride; i < n_total; i += stride)
            update(i, (float)reduced[i], params[i], rule.reads_m() ? m[i] : 0.f, v[i]);
    }
    cluster.sync();  // peers finished reading this CTA's shared memory; every CTA has read state
    if (crank == 0 && tid == 64) {
        if (s_any_abort) {
            if (err) *err = 1;  // the host raises; state, statistics and seq stay as they were
        } else {
            rule.finish(state, s_pow);
            pop.finish(s_pop);
            *seq = step64;
        }
    }
}

__global__ void __cluster_dims__(kAdamCluster, 1, 1) __launch_bounds__(kAdamThreads)
gather_clip_adam_kernel(float* __restrict__ params, double* __restrict__ reduced,
                        const ulonglong2* __restrict__ gather, long long* __restrict__ seq,
                        int64_t slot_stride, int64_t buf_stride, int world, int n_extra,
                        float* __restrict__ m, float* __restrict__ v, int64_t* __restrict__ state,
                        int64_t n_policy, int64_t n_total, float max_norm, float lr, float beta1,
                        float beta2, float eps, double* __restrict__ norms_out, int* __restrict__ err,
                        unsigned long long timeout_ns) {
    gather_clip_update(params, reduced, gather, seq, slot_stride, buf_stride, world, n_extra, m, v, state, n_policy,
                       n_total, max_norm, LrScalar{lr}, AdamRule{beta1, beta2, eps}, norms_out, err, timeout_ns);
}

template <class Rule>
__global__ void __cluster_dims__(kAdamCluster, 1, 1) __launch_bounds__(kAdamThreads)
gather_clip_optim_kernel(float* __restrict__ params, double* __restrict__ reduced,
                         const ulonglong2* __restrict__ gather, long long* __restrict__ seq,
                         int64_t slot_stride, int64_t buf_stride, int world, int n_extra,
                         float* __restrict__ m, float* __restrict__ v, int64_t* __restrict__ state,
                         int64_t n_policy, int64_t n_total, float max_norm, const float* __restrict__ lr_table,
                         int64_t n_lr, float h0, float h1, float eps, double* __restrict__ norms_out,
                         int* __restrict__ err, unsigned long long timeout_ns) {
    gather_clip_update(params, reduced, gather, seq, slot_stride, buf_stride, world, n_extra, m, v, state, n_policy,
                       n_total, max_norm, LrTable{lr_table, n_lr}, Rule{h0, h1, eps}, norms_out, err, timeout_ns);
}

template <class Rule>
__global__ void __cluster_dims__(kAdamCluster, 1, 1) __launch_bounds__(kAdamThreads)
gather_clip_optim_popart_kernel(float* __restrict__ params, double* __restrict__ reduced,
                                const ulonglong2* __restrict__ gather, long long* __restrict__ seq,
                                int64_t slot_stride, int64_t buf_stride, int world, int n_extra,
                                float* __restrict__ m, float* __restrict__ v, int64_t* __restrict__ state,
                                int64_t n_policy, int64_t n_total, float max_norm, const float* __restrict__ lr_table,
                                int64_t n_lr, float h0, float h1, float eps, double* __restrict__ norms_out,
                                int* __restrict__ err, unsigned long long timeout_ns, Popart pop) {
    gather_clip_update(params, reduced, gather, seq, slot_stride, buf_stride, world, n_extra, m, v, state, n_policy,
                       n_total, max_norm, LrTable{lr_table, n_lr}, Rule{h0, h1, eps}, norms_out, err, timeout_ns, pop);
}

// The checks of impala_clip_optim / impala_gather_clip_optim beyond those of the Adam entry points.
bool bad_optim_args(const float* lr_table, int64_t n_lr, int rule, float h0, float h1, float eps) {
    if (!lr_table || n_lr < 1 || !(eps >= 0.f)) return true;
    if (rule == IMPALA_OPT_ADAM) return false;
    if (rule == IMPALA_OPT_RMSPROP) return !(h0 >= 0.f && h0 < 1.f) || !(h1 >= 0.f);
    return true;
}

// The checks of the PopArt entry points beyond those of impala_clip_optim: the statistics, beta in (0, 1] and a
// value head (W2 block and b2, disjoint) inside the value net's entries [n_policy, n_total).
bool bad_popart_args(const double* popart, int64_t n_policy, int64_t n_total, int64_t w2_off, int64_t w2_len,
                     int64_t b2_off, float beta) {
    if (!popart || !(beta > 0.f && beta <= 1.f)) return true;
    if (w2_len < 1 || w2_off < n_policy || w2_off > n_total - w2_len) return true;
    if (b2_off < n_policy || b2_off >= n_total) return true;
    return b2_off >= w2_off && b2_off < w2_off + w2_len;
}

unsigned long long timeout_ns_of(double timeout_s) {
    return timeout_s > 0 ? (unsigned long long)(timeout_s * 1e9) : 600ull * 1000000000ull;
}

}  // namespace

extern "C" int impala_clip_adam(float* params, const double* grad, float* m, float* v,
                                int64_t* state, int64_t n_policy, int64_t n_total, float max_norm,
                                float lr, float beta1, float beta2, float eps, double* norms_out,
                                void* stream) {
    if (!params || !grad || !m || !v || !state) return IMPALA_ERR_BAD_ARG;
    if (n_total < 1 || n_policy < 0 || n_policy > n_total) return IMPALA_ERR_BAD_ARG;
    const cudaError_t e = impala_launch(clip_adam_kernel, kAdamCluster, kAdamThreads, 0, (cudaStream_t)stream, true, params,
                                        grad, m, v, state, n_policy, n_total, max_norm, lr, beta1, beta2, eps, norms_out);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

extern "C" int impala_clip_optim(float* params, const double* grad, float* m, float* v, int64_t* state,
                                 int64_t n_policy, int64_t n_total, float max_norm, const float* lr_table,
                                 int64_t n_lr, int rule, float h0, float h1, float eps, double* norms_out,
                                 void* stream) {
    if (!params || !grad || !m || !v || !state) return IMPALA_ERR_BAD_ARG;
    if (n_total < 1 || n_policy < 0 || n_policy > n_total) return IMPALA_ERR_BAD_ARG;
    if (bad_optim_args(lr_table, n_lr, rule, h0, h1, eps)) return IMPALA_ERR_BAD_ARG;
    const auto kernel = rule == IMPALA_OPT_ADAM ? clip_optim_kernel<AdamRule> : clip_optim_kernel<RmspropRule>;
    const cudaError_t e = impala_launch(kernel, kAdamCluster, kAdamThreads, 0, (cudaStream_t)stream, true, params, grad,
                                        m, v, state, n_policy, n_total, max_norm, lr_table, n_lr, h0, h1, eps, norms_out);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

extern "C" int impala_peer_push(const double* local, int64_t n, void* const* peer_gather, const long long* seq,
                                int64_t slot_stride, int64_t buf_stride, int rank, int world, void* stream) {
    if (!local || !peer_gather || !seq) return IMPALA_ERR_BAD_ARG;
    if (n < 1 || world < 1 || world > 8 || rank < 0 || rank >= world) return IMPALA_ERR_BAD_ARG;
    if (slot_stride < n || buf_stride < (int64_t)world * slot_stride) return IMPALA_ERR_BAD_ARG;
    PushArgs p{reinterpret_cast<ulonglong2* const*>(peer_gather), seq, slot_stride, buf_stride, rank, world};
    int sms = 0;
    cudaError_t e = impala_sm_count(&sms);
    if (e != cudaSuccess) return (int)e;
    int grid = (int)((n + kPushThreads - 1) / kPushThreads);
    if (grid > sms) grid = sms;
    e = impala_launch(peer_push_kernel, grid, kPushThreads, 0, (cudaStream_t)stream, true, local, n, p);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

// The checks both gather entry points make.
static bool bad_gather_args(float* params, double* reduced, const void* gather, long long* seq, int64_t slot_stride,
                            int64_t buf_stride, int world, int n_extra, float* m, float* v, int64_t* state,
                            int64_t n_policy, int64_t n_total) {
    if (!params || !reduced || !gather || !seq || !m || !v || !state) return true;
    if (n_total < 1 || n_policy < 0 || n_policy > n_total) return true;
    if (world < 1 || world > 8 || n_extra < 0 || n_extra > kAdamThreads) return true;
    if (slot_stride < n_total + n_extra || buf_stride < (int64_t)world * slot_stride) return true;
    return (reinterpret_cast<uintptr_t>(gather) & 15) != 0;
}

extern "C" int impala_gather_clip_adam(float* params, double* reduced, const void* gather, long long* seq,
                                       int64_t slot_stride, int64_t buf_stride, int world, int n_extra, float* m,
                                       float* v, int64_t* state, int64_t n_policy, int64_t n_total, float max_norm,
                                       float lr, float beta1, float beta2, float eps, double* norms_out, int* err,
                                       double timeout_s, void* stream) {
    if (bad_gather_args(params, reduced, gather, seq, slot_stride, buf_stride, world, n_extra, m, v, state, n_policy,
                        n_total))
        return IMPALA_ERR_BAD_ARG;
    const cudaError_t e = impala_launch(gather_clip_adam_kernel, kAdamCluster, kAdamThreads, 0, (cudaStream_t)stream, true,
                                        params, reduced, static_cast<const ulonglong2*>(gather), seq, slot_stride, buf_stride,
                                        world, n_extra, m, v, state, n_policy, n_total, max_norm, lr, beta1, beta2, eps,
                                        norms_out, err, timeout_ns_of(timeout_s));
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

extern "C" int impala_gather_clip_optim(float* params, double* reduced, const void* gather, long long* seq,
                                        int64_t slot_stride, int64_t buf_stride, int world, int n_extra, float* m,
                                        float* v, int64_t* state, int64_t n_policy, int64_t n_total, float max_norm,
                                        const float* lr_table, int64_t n_lr, int rule, float h0, float h1, float eps,
                                        double* norms_out, int* err, double timeout_s, void* stream) {
    if (bad_gather_args(params, reduced, gather, seq, slot_stride, buf_stride, world, n_extra, m, v, state, n_policy,
                        n_total))
        return IMPALA_ERR_BAD_ARG;
    if (bad_optim_args(lr_table, n_lr, rule, h0, h1, eps)) return IMPALA_ERR_BAD_ARG;
    const auto kernel = rule == IMPALA_OPT_ADAM ? gather_clip_optim_kernel<AdamRule> : gather_clip_optim_kernel<RmspropRule>;
    const cudaError_t e = impala_launch(kernel, kAdamCluster, kAdamThreads, 0, (cudaStream_t)stream, true, params, reduced,
                                        static_cast<const ulonglong2*>(gather), seq, slot_stride, buf_stride, world,
                                        n_extra, m, v, state, n_policy, n_total, max_norm, lr_table, n_lr, h0, h1, eps,
                                        norms_out, err, timeout_ns_of(timeout_s));
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

extern "C" int impala_clip_optim_popart(float* params, const double* grad, float* m, float* v, int64_t* state,
                                        int64_t n_policy, int64_t n_total, float max_norm, const float* lr_table,
                                        int64_t n_lr, int rule, float h0, float h1, float eps, double* norms_out,
                                        double* popart, int64_t sums_at, int64_t w2_off, int64_t w2_len,
                                        int64_t b2_off, float beta, void* stream) {
    if (!params || !grad || !m || !v || !state) return IMPALA_ERR_BAD_ARG;
    if (n_total < 1 || n_policy < 0 || n_policy > n_total) return IMPALA_ERR_BAD_ARG;
    if (bad_optim_args(lr_table, n_lr, rule, h0, h1, eps)) return IMPALA_ERR_BAD_ARG;
    if (bad_popart_args(popart, n_policy, n_total, w2_off, w2_len, b2_off, beta) || sums_at < n_total)
        return IMPALA_ERR_BAD_ARG;
    const Popart pop{popart, sums_at, w2_off, w2_len, b2_off, beta};
    const auto kernel =
        rule == IMPALA_OPT_ADAM ? clip_optim_popart_kernel<AdamRule> : clip_optim_popart_kernel<RmspropRule>;
    const cudaError_t e = impala_launch(kernel, kAdamCluster, kAdamThreads, 0, (cudaStream_t)stream, true, params, grad,
                                        m, v, state, n_policy, n_total, max_norm, lr_table, n_lr, h0, h1, eps, norms_out,
                                        pop);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

extern "C" int impala_gather_clip_optim_popart(float* params, double* reduced, const void* gather, long long* seq,
                                               int64_t slot_stride, int64_t buf_stride, int world, int n_extra,
                                               float* m, float* v, int64_t* state, int64_t n_policy, int64_t n_total,
                                               float max_norm, const float* lr_table, int64_t n_lr, int rule, float h0,
                                               float h1, float eps, double* norms_out, int* err, double timeout_s,
                                               double* popart, int64_t sums_at, int64_t w2_off, int64_t w2_len,
                                               int64_t b2_off, float beta, void* stream) {
    if (bad_gather_args(params, reduced, gather, seq, slot_stride, buf_stride, world, n_extra, m, v, state, n_policy,
                        n_total))
        return IMPALA_ERR_BAD_ARG;
    if (bad_optim_args(lr_table, n_lr, rule, h0, h1, eps)) return IMPALA_ERR_BAD_ARG;
    // the eight sums must be among the gathered extras
    if (bad_popart_args(popart, n_policy, n_total, w2_off, w2_len, b2_off, beta) || sums_at < n_total ||
        sums_at + 8 > n_total + n_extra)
        return IMPALA_ERR_BAD_ARG;
    const Popart pop{popart, sums_at, w2_off, w2_len, b2_off, beta};
    const auto kernel = rule == IMPALA_OPT_ADAM ? gather_clip_optim_popart_kernel<AdamRule>
                                                : gather_clip_optim_popart_kernel<RmspropRule>;
    const cudaError_t e = impala_launch(kernel, kAdamCluster, kAdamThreads, 0, (cudaStream_t)stream, true, params, reduced,
                                        static_cast<const ulonglong2*>(gather), seq, slot_stride, buf_stride, world,
                                        n_extra, m, v, state, n_policy, n_total, max_norm, lr_table, n_lr, h0, h1, eps,
                                        norms_out, err, timeout_ns_of(timeout_s), pop);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}
