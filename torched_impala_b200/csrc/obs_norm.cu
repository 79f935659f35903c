// Observation normalization: running per-feature statistics of the raw observations.  The step's first launch
// (impala_obs_normalize) writes the normalized float32 rows every later kernel reads and the batch's sums; one
// launch after the optimizer (impala_obs_norm_update) merges the rank-summed sums into the running statistics and
// writes the parameter block folded into raw-observation coordinates, which is what gets published.
//
// Both reductions are deterministic: fixed summation orders, integer counters only (see impala_b200.h).
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kTileF = 32;     // features per normalize CTA (one per lane)
constexpr int kLanesR = 8;     // row lanes per normalize CTA (one per warp)
constexpr int kMaxChunks = 1024;
constexpr int kUpdThreads = 256;

// Row chunks of the normalize grid: a function of the row count only, so the summation order is too.
struct Chunks {
    int64_t rows_per, n;
};
Chunks chunks_of(int64_t rows) {
    int64_t n = std::min<int64_t>(kMaxChunks, std::max<int64_t>(1, (rows + 63) / 64));
    const int64_t per = impala_round_up((rows + n - 1) / n, kLanesR);
    return {per, (rows + per - 1) / per};
}
int64_t ctl_bytes(int O) { return impala_round_up((int64_t)((O + kTileF - 1) / kTileF) * 4, 256); }

struct NormArgs {
    const void* obs;
    const int32_t* lens;
    const float* norm;  // [mu_f (O) | r_f (O)]
    float* out;         // (T+1, B, O)
    double* sums;       // [sum x (O) | sum x^2 (O) | valid rows]
    double* partial;    // (chunks, 2 O)
    unsigned* ctl;      // one zeroed counter per feature tile, left zeroed
    int64_t rows, rows_per_chunk, n_chunks;
    int T, B, F, k, O;
};

template <typename In>
__global__ void __launch_bounds__(kTileF * kLanesR) obs_normalize_kernel(const __grid_constant__ NormArgs a) {
    __shared__ double s1_sh[kLanesR][kTileF], s2_sh[kLanesR][kTileF];
    __shared__ int last_sh, count_sh;
    const int tx = threadIdx.x % kTileF, ty = threadIdx.x / kTileF;
    const int o = blockIdx.x * kTileF + tx, O = a.O;
    const bool on = o < O;
    const int j = on ? o / a.F : 0, f = on ? o - j * a.F : 0;
    // element o of dense row r lives at r F + col (frames: frame slot j of row r is frame row r + j B)
    const int64_t col = (int64_t)j * a.B * a.F + f;
    const float mu = on ? a.norm[o] : 0.f, rs = on ? a.norm[O + o] : 0.f;
    const In* __restrict__ in = static_cast<const In*>(a.obs);
    const int32_t* __restrict__ lens = a.lens;
    float* __restrict__ out = a.out;
    const int64_t c = blockIdx.y, r0 = c * a.rows_per_chunk, r1 = min(r0 + a.rows_per_chunk, a.rows);
    double s1 = 0.0, s2 = 0.0;
    if (on) {
        // kBatch rows per lane in flight: every load of the batch is issued before the first store
        constexpr int kBatch = 8;
        for (int64_t rb = r0 + ty; rb < r1; rb += kBatch * kLanesR) {
            float x[kBatch];
            bool valid[kBatch];
#pragma unroll
            for (int q = 0; q < kBatch; ++q) {
                const int64_t r = rb + q * kLanesR;
                const int t = (int)((unsigned)r / (unsigned)a.B);  // rows < 2^32
                x[q] = r < r1 ? (float)__ldg(in + r * a.F + col) : 0.f;
                valid[q] = r < r1 && t < a.T && t < __ldg(lens + (r - (int64_t)t * a.B));
            }
#pragma unroll
            for (int q = 0; q < kBatch; ++q) {
                const int64_t r = rb + q * kLanesR;
                if (r < r1) out[r * O + o] = __fmul_rn(__fsub_rn(x[q], mu), rs);
                if (valid[q]) {  // rows in order: the same additions as one row at a time
                    const double xd = (double)x[q];
                    s1 = __dadd_rn(s1, xd);
                    s2 = __dadd_rn(s2, __dmul_rn(xd, xd));
                }
            }
        }
    }
    s1_sh[ty][tx] = s1, s2_sh[ty][tx] = s2;
    __syncthreads();
    if (ty == 0 && on) {  // the chunk's partial: row lanes added in order
        double p1 = s1_sh[0][tx], p2 = s2_sh[0][tx];
#pragma unroll
        for (int l = 1; l < kLanesR; ++l) p1 = __dadd_rn(p1, s1_sh[l][tx]), p2 = __dadd_rn(p2, s2_sh[l][tx]);
        a.partial[c * 2 * O + o] = p1;
        a.partial[c * 2 * O + O + o] = p2;
    }
    // the last CTA of this feature tile adds the chunks' partials (lane g: chunks g, g + 8, .. in order, then the
    // lanes in order); the arrival order decides who adds, never the order of the additions
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last_sh = atomicAdd(&a.ctl[blockIdx.x], 1u) == gridDim.y - 1, count_sh = 0;
    __syncthreads();
    if (!last_sh) return;
    __threadfence();
    double q1 = 0.0, q2 = 0.0;
    if (on) {
        for (int64_t cc = ty; cc < a.n_chunks; cc += kLanesR) {
            q1 = __dadd_rn(q1, __ldcg(a.partial + cc * 2 * O + o));
            q2 = __dadd_rn(q2, __ldcg(a.partial + cc * 2 * O + O + o));
        }
    }
    __syncthreads();
    s1_sh[ty][tx] = q1, s2_sh[ty][tx] = q2;
    if (blockIdx.x == 0) {  // valid rows: sum_b clamp(lens[b], 0, T), integers
        int n = 0;
        for (int b = threadIdx.x; b < a.B; b += blockDim.x) n += min(max(a.lens[b], 0), a.T);
        atomicAdd(&count_sh, n);
    }
    __syncthreads();
    if (ty == 0 && on) {
        double t1 = s1_sh[0][tx], t2 = s2_sh[0][tx];
#pragma unroll
        for (int l = 1; l < kLanesR; ++l) t1 = __dadd_rn(t1, s1_sh[l][tx]), t2 = __dadd_rn(t2, s2_sh[l][tx]);
        a.sums[o] = t1;
        a.sums[O + o] = t2;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.sums[2 * O] = (double)count_sh;
    if (threadIdx.x == 0) a.ctl[blockIdx.x] = 0u;  // every CTA of the tile has arrived: ready for the next launch
}

struct UpdArgs {
    double* stats;       // [count | mean (O) | var (O)]
    float* norm;         // [mu_f (O) | r_f (O)]
    const double* sums;  // [sum x (O) | sum x^2 (O) | rows], summed over the ranks (gather == nullptr)
    double eps;
    const float* params;
    float* folded;
    int64_t n_total;
    int64_t w1[2], b1[2];
    int H[2];
    int O;
    unsigned* ctl;
    // peer route: every rank's sums in this rank's gather buffer, added here in rank order
    const ulonglong2* gather;
    const long long* seq;
    int64_t slot_stride, buf_stride, sums_at;
    int world;
    int* err;
    unsigned long long timeout_ns;
};

__device__ __forceinline__ unsigned long long now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// Entry i of the rank-summed sums: read locally, or added over the ranks' gather slots in rank order.
__device__ __forceinline__ double summed(const UpdArgs& a, int i, unsigned step, bool& ok) {
    if (!a.gather) return a.sums[i];
    const ulonglong2* gb = a.gather + (int64_t)(step & 1) * a.buf_stride + a.sums_at + i;
    const unsigned long long t0 = now_ns();
    double s = 0.0;
    for (int r = 0; r < a.world; ++r) {
        ulonglong2 w = ll_load(gb + (int64_t)r * a.slot_stride);
        unsigned spins = 0;
        while (!ll_ready(w, step)) {
            if ((++spins & 255u) == 0 && now_ns() - t0 > a.timeout_ns) {
                ok = false;
                return 0.0;
            }
            if (spins > 16) __nanosleep(20);
            w = ll_load(gb + (int64_t)r * a.slot_stride);
        }
        s = __dadd_rn(s, ll_value(w));
    }
    return s;
}

// Chan's merge of a batch (n_b rows, sums s1, s2) into (n_a, mean, var) in float64; n_b = 0 keeps them.
struct Merged {
    double count, mean, var;
};
__device__ __forceinline__ Merged chan_merge(double n_a, double mean_a, double var_a, double n_b, double s1,
                                             double s2) {
    if (!(n_b > 0.0)) return {n_a, mean_a, var_a};
    const double n = __dadd_rn(n_a, n_b);
    const double mean_b = __ddiv_rn(s1, n_b);
    const double m2_b = fmax(__dadd_rn(s2, -__dmul_rn(s1, mean_b)), 0.0);
    const double delta = __dadd_rn(mean_b, -mean_a);
    const double mean = __dadd_rn(mean_a, __dmul_rn(delta, __ddiv_rn(n_b, n)));
    const double m2 = __dadd_rn(__dadd_rn(__dmul_rn(var_a, n_a), m2_b),
                                __dmul_rn(__dmul_rn(delta, delta), __ddiv_rn(__dmul_rn(n_a, n_b), n)));
    return {n, mean, __ddiv_rn(m2, n)};
}

__global__ void __launch_bounds__(kUpdThreads) obs_norm_update_kernel(const __grid_constant__ UpdArgs a) {
    extern __shared__ float s_norm[];  // the new [mu_f | r_f]
    __shared__ int skip_sh, last_sh, fail_sh;
    const int O = a.O, tid = threadIdx.x;
    const unsigned step = a.gather ? (unsigned)*a.seq : 0u;
    if (tid == 0) skip_sh = a.err && *a.err, fail_sh = 0;
    __syncthreads();
    if (skip_sh) return;  // the optimizer gave up waiting for a peer: nothing moves
    // every CTA forms the new statistics of every feature (the same bits in each); the stored ones change last
    bool ok = true;
    const double n_b = summed(a, 2 * O, step, ok), n_a = a.stats[0];
    for (int o = tid; o < O; o += blockDim.x) {
        const Merged m = chan_merge(n_a, a.stats[1 + o], a.stats[1 + O + o], n_b, summed(a, o, step, ok),
                                    summed(a, O + o, step, ok));
        s_norm[o] = (float)m.mean;
        s_norm[O + o] = (float)__drcp_rn(__dsqrt_rn(__dadd_rn(m.var, a.eps)));
    }
    if (!ok) fail_sh = 1;
    __syncthreads();
    const float* mu_f = s_norm;
    const float* r_f = s_norm + O;
    // a CTA that gave up waiting for a peer writes nothing, but still arrives at the counter below
    if (fail_sh) {
        if (tid == 0) atomicOr(a.ctl + 1, 1u);
    } else {
        // the folded block: W1' = W1 diag(r_f), b1' = b1 - W1' mu_f (float64 sum), everything else copied
        const int64_t stride = (int64_t)gridDim.x * blockDim.x;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + tid; i < a.n_total; i += stride) {
            float v = a.params[i];
            bool b1 = false;
    #pragma unroll
            for (int g = 0; g < 2; ++g) {
                if (i >= a.w1[g] && i < a.w1[g] + (int64_t)a.H[g] * O) v = __fmul_rn(v, r_f[(i - a.w1[g]) % O]);
                b1 |= i >= a.b1[g] && i < a.b1[g] + a.H[g];
            }
            if (!b1) a.folded[i] = v;
        }
        const int lane = tid & 31, warps = (int)(gridDim.x * blockDim.x / 32);
        for (int w = (int)((blockIdx.x * blockDim.x + tid) / 32); w < a.H[0] + a.H[1]; w += warps) {
            const int g = w < a.H[0] ? 0 : 1, h = g ? w - a.H[0] : w;
            const float* row = a.params + a.w1[g] + (int64_t)h * O;
            double s = 0.0;
            for (int o = lane; o < O; o += 32) s = __dadd_rn(s, __dmul_rn((double)__fmul_rn(row[o], r_f[o]), (double)mu_f[o]));
            s = warp_sum_f64(s);
            if (lane == 0) a.folded[a.b1[g] + h] = (float)__dadd_rn((double)a.params[a.b1[g] + h], -s);
        }
    }
    // the last CTA to arrive stores the statistics (every CTA has read the old ones by then) and re-arms the
    // counters; if any CTA timed out it raises *err instead, and the statistics stay as they were
    __threadfence();
    __syncthreads();
    if (tid == 0) last_sh = atomicAdd(a.ctl, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last_sh) return;
    __threadfence();
    if (tid == 0) skip_sh = __ldcg(a.ctl + 1) != 0u;
    __syncthreads();
    if (skip_sh) {
        if (tid == 0) {
            if (a.err) *a.err = 1;
            a.ctl[0] = a.ctl[1] = 0u;
        }
        return;
    }
    for (int o = tid; o < O; o += blockDim.x) {
        const Merged m = chan_merge(n_a, a.stats[1 + o], a.stats[1 + O + o], n_b, summed(a, o, step, ok),
                                    summed(a, O + o, step, ok));
        a.stats[1 + o] = m.mean;
        a.stats[1 + O + o] = m.var;
        a.norm[o] = mu_f[o];
        a.norm[O + o] = r_f[o];
    }
    __syncthreads();
    if (tid == 0) {
        if (n_b > 0.0) a.stats[0] = __dadd_rn(n_a, n_b);
        a.ctl[0] = 0u;
    }
}

}  // namespace

extern "C" int64_t impala_obs_normalize_workspace(int T, int B, int O) {
    if (T < 1 || B < 1 || O < 1 || O > IMPALA_OBS_NORM_MAX_FEATURES) return IMPALA_ERR_BAD_ARG;
    const Chunks ch = chunks_of((int64_t)(T + 1) * B);
    return ctl_bytes(O) + ch.n * 2 * O * (int64_t)sizeof(double);
}

extern "C" int impala_obs_normalize(const void* obs, int in_dtype, int T, int B, int F, int k, const int32_t* lens,
                                    const float* norm, float* out, double* sums, void* workspace,
                                    int64_t workspace_bytes, void* stream) {
    if (!obs || !lens || !norm || !out || !sums || !workspace) return IMPALA_ERR_BAD_ARG;
    if (T < 1 || B < 1 || F < 1 || k < 1 || (in_dtype != IMPALA_OBS_F32 && in_dtype != IMPALA_OBS_U8))
        return IMPALA_ERR_BAD_ARG;
    const int64_t O = (int64_t)F * k;
    if (O > IMPALA_OBS_NORM_MAX_FEATURES) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    const int64_t need = impala_obs_normalize_workspace(T, B, (int)O);
    if (workspace_bytes < need) return IMPALA_ERR_WORKSPACE_TOO_SMALL;
    const Chunks ch = chunks_of((int64_t)(T + 1) * B);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    const NormArgs a{obs, lens, norm, out, sums, reinterpret_cast<double*>(ws + ctl_bytes((int)O)),
                     reinterpret_cast<unsigned*>(ws), (int64_t)(T + 1) * B, ch.rows_per, ch.n, T, B, F, k, (int)O};
    const dim3 grid((unsigned)((O + kTileF - 1) / kTileF), (unsigned)ch.n);
    const cudaError_t e = in_dtype == IMPALA_OBS_U8
        ? impala_launch(obs_normalize_kernel<uint8_t>, grid, kTileF * kLanesR, 0, (cudaStream_t)stream, false, a)
        : impala_launch(obs_normalize_kernel<float>, grid, kTileF * kLanesR, 0, (cudaStream_t)stream, false, a);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

extern "C" int impala_obs_norm_update(double* stats, float* norm, const double* sums, double eps, const float* params,
                                      float* folded, int64_t n_total, int O, int64_t w1_off0, int64_t b1_off0, int H0,
                                      int64_t w1_off1, int64_t b1_off1, int H1, unsigned* ctl, const void* gather,
                                      const long long* seq, int64_t slot_stride, int64_t buf_stride, int world,
                                      int64_t sums_at, int* err, double timeout_s, void* stream) {
    if (!stats || !norm || !params || !folded || !ctl || (!gather && !sums)) return IMPALA_ERR_BAD_ARG;
    if (O < 1 || O > IMPALA_OBS_NORM_MAX_FEATURES || !(eps > 0.0) || !(eps < 1e300) || n_total < 1) return IMPALA_ERR_BAD_ARG;
    if (H0 < 1 || H1 < 0 || w1_off0 < 0 || b1_off0 < 0 || w1_off0 + (int64_t)H0 * O > n_total || b1_off0 + H0 > n_total)
        return IMPALA_ERR_BAD_ARG;
    if (H1 > 0 && (w1_off1 < 0 || b1_off1 < 0 || w1_off1 + (int64_t)H1 * O > n_total || b1_off1 + H1 > n_total))
        return IMPALA_ERR_BAD_ARG;
    if (gather && (!seq || world < 1 || world > 8 || sums_at < 0 || slot_stride < sums_at + 2 * O + 1 ||
                   buf_stride < (int64_t)world * slot_stride || (reinterpret_cast<uintptr_t>(gather) & 15) != 0))
        return IMPALA_ERR_BAD_ARG;
    UpdArgs a{};
    a.stats = stats, a.norm = norm, a.sums = sums, a.eps = eps, a.params = params, a.folded = folded;
    a.n_total = n_total, a.O = O, a.ctl = ctl;
    a.w1[0] = w1_off0, a.b1[0] = b1_off0, a.H[0] = H0;
    a.w1[1] = H1 > 0 ? w1_off1 : 0, a.b1[1] = H1 > 0 ? b1_off1 : 0, a.H[1] = H1;
    a.gather = static_cast<const ulonglong2*>(gather), a.seq = seq, a.slot_stride = slot_stride;
    a.buf_stride = buf_stride, a.sums_at = sums_at, a.world = world, a.err = err;
    a.timeout_ns = timeout_s > 0 ? (unsigned long long)(timeout_s * 1e9) : 600ull * 1000000000ull;
    int sms = 0;
    if (const cudaError_t e = impala_sm_count(&sms); e != cudaSuccess) return (int)e;
    const int64_t want = std::max<int64_t>((n_total + kUpdThreads - 1) / kUpdThreads, (H0 + H1 + 7) / 8);
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, 2 * (int64_t)sms));
    const cudaError_t e = impala_launch(obs_norm_update_kernel, grid, kUpdThreads, 2 * O * sizeof(float),
                                        (cudaStream_t)stream, false, a);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}
