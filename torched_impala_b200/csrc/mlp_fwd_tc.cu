// MLP forward on the Hopper tensor cores (wgmma, fp32 accumulators in registers), error-compensated
// 3xTF32.
//
//   out[m,:] = relu(x[m,:] W1^T + b1) W2^T + b2          (models.py:23-25 / :51-52, eval mode)
//
// Layer 1 is the GEMM: per 64-row tile  D[64, HB] = X[64, K] * W1_blk[HB, K]^T  with K = the
// observation width padded to 32 (one 128-byte swizzle atom, narrow kernels) or 64 (two atoms:
// BASELINE config c5, obs = 64).  To stay within 1e-5 of the float64 reference, every fp32 operand
// is split into a tf32 "hi" (round-to-nearest) and a "lo" remainder and three MMAs are accumulated
// per K step: lo*hi + hi*lo first, hi*hi last (the dropped lo*lo term is ~2^-22 relative; the
// small terms go first so that only the last additions into the accumulator are full-magnitude).
//
// The accumulator of a 32-unit slice of the hidden layer is 16 registers per thread, so the CUDA
// cores see each hidden activation exactly once, in the registers wgmma left it in: bias, ReLU and
// the tiny second layer (<= 4 outputs) run on the thread's two rows and eight columns, and the four
// threads of a quad that share a row combine their partial sums with two shuffles (fixed order).
//
// One CTA = kWG independent warpgroups, each owning its own 64-row tiles and x stage; the weights
// W1 hi / lo of up to 256 hidden units (a "block") sit in shared memory and are shared.  While one
// warpgroup runs its epilogue the other's MMAs keep the tensor cores busy, and every warpgroup has
// the next tile's x rows in flight in registers while it computes the current one.  Wider hidden
// layers walk their blocks in passes: out[row] = ((b2 + z_0) + z_1) + ...  where the thread that
// owns a row adds the block's partial second-layer sum to what the SAME thread wrote in the
// previous pass (fixed order, bitwise reproducible, no workspace).
#include <map>
#include <mutex>
#include <tuple>

#include "mlp_kernels.cuh"
#include "tc_common.cuh"

namespace {

constexpr int kTileM = 64;                 // rows per tile (wgmma M)
constexpr int kWG = 2;                      // warpgroups per CTA
constexpr int kThreads = kWG * 128;
constexpr int kXAtomBytes = kTileM * 128;   // 8 KiB: 64 rows x 32 floats

struct FwdTcArgs {
    const float* x;
    const float* params;
    float* out;
    int M, O, H, N2, num_tiles;
    int hb;  // hidden units per pass (multiple of 32, <= 256, divides H)
    MlpLayout lay;
};

__host__ __device__ constexpr size_t fwd_smem_bytes(int hb, int ka, int np) {
    return 1024 /*alignment slack*/ + (size_t)2 * ka * hb * 128 + (size_t)kWG * 2 * ka * kXAtomBytes +
           (size_t)hb * (np + 1) * sizeof(float);
}

// One CTA's share of a network: CTA `cta` of `ncta`; warpgroup w takes tiles u, u + ncta * kWG, ...
// with u = cta * kWG + w (a launch may give different CTA ranges to different networks).
template <int NP, int KA>
__device__ __forceinline__ void fwd_tc_body(const FwdTcArgs& a, const int cta, const int ncta) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment (SWIZZLE_128B atoms) by OFFSETTING the __shared__ array
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const int HB = a.hb;
    uint8_t* w_hi = smem;                          // [KA atoms][HB rows][128 B]
    uint8_t* w_lo = w_hi + KA * HB * 128;
    const int tid = threadIdx.x, wg = tid >> 7, lt = tid & 127, warp = lt >> 5, lane = tid & 31;
    uint8_t* x_hi = w_lo + KA * HB * 128 + wg * 2 * KA * kXAtomBytes;  // this warpgroup's [KA][64 rows][128 B]
    uint8_t* x_lo = x_hi + KA * kXAtomBytes;
    float* b1s = reinterpret_cast<float*>(smem + 2 * KA * HB * 128 + kWG * 2 * KA * kXAtomBytes);  // [HB]
    float* w2s = b1s + HB;                                                                         // [HB][NP]

    const int O = a.O, ochunks = O >> 2, ksteps = (O + 7) >> 3;
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;
    const float* __restrict__ b2 = a.params + a.lay.ob2;
    const int unit = cta * kWG + wg, nunits = ncta * kWG;
    const int g = lane >> 2, q = lane & 3;

    // x rows of a tile -> registers: chunk idx = lt + 128 k is (row idx / (8 KA), 16-byte chunk idx % (8 KA))
    constexpr int kLd = 4 * KA;
    float4 v[kLd];
    auto load = [&](int tile) {
#pragma unroll
        for (int k = 0; k < kLd; ++k) {
            const int idx = lt + 128 * k, r = idx / (8 * KA), c = idx % (8 * KA);
            const int row = tile * kTileM + r;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tile < a.num_tiles && row < a.M && c < ochunks)
                v[k] = __ldg(reinterpret_cast<const float4*>(a.x + (size_t)row * O) + c);
        }
    };

    const int npass = a.H / HB;
    for (int p = 0; p < npass; ++p) {
        // ---- stage this block's W1 rows (hi / lo swizzled tiles), b1 and W2 (transposed)
        __syncthreads();  // the previous pass is done with the weights
        for (int idx = tid; idx < HB * 8 * KA; idx += kThreads) {
            const int r = idx / (8 * KA), c = idx % (8 * KA);
            float4 w = make_float4(0.f, 0.f, 0.f, 0.f), hi, lo;
            if (c < ochunks) w = __ldg(reinterpret_cast<const float4*>(W1 + (size_t)(p * HB + r) * O) + c);
            tc::split4(w, hi, lo);
            const uint32_t off = (c >> 3) * (HB * 128) + tc::sw128_offset(r, c & 7);
            *reinterpret_cast<float4*>(w_hi + off) = hi;
            *reinterpret_cast<float4*>(w_lo + off) = lo;
        }
        for (int idx = tid; idx < HB; idx += kThreads) b1s[idx] = __ldg(b1 + p * HB + idx);
        for (int idx = tid; idx < HB * NP; idx += kThreads) {
            const int j = idx / NP, n = idx - j * NP;
            w2s[idx] = n < a.N2 ? __ldg(W2 + (size_t)n * a.H + p * HB + j) : 0.f;
        }
        tc::fence_proxy_async();
        __syncthreads();

        load(unit);
        for (int tile = unit; tile < a.num_tiles; tile += nunits) {
            // ---- x tile -> hi / lo swizzled tiles (the warpgroup's previous MMAs have all retired)
            tc::named_bar(1 + wg, 128);
#pragma unroll
            for (int k = 0; k < kLd; ++k) {
                const int idx = lt + 128 * k, r = idx / (8 * KA), c = idx % (8 * KA);
                float4 hi, lo;
                tc::split4(v[k], hi, lo);
                const uint32_t off = (c >> 3) * kXAtomBytes + tc::sw128_offset(r, c & 7);
                *reinterpret_cast<float4*>(x_hi + off) = hi;
                *reinterpret_cast<float4*>(x_lo + off) = lo;
            }
            tc::fence_proxy_async();
            tc::named_bar(1 + wg, 128);
            load(tile + nunits);  // in flight during this tile's MMAs and epilogue

            float p0[NP], p1[NP];  // partial second-layer sums of rows 16 warp + g and + 8
#pragma unroll
            for (int n = 0; n < NP; ++n) p0[n] = 0.f, p1[n] = 0.f;
            for (int nc = 0; nc < HB / 32; ++nc) {
                float d[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) d[i] = 0.f;
                tc::fence_acc(d);  // zeroed before the warpgroup fence (see mlp_bwd_tc.cu)
                tc::wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t xo = (kk >> 2) * kXAtomBytes + (kk & 3) * 32;
                        const uint32_t wo = (kk >> 2) * (HB * 128) + nc * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d, tc::smem_desc_k_sw128(x_lo, xo), tc::smem_desc_k_sw128(w_hi, wo), kk > 0);
                        tc::wgmma_n32_ss(d, tc::smem_desc_k_sw128(x_hi, xo), tc::smem_desc_k_sw128(w_lo, wo), true);
                    }
                }
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t xo = (kk >> 2) * kXAtomBytes + (kk & 3) * 32;
                        const uint32_t wo = (kk >> 2) * (HB * 128) + nc * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d, tc::smem_desc_k_sw128(x_hi, xo), tc::smem_desc_k_sw128(w_hi, wo), true);
                    }
                }
                tc::wgmma_commit();
                tc::wgmma_wait<0>();
                tc::fence_acc(d);
                // ---- epilogue of the slice: bias, ReLU, second layer (this thread's 2 rows x 8 units)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int j = nc * 32 + 8 * i + 2 * q + e;
                        const float bj = b1s[j];
                        const float h0 = fmaxf(d[4 * i + e] + bj, 0.f);
                        const float h1 = fmaxf(d[4 * i + 2 + e] + bj, 0.f);
                        if constexpr (NP == 4) {
                            const float4 w = *reinterpret_cast<const float4*>(w2s + 4 * j);
                            p0[0] = fmaf(h0, w.x, p0[0]), p0[1] = fmaf(h0, w.y, p0[1]);
                            p0[2] = fmaf(h0, w.z, p0[2]), p0[3] = fmaf(h0, w.w, p0[3]);
                            p1[0] = fmaf(h1, w.x, p1[0]), p1[1] = fmaf(h1, w.y, p1[1]);
                            p1[2] = fmaf(h1, w.z, p1[2]), p1[3] = fmaf(h1, w.w, p1[3]);
                        } else {
                            const float w = w2s[j];
                            p0[0] = fmaf(h0, w, p0[0]), p1[0] = fmaf(h1, w, p1[0]);
                        }
                    }
                }
            }
            // the quad's four column sets meet (fixed order), lane q == 0 writes the two rows
#pragma unroll
            for (int n = 0; n < NP; ++n) {
                p0[n] += __shfl_xor_sync(IMPALA_FULL_MASK, p0[n], 1);
                p1[n] += __shfl_xor_sync(IMPALA_FULL_MASK, p1[n], 1);
                p0[n] += __shfl_xor_sync(IMPALA_FULL_MASK, p0[n], 2);
                p1[n] += __shfl_xor_sync(IMPALA_FULL_MASK, p1[n], 2);
            }
            if (q == 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = tile * kTileM + 16 * warp + g + 8 * h;
                    if (row < a.M) {
                        float* o = a.out + (size_t)row * a.N2;
#pragma unroll
                        for (int n = 0; n < NP; ++n)
                            if (n < a.N2) o[n] = (p == 0 ? __ldg(b2 + n) : o[n]) + (h ? p1[n] : p0[n]);
                    }
                }
            }
        }
    }
}

template <int NP, int KA>
__global__ void __launch_bounds__(kThreads) mlp_fwd_tc_kernel(const __grid_constant__ FwdTcArgs a) {
    fwd_tc_body<NP, KA>(a, blockIdx.x, gridDim.x);
}

// Policy and value network of one learner step in ONE launch: CTAs [0, n_pi) run the policy
// tiles, the rest the value-function tiles.  Both read the same observations; one launch means
// one weight staging per CTA and a finer tile quantisation than two launches.
__global__ void __launch_bounds__(kThreads)
mlp_fwd_tc_pair_kernel(const __grid_constant__ FwdTcArgs a_pi, const __grid_constant__ FwdTcArgs a_vf,
                       const int n_pi) {
    if ((int)blockIdx.x < n_pi) fwd_tc_body<4, 1>(a_pi, blockIdx.x, n_pi);
    else fwd_tc_body<1, 1>(a_vf, (int)blockIdx.x - n_pi, (int)gridDim.x - n_pi);
}

FwdTcArgs make_fwd_args(const float* x, const float* params, float* out, int M, int O, int H, int N2) {
    FwdTcArgs a{};
    a.x = x, a.params = params, a.out = out;
    a.M = M, a.O = O, a.H = H, a.N2 = N2;
    a.num_tiles = (M + kTileM - 1) / kTileM;
    a.hb = H <= 256 ? H : (H % 256 == 0 ? 256 : 128);
    a.lay = impala_make_layout(O, H, N2);
    return a;
}

// Resident CTAs per SM of `kernel` at `smem` bytes (dynamic shared memory opted in on first use;
// the attribute is only ever raised) times the SM count.
template <typename K>
int resident_grid(K kernel, size_t smem, int* grid) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> opted;          // (kernel, dev) -> smem opted in
    static std::map<std::tuple<const void*, int, size_t>, int> cached;  // (kernel, dev, smem) -> grid
    int dev = 0, sms = 0;
    cudaError_t e;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess) return (int)e;
    std::lock_guard<std::mutex> lock(mu);
    const auto key = std::make_tuple((const void*)kernel, dev, smem);
    auto it = cached.find(key);
    if (it != cached.end()) return *grid = it->second, IMPALA_OK;
    size_t& o = opted[std::make_pair((const void*)kernel, dev)];
    if (smem > o) {
        if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return (int)e;
        o = smem;
    }
    int per_sm = 0;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem)) != cudaSuccess) return (int)e;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    if (per_sm < 1) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    *grid = cached[key] = per_sm * sms;
    return IMPALA_OK;
}

template <int NP, int KA>
int launch_fwd(const FwdTcArgs& a, cudaStream_t st) {
    const size_t smem = fwd_smem_bytes(a.hb, KA, NP);
    int grid = 0;
    const int rc = resident_grid(mlp_fwd_tc_kernel<NP, KA>, smem, &grid);
    if (rc != IMPALA_OK) return rc;
    const int want = (a.num_tiles + kWG - 1) / kWG;
    mlp_fwd_tc_kernel<NP, KA><<<want < grid ? want : grid, kThreads, smem, st>>>(a);
    return impala_launch_status();
}

}  // namespace

// Shapes the narrow tensor-core path covers (one K atom, the whole hidden layer in one pass).
bool impala_mlp_fwd_tc_eligible(const float* x, int M, int O, int H, int N2) {
    return M >= 1 && O >= 4 && O <= 28 && (O & 3) == 0 && H >= 16 && H <= 256 && (H & 31) == 0 &&
           N2 >= 1 && N2 <= 4 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
}

int impala_mlp_fwd_tc(const float* x, const float* params, float* out, int M, int O, int H, int N2,
                      cudaStream_t st) {
    const FwdTcArgs a = make_fwd_args(x, params, out, M, O, H, N2);
    return N2 == 1 ? launch_fwd<1, 1>(a, st) : launch_fwd<4, 1>(a, st);
}

// Both networks in one launch (policy: 2..4 outputs, value fn: 1 output); the caller has checked
// impala_mlp_fwd_tc_eligible for each.  Per-tile cost weights (policy epilogue does 4 FMA per
// hidden unit, the value fn 1) split the CTAs between the two tile lists.
int impala_mlp_fwd_tc_pair(const float* x, const float* params_pi, const float* params_vf, float* logits,
                           float* values, int M_pi, int M_vf, int O, int H_pi, int H_vf, int A,
                           cudaStream_t st) {
    const FwdTcArgs a_pi = make_fwd_args(x, params_pi, logits, M_pi, O, H_pi, A);
    const FwdTcArgs a_vf = make_fwd_args(x, params_vf, values, M_vf, O, H_vf, 1);
    const size_t s_pi = fwd_smem_bytes(a_pi.hb, 1, 4), s_vf = fwd_smem_bytes(a_vf.hb, 1, 1);
    const size_t smem = s_pi > s_vf ? s_pi : s_vf;
    int grid = 0;
    const int rc = resident_grid(mlp_fwd_tc_pair_kernel, smem, &grid);
    if (rc != IMPALA_OK) return rc;
    const int units_pi = (a_pi.num_tiles + kWG - 1) / kWG, units_vf = (a_vf.num_tiles + kWG - 1) / kWG;
    if (grid > units_pi + units_vf) grid = units_pi + units_vf;
    const int n_pi = impala_pair_split(units_pi, units_vf, grid,
                                       impala_env_int("IMPALA_PAIR_W_FWD", 160) * (H_pi / 32),
                                       100 * (H_vf / 32));
    mlp_fwd_tc_pair_kernel<<<grid, kThreads, smem, st>>>(a_pi, a_vf, n_pi);
    return impala_launch_status();
}

// Wide shapes (observation width up to 64 = two K atoms, hidden layers a multiple of 128 of any
// size, walked in passes): BASELINE config c5 (obs = 64, hidden = 512).  IMPALA_MLP_TCW=0 disables.
bool impala_mlp_tcw_eligible(const float* x, int M, int O, int H, int N2) {
    return M >= 1 && O >= 4 && O <= 64 && (O & 3) == 0 && H >= 128 && H % 128 == 0 && H <= 4096 && N2 >= 1 &&
           N2 <= 4 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && impala_env_int("IMPALA_MLP_TCW", 1) != 0;
}

int impala_mlp_fwd_tcw(const float* x, const float* params, float* out, int M, int O, int H, int N2,
                       cudaStream_t st) {
    const FwdTcArgs a = make_fwd_args(x, params, out, M, O, H, N2);
    if (O <= 32) return N2 == 1 ? launch_fwd<1, 1>(a, st) : launch_fwd<4, 1>(a, st);
    return N2 == 1 ? launch_fwd<1, 2>(a, st) : launch_fwd<4, 2>(a, st);
}
