// MLP backward on the Hopper tensor cores (wgmma, fp32 accumulators in registers), error-compensated
// 3xTF32.
//
// Gradient of sum_m <dout[m,:], mlp(x[m,:])> w.r.t. (W1, b1, W2, b2)  (autograd at learner.py:175).
// Transposed formulation so that a thread owns HIDDEN units (accumulator rows = hidden units), per
// tile of 64 batch rows and warpgroup (64 hidden units):
//
//   GEMM1 (SS, recompute)  PRE[64 hid, 64 rows] = W1_blk[64, K] * X[64 rows, K]^T
//   CUDA cores             h = relu(PRE + b1); dh = W2^T dz; dW2 += dz h; DP = (PRE + b1 > 0) ? dh : 0;
//                          db1 += DP
//   GEMM2 (RS, reduction)  dW1_blk[64 hid, K] += DP[64 hid, 64 rows] * X[64 rows, K]
//
// K = the observation width padded to 32 (one 128-byte swizzle atom) or 64 (two atoms, BASELINE c5).
// DP never leaves the registers: the GEMM1 accumulator layout of a thread (two hidden units, 16 batch
// columns) becomes the A operand of GEMM2 directly, by reordering the batch rows INSIDE each group of
// 8 in the B operand of GEMM2 (K is a sum, so any order does, as long as A and B agree): A fragment
// column q holds batch row 2q and column q + 4 batch row 2q + 1 of the group, which is where the
// accumulator left them.  GEMM2's B operand is therefore the x tile transposed (rows = features,
// K = batch rows, K-major as tf32 requires) with that order, written by the loader beside the
// row-major tile GEMM1 reads.
//
// Operands are split into tf32 hi + lo and three products are accumulated per K step (x and W1:
// hi = round-to-nearest tf32; DP: hi = dp with the low 13 mantissa bits cleared, lo = the exact
// remainder); the small terms go into their own accumulator (dW1) or first (PRE), so that the
// full-magnitude hi*hi additions are the only ones that round at full size.  dW1 accumulates in
// registers over every tile of the persistent CTA and is written out once per pass.
//
// One CTA = 2 warpgroups = 128 hidden units per pass; wider layers are walked in passes (x is
// re-read once per pass).  Every gradient entry of W1 / b1 / W2 belongs to exactly one hidden unit,
// so each CTA writes a float32 partial gradient row (same layout as the FP32 kernels) and the rows
// are summed in float64 in a fixed order: in-kernel after a grid barrier (narrow shapes, paired
// launch, optional peer push), or by reduce_partials_kernel (wide shapes).
#include <map>
#include <mutex>
#include <tuple>

#include "mlp_kernels.cuh"
#include "tc_common.cuh"

namespace {

constexpr int kRowsT = 64;                   // batch rows per tile: N of GEMM1, K of GEMM2
constexpr int kWG = 2;                       // warpgroups per CTA, 64 hidden units each
constexpr int kThreads = kWG * 128;
constexpr int kWarps = kThreads / 32;
constexpr int kHB = 64 * kWG;                // hidden units per pass
constexpr int kXAtomBytes = kRowsT * 128;    // 8 KiB: 64 rows x 32 floats

struct BwdTcArgs {
    const float* x;
    const float* params;
    const float* dout;
    float* ws;
    double* grad;        // float64 [lay.total], written by the in-kernel reduction
    unsigned int* ctl;   // {arrivals, departures}: zero on entry, zero on exit
    int M, O, H, N2, num_tiles;
    MlpLayout lay;
};

__host__ __device__ constexpr size_t bwd_smem_bytes(int ka, int np) {
    // W1 block hi / lo [KA][128 hidden][128 B] + x hi / lo [KA][64][128 B] + x^T hi / lo
    // [2 K atoms][32 KA features][128 B] + dz [64][NP] + db2 exchange
    return 1024 + (size_t)2 * ka * kHB * 128 + (size_t)2 * ka * kXAtomBytes + (size_t)2 * 2 * 32 * ka * 128 +
           (size_t)kRowsT * np * sizeof(float) + 4 * sizeof(float);
}

// component e of a float4 (e known at compile time)
__device__ __forceinline__ float f4(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

// One persistent CTA's share of a network's backward: CTA `cta` of `ncta` takes tiles cta,
// cta + ncta, ... and leaves its float32 partial gradient in row `cta` of a.ws.  Returns a shared
// memory region of >= 16 KiB the caller may use as scratch once every thread is past it.
template <int NP, int KA>
__device__ __forceinline__ uint8_t* bwd_tc_body(const BwdTcArgs& a, const int cta, const int ncta) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr int kWBytes = KA * kHB * 128;          // one of hi / lo, [KA][128 rows][128 B]
    constexpr int kXBytes = KA * kXAtomBytes;        // one of hi / lo, [KA][64 rows][128 B]
    constexpr int kXtAtomBytes = 32 * KA * 128;      // 32 batch rows of K x 32 KA feature rows
    uint8_t* w_hi = smem;
    uint8_t* w_lo = w_hi + kWBytes;
    uint8_t* x_hi = w_lo + kWBytes;
    uint8_t* x_lo = x_hi + kXBytes;
    uint8_t* xt_hi = x_lo + kXBytes;                 // [2 K atoms][32 KA rows][128 B]
    uint8_t* xt_lo = xt_hi + 2 * kXtAtomBytes;
    float* dzs = reinterpret_cast<float*>(xt_lo + 2 * kXtAtomBytes);  // [64 rows][NP]
    float* gb2x = dzs + kRowsT * NP;                                   // [4]

    const int tid = threadIdx.x, wg = tid >> 7, lt = tid & 127, warp = lt >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int O = a.O, H = a.H, ochunks = O >> 2, ksteps = (O + 7) >> 3;
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;
    float* wsb = a.ws + (size_t)cta * a.lay.total;  // this CTA's partial gradient row

    // x rows of a tile -> registers (chunk idx = tid + kThreads k is (row idx / (8 KA), 16-byte chunk
    // idx % (8 KA))); dz row `tid` for tid < 64
    constexpr int kLd = kRowsT * 8 * KA / kThreads;
    float4 v[kLd];
    float z[NP];
    auto load = [&](int tile) {
#pragma unroll
        for (int k = 0; k < kLd; ++k) {
            const int idx = tid + kThreads * k, r = idx / (8 * KA), c = idx % (8 * KA);
            const int row = tile * kRowsT + r;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tile < a.num_tiles && row < a.M && c < ochunks)
                v[k] = __ldg(reinterpret_cast<const float4*>(a.x + (size_t)row * O) + c);
        }
        const int row = tile * kRowsT + tid;
#pragma unroll
        for (int n = 0; n < NP; ++n)
            z[n] = (tid < kRowsT && tile < a.num_tiles && row < a.M && n < a.N2) ? __ldg(a.dout + (size_t)row * a.N2 + n) : 0.f;
    };
    float gb2[NP];  // db2 = column sums of dout: this thread's rows (tid < 64), first pass only
#pragma unroll
    for (int n = 0; n < NP; ++n) gb2[n] = 0.f;

    // pads of the partial row
    {
        const int64_t lo4[4] = {a.lay.oW1 + (int64_t)H * O, a.lay.ob1 + H, a.lay.oW2 + (int64_t)a.N2 * H,
                                a.lay.ob2 + a.N2};
        const int64_t hi4[4] = {a.lay.ob1, a.lay.oW2, a.lay.ob2, a.lay.total};
        for (int sgm = 0; sgm < 4; ++sgm)
            for (int64_t p = lo4[sgm] + tid; p < hi4[sgm]; p += kThreads) wsb[p] = 0.f;
    }

    // dz of the tile is the output of the kernel before this one (PDL, common.cuh)
    pdl_wait();
    const int npass = H / kHB;
    for (int p = 0; p < npass; ++p) {
        // ---- this pass's W1 rows -> hi / lo swizzled tiles (warpgroup w: rows [64 w, 64 w + 64))
        __syncthreads();  // the previous pass is done with the weights
        for (int idx = tid; idx < kHB * 8 * KA; idx += kThreads) {
            const int r = idx / (8 * KA), c = idx % (8 * KA);
            float4 w = make_float4(0.f, 0.f, 0.f, 0.f), hi, lo;
            if (c < ochunks) w = __ldg(reinterpret_cast<const float4*>(W1 + (size_t)(p * kHB + r) * O) + c);
            tc::split4(w, hi, lo);
            const uint32_t off = (r >> 6) * (KA * 64 * 128) + (c >> 3) * (64 * 128) + tc::sw128_offset(r & 63, c & 7);
            *reinterpret_cast<float4*>(w_hi + off) = hi;
            *reinterpret_cast<float4*>(w_lo + off) = lo;
        }
        uint8_t* wa_hi = w_hi + wg * (KA * 64 * 128);  // this warpgroup's A operand of GEMM1
        uint8_t* wa_lo = w_lo + wg * (KA * 64 * 128);
        // the thread's two hidden units
        const int j0 = p * kHB + 64 * wg + 16 * warp + g, j1 = j0 + 8;
        const float bj0 = __ldg(b1 + j0), bj1 = __ldg(b1 + j1);
        float w2r0[NP], w2r1[NP], gw0[NP], gw1[NP], gb10 = 0.f, gb11 = 0.f;
#pragma unroll
        for (int n = 0; n < NP; ++n) {
            w2r0[n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + j0) : 0.f;
            w2r1[n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + j1) : 0.f;
            gw0[n] = gw1[n] = 0.f;
        }
        float acc_hh[KA][16], acc_c[KA][16];  // dW1: dp_hi * x_hi | dp_hi * x_lo + dp_lo * x_hi
#pragma unroll
        for (int fa = 0; fa < KA; ++fa)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc_hh[fa][i] = acc_c[fa][i] = 0.f;
#pragma unroll
        for (int fa = 0; fa < KA; ++fa) tc::fence_acc(acc_hh[fa]), tc::fence_acc(acc_c[fa]);

        load(cta);
        for (int tile = cta, it = 0; tile < a.num_tiles; tile += ncta, ++it) {
            // ---- stage the tile: x row-major (B of GEMM1) and transposed (B of GEMM2), hi / lo; dz
            __syncthreads();  // every MMA that read the previous tile has retired
#pragma unroll
            for (int k = 0; k < kLd; ++k) {
                const int idx = tid + kThreads * k, r = idx / (8 * KA), c = idx % (8 * KA);
                float4 hi, lo;
                tc::split4(v[k], hi, lo);
                const uint32_t off = (c >> 3) * kXAtomBytes + tc::sw128_offset(r, c & 7);
                *reinterpret_cast<float4*>(x_hi + off) = hi;
                *reinterpret_cast<float4*>(x_lo + off) = lo;
                // batch row r -> K atom r / 32, position 8 kk + (qq >> 1) + 4 (qq & 1) with r % 32 = 8 kk + qq
                const int rr = r & 31, pos = (rr & ~7) + ((rr & 7) >> 1) + 4 * (rr & 1);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int f = 4 * c + e;
                    const uint32_t toff = (r >> 5) * kXtAtomBytes + (f >> 3) * 1024 + (f & 7) * 128 +
                                          (((pos >> 2) ^ (f & 7)) << 4) + (pos & 3) * 4;
                    *reinterpret_cast<float*>(xt_hi + toff) = f4(hi, e);
                    *reinterpret_cast<float*>(xt_lo + toff) = f4(lo, e);
                }
            }
            if (tid < kRowsT) {
#pragma unroll
                for (int n = 0; n < NP; ++n) {
                    dzs[tid * NP + n] = z[n];
                    if (p == 0) gb2[n] += z[n];
                }
            }
            tc::fence_proxy_async();
            __syncthreads();
            load(tile + ncta);  // in flight during this tile's MMAs and epilogue

            // ---- GEMM1: PRE = W1_blk * X^T (two N = 32 halves of the tile's batch rows)
            float d[2][16];
#pragma unroll
            for (int nb = 0; nb < 2; ++nb)
#pragma unroll
                for (int i = 0; i < 16; ++i) d[nb][i] = 0.f;
            // the zeroed accumulators are defined HERE, before the warpgroup fence: left alone, the compiler
            // sinks the moves behind the K-step guards, past the fence, and ptxas then serializes every wgmma
            tc::fence_acc(d[0]);
            tc::fence_acc(d[1]);
            tc::wgmma_fence();
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) {
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t wo = (kk >> 2) * (64 * 128) + (kk & 3) * 32;
                        const uint32_t xo = (kk >> 2) * kXAtomBytes + nb * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d[nb], tc::smem_desc_k_sw128(wa_lo, wo), tc::smem_desc_k_sw128(x_hi, xo), kk > 0);
                        tc::wgmma_n32_ss(d[nb], tc::smem_desc_k_sw128(wa_hi, wo), tc::smem_desc_k_sw128(x_lo, xo), true);
                    }
                }
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t wo = (kk >> 2) * (64 * 128) + (kk & 3) * 32;
                        const uint32_t xo = (kk >> 2) * kXAtomBytes + nb * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d[nb], tc::smem_desc_k_sw128(wa_hi, wo), tc::smem_desc_k_sw128(x_hi, xo), true);
                    }
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
            tc::fence_acc(d[0]);
            tc::fence_acc(d[1]);

            // ---- epilogue: d <- DP in place (thread: hidden units j0 / j1, batch columns 8 i + 2 q + e)
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int m = 32 * nb + 8 * i + 2 * q + e;
                        float dz[NP];
                        if constexpr (NP == 4) {
                            const float4 t = *reinterpret_cast<const float4*>(dzs + 4 * m);
                            dz[0] = t.x, dz[1] = t.y, dz[2] = t.z, dz[3] = t.w;
                        } else {
                            dz[0] = dzs[m];
                        }
                        // relu'(0) = 0 as in torch
                        const float pre0 = d[nb][4 * i + e] + bj0, pre1 = d[nb][4 * i + 2 + e] + bj1;
                        const float h0 = fmaxf(pre0, 0.f), h1 = fmaxf(pre1, 0.f);
                        float dh0 = dz[0] * w2r0[0], dh1 = dz[0] * w2r1[0];
#pragma unroll
                        for (int n = 1; n < NP; ++n) dh0 = fmaf(dz[n], w2r0[n], dh0), dh1 = fmaf(dz[n], w2r1[n], dh1);
#pragma unroll
                        for (int n = 0; n < NP; ++n) gw0[n] = fmaf(dz[n], h0, gw0[n]), gw1[n] = fmaf(dz[n], h1, gw1[n]);
                        const float dp0 = pre0 > 0.f ? dh0 : 0.f, dp1 = pre1 > 0.f ? dh1 : 0.f;
                        gb10 += dp0, gb11 += dp1;
                        d[nb][4 * i + e] = dp0, d[nb][4 * i + 2 + e] = dp1;
                    }
                }
            }

            // ---- GEMM2: dW1 += DP * X (A = DP from registers).  Phase 1: dp_lo * x_hi; phase 2 (DP
            // overwritten by dp_hi in place): dp_hi * x_lo, then dp_hi * x_hi into its own accumulator.
            uint32_t lo[2][16];
#pragma unroll
            for (int nb = 0; nb < 2; ++nb)
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const float hi = __uint_as_float(__float_as_uint(d[nb][i]) & 0xffffe000u);
                    lo[nb][i] = __float_as_uint(d[nb][i] - hi);
                    d[nb][i] = hi;
                }
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const int nb = kk >> 2, i = kk & 3;
                const uint32_t al[4] = {lo[nb][4 * i], lo[nb][4 * i + 2], lo[nb][4 * i + 1], lo[nb][4 * i + 3]};
                const uint32_t ah[4] = {__float_as_uint(d[nb][4 * i]), __float_as_uint(d[nb][4 * i + 2]),
                                        __float_as_uint(d[nb][4 * i + 1]), __float_as_uint(d[nb][4 * i + 3])};
#pragma unroll
                for (int fa = 0; fa < KA; ++fa) {
                    const uint32_t xo = nb * kXtAtomBytes + fa * 32 * 128 + i * 32;
                    tc::wgmma_n32_rs(acc_c[fa], al, tc::smem_desc_k_sw128(xt_hi, xo), true);
                    tc::wgmma_n32_rs(acc_c[fa], ah, tc::smem_desc_k_sw128(xt_lo, xo), true);
                    tc::wgmma_n32_rs(acc_hh[fa], ah, tc::smem_desc_k_sw128(xt_hi, xo), true);
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
            // the A registers are read asynchronously: keep them (and the accumulators) untouched until here
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) {
                tc::fence_acc(d[nb]);
#pragma unroll
                for (int i = 0; i < 16; ++i) asm volatile("" : "+r"(lo[nb][i])::"memory");
            }
#pragma unroll
            for (int fa = 0; fa < KA; ++fa) tc::fence_acc(acc_hh[fa]), tc::fence_acc(acc_c[fa]);
        }

        // ---- end of the pass: the quad's column sets meet (fixed order); dW1 / db1 / dW2 of the block
#pragma unroll
        for (int s = 1; s <= 2; s <<= 1) {
            gb10 += __shfl_xor_sync(IMPALA_FULL_MASK, gb10, s);
            gb11 += __shfl_xor_sync(IMPALA_FULL_MASK, gb11, s);
#pragma unroll
            for (int n = 0; n < NP; ++n) {
                gw0[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gw0[n], s);
                gw1[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gw1[n], s);
            }
        }
        if (q == 0) {
            wsb[a.lay.ob1 + j0] = gb10;
            wsb[a.lay.ob1 + j1] = gb11;
#pragma unroll
            for (int n = 0; n < NP; ++n)
                if (n < a.N2) wsb[a.lay.oW2 + (size_t)n * H + j0] = gw0[n], wsb[a.lay.oW2 + (size_t)n * H + j1] = gw1[n];
        }
#pragma unroll
        for (int fa = 0; fa < KA; ++fa) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int f = 32 * fa + 8 * i + 2 * q;  // features f, f + 1 (O % 4 == 0: both or neither valid)
                if (f < O) {
                    *reinterpret_cast<float2*>(wsb + a.lay.oW1 + (size_t)j0 * O + f) =
                        make_float2(acc_hh[fa][4 * i] + acc_c[fa][4 * i], acc_hh[fa][4 * i + 1] + acc_c[fa][4 * i + 1]);
                    *reinterpret_cast<float2*>(wsb + a.lay.oW1 + (size_t)j1 * O + f) =
                        make_float2(acc_hh[fa][4 * i + 2] + acc_c[fa][4 * i + 2], acc_hh[fa][4 * i + 3] + acc_c[fa][4 * i + 3]);
                }
            }
        }
    }

    // db2: fixed-order tree over the 64 threads that loaded dz rows
#pragma unroll
    for (int n = 0; n < NP; ++n) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) gb2[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gb2[n], off);
    }
    if (tid == 32) {
#pragma unroll
        for (int n = 0; n < NP; ++n) gb2x[n] = gb2[n];
    }
    __syncthreads();
    if (tid == 0) {
#pragma unroll
        for (int n = 0; n < NP; ++n)
            if (n < a.N2) wsb[a.lay.ob2 + n] = gb2[n] + gb2x[n];
    }
    __threadfence();  // this thread's partial-row stores are visible device-wide
    __syncthreads();
    return x_hi;
}

// Grid barrier: every CTA of the launch is resident (grid <= SM count, COOPERATIVE launch - it
// fails instead of hanging where co-residency cannot be had).  ctl[0] counts arrivals; a workspace
// that was not zero-filled once traps instead of hanging.
__device__ __forceinline__ void grid_arrive_and_wait(unsigned int* ctl) {
    if (threadIdx.x == 0) {
        atomicAdd(ctl, 1u);
        const long long t0 = clock64();
        unsigned int seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(ctl) : "memory");
            if (seen != gridDim.x && clock64() - t0 > (1ll << 32)) __trap();
        } while (seen != gridDim.x);
    }
    __syncthreads();
}

// The last CTA out re-arms the barrier for the next launch.
__device__ __forceinline__ void grid_depart(unsigned int* ctl) {
    if (threadIdx.x == 0 && atomicAdd(ctl + 1, 1u) == gridDim.x - 1) {
        ctl[0] = 0u;
        ctl[1] = 0u;
    }
}

// Deterministic float64 sum of `nparts` partial rows: chunk c = entries [64c, 64c + 64); this CTA
// takes chunks first, first + stride, ...; warp w adds rows w, w + kWarps, ... and warp 0 combines.
// `push`: the sums go to entry push_off + e of slot `rank` in every rank's gather buffer instead of
// a.grad (posted, step-tagged peer stores; the all-reduce of the data-parallel learner starts here).
__device__ __forceinline__ void reduce_rows(const BwdTcArgs& a, const int nparts, const int first,
                                            const int stride, double* s_red, const PushArgs* push = nullptr,
                                            const int64_t push_off = 0) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t total = a.lay.total;  // multiple of 32
    const int nchunks = (int)((total + 63) >> 6);
    for (int c = first; c < nchunks; c += stride) {
        const int64_t e0 = (int64_t)c * 64 + 2 * lane;
        double sx = 0.0, sy = 0.0;
        if (e0 < total) {
            const float* col = a.ws + e0;
            int p = warp;
            for (; p + 3 * kWarps < nparts; p += 4 * kWarps) {
                const float2 v0 = __ldcg(reinterpret_cast<const float2*>(col + (size_t)p * total));
                const float2 v1 = __ldcg(reinterpret_cast<const float2*>(col + (size_t)(p + kWarps) * total));
                const float2 v2 = __ldcg(reinterpret_cast<const float2*>(col + (size_t)(p + 2 * kWarps) * total));
                const float2 v3 = __ldcg(reinterpret_cast<const float2*>(col + (size_t)(p + 3 * kWarps) * total));
                sx += v0.x, sy += v0.y, sx += v1.x, sy += v1.y;
                sx += v2.x, sy += v2.y, sx += v3.x, sy += v3.y;
            }
            for (; p < nparts; p += kWarps) {
                const float2 v0 = __ldcg(reinterpret_cast<const float2*>(col + (size_t)p * total));
                sx += v0.x, sy += v0.y;
            }
        }
        s_red[warp * 64 + 2 * lane] = sx;
        s_red[warp * 64 + 2 * lane + 1] = sy;
        __syncthreads();
        if (push) {
            // Warp r sends the chunk to rank r: lane l carries entries l and l + 32, so each store
            // instruction covers 512 contiguous bytes of the peer's slot (4 full 128-byte lines).
            // Same summation order as below: every rank (and the single-GPU path) forms bit-identical
            // values.
            if (warp < push->world) {
                const int64_t ea = (int64_t)c * 64 + lane, eb = ea + 32;
                double va = 0.0, vb = 0.0;
#pragma unroll
                for (int w = 0; w < kWarps; ++w) va += s_red[w * 64 + lane], vb += s_red[w * 64 + 32 + lane];
                const long long step = *push->seq + 1;
                ulonglong2* dst = push->gather[warp] + (step & 1) * push->buf_stride +
                                  (int64_t)push->rank * push->slot_stride + push_off;
                if (ea < total) ll_store(dst + ea, va, (unsigned)step);
                if (eb < total) ll_store(dst + eb, vb, (unsigned)step);
            }
        } else if (warp == 0 && e0 < total) {
            double tx = 0.0, ty = 0.0;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) tx += s_red[w * 64 + 2 * lane], ty += s_red[w * 64 + 2 * lane + 1];
            *reinterpret_cast<double2*>(a.grad + e0) = make_double2(tx, ty);
        }
        __syncthreads();
    }
}

template <int NP>
__global__ void __launch_bounds__(kThreads, 1) mlp_bwd_tc_kernel(const __grid_constant__ BwdTcArgs a) {
    uint8_t* scratch = bwd_tc_body<NP, 1>(a, blockIdx.x, gridDim.x);
    grid_arrive_and_wait(a.ctl);
    reduce_rows(a, gridDim.x, blockIdx.x, gridDim.x, reinterpret_cast<double*>(scratch));
    grid_depart(a.ctl);
}

// Policy and value network of one learner step in ONE launch: CTAs [0, n_pi) take the policy's
// tiles (partial rows 0 .. n_pi of its workspace), the rest the value function's.  After the grid
// barrier every CTA helps reduce both sets of rows (the value function's chunks are dealt from
// the far end so that no CTA gets two chunks of each).  Uses the policy workspace's control words.
// PUSH: data-parallel learner - the reduced gradient [policy | value fn] and `n_extra` local
// scalars (the loss sums the V-trace kernel left at `extra`) go straight into every rank's gather
// buffer as step-tagged LL elements (protocol in optim.cu); nothing is written to a.grad.
template <bool PUSH>
__global__ void __launch_bounds__(kThreads, 1)
mlp_bwd_tc_pair_kernel(const __grid_constant__ BwdTcArgs a_pi, const __grid_constant__ BwdTcArgs a_vf,
                       const int n_pi, const __grid_constant__ PushArgs push, const double* extra,
                       const int n_extra) {
    const int n_vf = (int)gridDim.x - n_pi;
    uint8_t* scratch;
    if ((int)blockIdx.x < n_pi) scratch = bwd_tc_body<4, 1>(a_pi, blockIdx.x, n_pi);
    else scratch = bwd_tc_body<1, 1>(a_vf, (int)blockIdx.x - n_pi, n_vf);
    grid_arrive_and_wait(a_pi.ctl);
    const PushArgs* pp = PUSH ? &push : nullptr;
    reduce_rows(a_pi, n_pi, blockIdx.x, gridDim.x, reinterpret_cast<double*>(scratch), pp, 0);
    reduce_rows(a_vf, n_vf, (int)gridDim.x - 1 - (int)blockIdx.x, gridDim.x, reinterpret_cast<double*>(scratch), pp,
                a_pi.lay.total);
    if (PUSH && blockIdx.x == gridDim.x / 2 && (int)threadIdx.x < n_extra) {
        const long long step = *push.seq + 1;
        const int64_t off = (step & 1) * push.buf_stride + (int64_t)push.rank * push.slot_stride + a_pi.lay.total +
                            a_vf.lay.total + threadIdx.x;
        const double val = extra[threadIdx.x];
        for (int r = 0; r < push.world; ++r) ll_store(push.gather[r] + off, val, (unsigned)step);
    }
    grid_depart(a_pi.ctl);
}

// Wide shapes: partial rows only (reduce_partials_kernel sums them)
template <int NP, int KA>
__global__ void __launch_bounds__(kThreads) mlp_bwd_tcw_kernel(const __grid_constant__ BwdTcArgs a) {
    bwd_tc_body<NP, KA>(a, blockIdx.x, gridDim.x);
}

static_assert(kWarps * 64 * sizeof(double) <= 2 * kXAtomBytes, "reduction scratch fits the x stage");

// Dynamic shared memory opt-in (only ever raised, per kernel and device).
template <typename K>
cudaError_t opt_in(K kernel, size_t smem) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> opted;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    size_t& o = opted[std::make_pair((const void*)kernel, dev)];
    if (smem > o) {
        if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return e;
        o = smem;
    }
    return cudaSuccess;
}

BwdTcArgs make_bwd_args(const float* x, const float* params, const float* dout, float* ws, double* grad,
                        unsigned int* ctl, int M, int O, int H, int N2) {
    BwdTcArgs a{};
    a.x = x, a.params = params, a.dout = dout, a.ws = ws, a.grad = grad, a.ctl = ctl;
    a.M = M, a.O = O, a.H = H, a.N2 = N2;
    a.num_tiles = (M + kRowsT - 1) / kRowsT;
    a.lay = impala_make_layout(O, H, N2);
    return a;
}

}  // namespace

bool impala_mlp_bwd_tc_eligible(const float* x, const float* dout, int M, int O, int H, int N2) {
    return M >= 1 && O >= 4 && O <= 28 && (O & 3) == 0 && (H == 128 || H == 256) && N2 >= 1 &&
           N2 <= 4 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
           (reinterpret_cast<uintptr_t>(dout) & 15) == 0;
}

// Per-CTA partial gradient rows go to ws (same layout as the FP32 kernel), their float64 sum to
// grad; ctl = two zeroed control words (see the grid barrier in the kernel).
int impala_mlp_bwd_tc(const float* x, const float* params, const float* dout, float* ws,
                      double* grad, unsigned int* ctl, int M, int O, int H, int N2, cudaStream_t st) {
    const BwdTcArgs a = make_bwd_args(x, params, dout, ws, grad, ctl, M, O, H, N2);
    const size_t smem = bwd_smem_bytes(1, 4);
    cudaError_t e;
    int sms = 0;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    auto kernel = N2 == 1 ? mlp_bwd_tc_kernel<1> : mlp_bwd_tc_kernel<4>;
    if ((e = opt_in(kernel, smem)) != cudaSuccess) return (int)e;
    int grid = a.num_tiles < sms ? a.num_tiles : sms;  // <= SM count: the grid barrier needs residency
    if (grid > kMaxParts) grid = kMaxParts;
    if ((e = impala_launch_ex(kernel, grid, kThreads, smem, st, true, true, a)) != cudaSuccess) return (int)e;
    return impala_launch_status();
}

// Both networks in one launch; the caller has checked eligibility of each and 2 <= A <= 4.
// push != nullptr: data-parallel variant (see mlp_bwd_tc_pair_kernel).
int impala_mlp_bwd_tc_pair(const float* x, const float* params_pi, const float* params_vf,
                           const float* dlogits, const float* dv, float* ws_pi, float* ws_vf,
                           double* grad_pi, double* grad_vf, unsigned int* ctl, int M_pi, int M_vf, int O,
                           int H_pi, int H_vf, int A, cudaStream_t st, const PushArgs* push, const double* extra,
                           int n_extra) {
    const BwdTcArgs a_pi = make_bwd_args(x, params_pi, dlogits, ws_pi, grad_pi, ctl, M_pi, O, H_pi, A);
    const BwdTcArgs a_vf = make_bwd_args(x, params_vf, dv, ws_vf, grad_vf, ctl, M_vf, O, H_vf, 1);
    const size_t smem = bwd_smem_bytes(1, 4);
    cudaError_t e;
    int sms = 0;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    e = push ? opt_in(mlp_bwd_tc_pair_kernel<true>, smem) : opt_in(mlp_bwd_tc_pair_kernel<false>, smem);
    if (e != cudaSuccess) return (int)e;
    const int total_tiles = a_pi.num_tiles + a_vf.num_tiles;
    int grid = total_tiles < sms ? total_tiles : sms;
    if (grid > kMaxParts) grid = kMaxParts;
    if (grid < 2) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    const int n_pi = impala_pair_split(a_pi.num_tiles, a_vf.num_tiles, grid,
                                       impala_env_int("IMPALA_PAIR_W_BWD", 105) * (H_pi / 128),
                                       100 * (H_vf / 128));
    // cooperative launch: the in-kernel grid barrier needs every CTA resident
    e = push ? impala_launch_ex(mlp_bwd_tc_pair_kernel<true>, grid, kThreads, smem, st, true, true, a_pi, a_vf, n_pi,
                                *push, extra, n_extra)
             : impala_launch_ex(mlp_bwd_tc_pair_kernel<false>, grid, kThreads, smem, st, true, true, a_pi, a_vf, n_pi,
                                PushArgs{}, (const double*)nullptr, 0);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

// Wide shapes (impala_mlp_tcw_eligible): per-CTA float32 partial gradient rows into ws (row stride =
// layout total); *nparts = rows written.
int impala_mlp_bwd_tcw(const float* x, const float* params, const float* dout, float* ws, int M, int O, int H,
                       int N2, cudaStream_t st, int* nparts) {
    const BwdTcArgs a = make_bwd_args(x, params, dout, ws, nullptr, nullptr, M, O, H, N2);
    const int ka = O <= 32 ? 1 : 2;
    const size_t smem = bwd_smem_bytes(ka, N2 == 1 ? 1 : 4);
    auto kernel = ka == 1 ? (N2 == 1 ? mlp_bwd_tcw_kernel<1, 1> : mlp_bwd_tcw_kernel<4, 1>)
                          : (N2 == 1 ? mlp_bwd_tcw_kernel<1, 2> : mlp_bwd_tcw_kernel<4, 2>);
    cudaError_t e;
    int sms = 0, per_sm = 0;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    if ((e = opt_in(kernel, smem)) != cudaSuccess) return (int)e;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem)) != cudaSuccess) return (int)e;
    if (per_sm < 1) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    int grid = per_sm * sms;
    if (grid > a.num_tiles) grid = a.num_tiles;
    if (grid > kMaxParts) grid = kMaxParts;
    if ((e = impala_launch(kernel, grid, kThreads, smem, st, true, a)) != cudaSuccess) return (int)e;
    *nparts = grid;
    return impala_launch_status();
}
