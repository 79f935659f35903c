// MLP backward on the Hopper tensor cores (wgmma, fp32 accumulators in registers), error-compensated
// 3xTF32.
//
// Gradient of sum_m <dout[m,:], mlp(x[m,:])> w.r.t. (W1, b1, W2, b2)  (autograd at learner.py:175).
// Transposed formulation so that a thread owns HIDDEN units (accumulator rows = hidden units), per
// tile of 64 batch rows and warpgroup (64 hidden units):
//
//   GEMM1 (recompute)      PRE[64 hid, 64 rows] = W1_blk[64, K] * X[64 rows, K]^T
//   CUDA cores             h = relu(PRE + b1); dh = W2^T dz; dW2 += dz h; DP = (PRE + b1 > 0) ? dh : 0;
//                          db1 += DP
//   GEMM2 (RS, reduction)  dW1_blk[64 hid, K] += DP[64 hid, 64 rows] * X[64 rows, K]
//
// K = the observation width padded to 32 (one 128-byte swizzle atom), 64 (two atoms, BASELINE c5) or
// 128 (four atoms, Atari RAM; see bwd_tc_body).
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
// registers over every tile of the persistent CTA (or warpgroup) and is written out once per pass.
//
// Every gradient entry of W1 / b1 / W2 belongs to exactly one hidden unit, so each CTA writes a float32
// partial gradient row (same layout as the FP32 kernels) and the rows are summed in float64 in a fixed
// order.
//
// Narrow shapes (Narrow plans: one K atom, <= 4 outputs; bwd_blk_body): a CTA owns ONE
// 64-unit hidden block of one network for the whole launch, so W1 of the block is loaded once and held
// in registers as GEMM1's A operand (only the x tile is read from shared memory).  Its two warpgroups
// are independent - each takes alternate tiles of the CTA's share, with its own x stage and named
// barrier - so one warpgroup's MMAs overlap the other's CUDA-core epilogue (their GEMM2s are issued in
// turn, see the ping-pong comment in the body).  The warpgroups meet once,
// at the end (fixed order), and the rows are summed in-kernel after a grid barrier (paired launch,
// optional peer push).  GEMM1 covers the tile's 64 batch rows with one m64n64 MMA per product (the
// accumulator is the two 32-row halves side by side, so every entry takes the same products in the same
// order as with two m64n32 chains); GEMM2 (N = 32 features) stays m64n32.
//
// Wide shapes (bwd_tc_body): one CTA = 2 warpgroups = 128 hidden units per pass, wider layers walked
// in passes (x is re-read once per pass); reduce_partials_kernel sums the rows.
#include "mlp_kernels.cuh"
#include "phase_clocks.cuh"
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

// The arguments of the split-head twins (SPLIT kernels): dout is head a, dout_b head b (split_dz).  A
// struct of its own, so the kernels of the interleaved layout keep their parameter space.
struct BwdTcSplitArgs : BwdTcArgs {
    const float* dout_b;
    int M_a;
};
template <bool SPLIT>
using BwdArgs = std::conditional_t<SPLIT, BwdTcSplitArgs, BwdTcArgs>;

// dz entry (row, n0 + n) of the tile loads: interleaved (M, N2) rows, or the split heads (SPLIT twins).  The dense
// address is formed as the loads always formed it, row start + n0 + n, so the dense kernels keep their code
template <bool SPLIT>
__device__ __forceinline__ float load_dz(const BwdArgs<SPLIT>& a, int row, int n0, int n) {
    if constexpr (SPLIT) return split_dz(a.dout, a.dout_b, a.M_a, a.N2, row, n0 + n);
    else return __ldg(a.dout + (size_t)row * a.N2 + n0 + n);
}

__host__ __device__ constexpr size_t bwd_smem_bytes(int ka, int np) {
    // W1 block hi / lo [KA][128 hidden][128 B] + x hi / lo [KA][RT rows][128 B] + x^T hi / lo
    // [RT / 32 K atoms][32 KA features][128 B] + dz [RT][NPS] + db2 exchange; NP = 32 (layer 2 through
    // shared memory): + W2 block [128 hidden][NPS] + db2 exchange [8 warps][32]
    return 1024 + (size_t)2 * ka * kHB * 128 + (size_t)2 * ka * (ka == 4 ? 32 : kRowsT) * 128 +
           (size_t)2 * ((ka == 4 ? 32 : kRowsT) / 32) * 32 * ka * 128 +
           (size_t)(ka == 4 ? 32 : kRowsT) * (np > 4 ? np + 4 : np) * sizeof(float) +
           (np > 4 ? (size_t)kHB * (np + 4) * sizeof(float) + 8 * 32 * sizeof(float) : 4 * sizeof(float));
}

// component e of a float4 (e known at compile time)
__device__ __forceinline__ float f4(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

// One persistent CTA's share of a network's backward: CTA `cta` of `ncta` takes tiles cta,
// cta + ncta, ... and leaves its float32 partial gradient in row `cta` of a.ws.  Returns a shared
// memory region of >= 16 KiB the caller may use as scratch once every thread is past it.
//
// KA = 4 (observations up to 128): the dW1 accumulators of all four feature atoms would be 128
// registers per thread, so a pass holds one 64-feature half of dW1 (two atoms) and the hidden blocks
// are walked once per half, GEMM1 re-run for each (x is re-read once per pass).  Tiles are 32 batch rows
// so that W1 hi / lo of 128 hidden units, the tile and its transpose fit in shared memory.
// NP = 16 / 32 (5..16 outputs at one or two K atoms, 17..32 outputs at four): layer 2 goes through shared
// memory - the pass's W2 block [128][NP + 4] (rows padded so the lanes of a quad, two batch rows or hidden
// units apart, hit different banks) - and dW2 is formed per tile in chunks of NP / 4 outputs, summed over
// the quad and kept by lane q for outputs [NP / 4 q, NP / 4 (q + 1)).  dW2 / db1 are accumulated in the
// first feature half only.
template <int NP, int KA, bool SPLIT = false>
__device__ __forceinline__ uint8_t* bwd_tc_body(const BwdArgs<SPLIT>& a, const int cta, const int ncta) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr bool X4 = KA == 4;
    constexpr bool L2S = NP > 4;                      // layer 2 through shared memory
    constexpr int RT = X4 ? 32 : kRowsT;             // batch rows per tile
    constexpr int NB = RT / 32;                       // N = 32 halves of GEMM1 / K atoms of GEMM2
    constexpr int FA = X4 ? 2 : KA;                   // feature atoms of dW1 per pass
    constexpr int NPS = L2S ? NP + 4 : NP;            // row stride of dz (and W2) in shared memory
    constexpr int NPR = L2S ? 1 : NP;                 // layer-2 values held in registers
    constexpr int kXA = RT * 128;                     // one x atom: RT rows x 128 B
    constexpr int kWBytes = KA * kHB * 128;          // one of hi / lo, [KA][128 rows][128 B]
    constexpr int kXBytes = KA * kXA;                // one of hi / lo, [KA][RT rows][128 B]
    constexpr int kXtAtomBytes = 32 * KA * 128;      // 32 batch rows of K x 32 KA feature rows
    uint8_t* w_hi = smem;
    uint8_t* w_lo = w_hi + kWBytes;
    uint8_t* x_hi = w_lo + kWBytes;
    uint8_t* x_lo = x_hi + kXBytes;
    uint8_t* xt_hi = x_lo + kXBytes;                 // [NB K atoms][32 KA rows][128 B]
    uint8_t* xt_lo = xt_hi + NB * kXtAtomBytes;
    float* dzs = reinterpret_cast<float*>(xt_lo + NB * kXtAtomBytes);  // [RT rows][NPS]
    float* gb2x = dzs + RT * NPS;                                      // [4] | [8 warps][32]
    float* w2s = gb2x + (L2S ? 8 * 32 : 4);                            // L2S: [128 hidden][NPS]

    const int tid = threadIdx.x, wg = tid >> 7, lt = tid & 127, warp = lt >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int O = a.O, H = a.H, ochunks = O >> 2, ksteps = (O + 7) >> 3;
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;
    float* wsb = a.ws + (size_t)cta * a.lay.total;  // this CTA's partial gradient row

    // x rows of a tile -> registers (chunk idx = tid + kThreads k is (row idx / (8 KA), 16-byte chunk
    // idx % (8 KA))); dz row `tid` for tid < RT (L2S: dz row tid / NQ, outputs 4 (tid % NQ) .. + 3)
    constexpr int kLd = RT * 8 * KA / kThreads;
    constexpr int NZ = L2S ? 4 : NP;
    constexpr int NQ = L2S ? NP / 4 : 1;  // L2S: float4s of a dz row
    constexpr int CW = L2S ? NP / 4 : 1;  // L2S: outputs of a dW2 chunk (lane q keeps chunk q)
    float4 v[kLd];
    float z[NZ];
    auto load = [&](int tile) {
#pragma unroll
        for (int k = 0; k < kLd; ++k) {
            const int idx = tid + kThreads * k, r = idx / (8 * KA), c = idx % (8 * KA);
            const int row = tile * RT + r;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tile < a.num_tiles && row < a.M && c < ochunks)
                v[k] = __ldg(reinterpret_cast<const float4*>(a.x + (size_t)row * O) + c);
        }
        if constexpr (L2S) {
            // NP = 32 at RT = 32 (four K atoms) or NP = 16 at RT = 64
            static_assert(RT * NP == 4 * kThreads, "one float4 of dz per thread");
            const int row = tile * RT + tid / NQ, n0 = 4 * (tid % NQ);
#pragma unroll
            for (int n = 0; n < 4; ++n)
                z[n] = (tile < a.num_tiles && row < a.M && n0 + n < a.N2) ? load_dz<SPLIT>(a, row, n0, n) : 0.f;
        } else {
            const int row = tile * RT + tid;
#pragma unroll
            for (int n = 0; n < NP; ++n)
                z[n] = (tid < RT && tile < a.num_tiles && row < a.M && n < a.N2) ? load_dz<SPLIT>(a, row, 0, n) : 0.f;
        }
    };
    float gb2[NZ];  // db2 = column sums of dout: this thread's dz values, first pass only
#pragma unroll
    for (int n = 0; n < NZ; ++n) gb2[n] = 0.f;

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
    const int nfh = X4 ? (O + 63) / 64 : 1;  // feature halves of dW1
    const int npass = H / kHB * nfh;
    for (int p = 0; p < npass; ++p) {
        const int blk = X4 ? p / nfh : p, fh = X4 ? p % nfh : 0;
        const bool l2 = X4 ? fh == 0 : true;  // this pass forms db1 / dW2 (and, first of all, db2)
        const int fa0 = X4 ? 2 * fh : 0;      // first feature atom of this pass's dW1
        // ---- this pass's W1 rows -> hi / lo swizzled tiles (warpgroup w: rows [64 w, 64 w + 64))
        __syncthreads();  // the previous pass is done with the weights
        for (int idx = tid; idx < kHB * 8 * KA; idx += kThreads) {
            const int r = idx / (8 * KA), c = idx % (8 * KA);
            float4 w = make_float4(0.f, 0.f, 0.f, 0.f), hi, lo;
            if (c < ochunks) w = __ldg(reinterpret_cast<const float4*>(W1 + (size_t)(blk * kHB + r) * O) + c);
            tc::split4(w, hi, lo);
            const uint32_t off = (r >> 6) * (KA * 64 * 128) + (c >> 3) * (64 * 128) + tc::sw128_offset(r & 63, c & 7);
            *reinterpret_cast<float4*>(w_hi + off) = hi;
            *reinterpret_cast<float4*>(w_lo + off) = lo;
        }
        if constexpr (L2S) {
            for (int idx = tid; idx < kHB * NP; idx += kThreads) {
                const int j = idx / NP, n = idx - j * NP;
                w2s[j * NPS + n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + blk * kHB + j) : 0.f;
            }
        }
        uint8_t* wa_hi = w_hi + wg * (KA * 64 * 128);  // this warpgroup's A operand of GEMM1
        uint8_t* wa_lo = w_lo + wg * (KA * 64 * 128);
        // the thread's two hidden units
        const int j0 = blk * kHB + 64 * wg + 16 * warp + g, j1 = j0 + 8;
        const float bj0 = __ldg(b1 + j0), bj1 = __ldg(b1 + j1);
        float w2r0[NPR], w2r1[NPR], gw0[NPR], gw1[NPR], gb10 = 0.f, gb11 = 0.f;
        float gq0[CW], gq1[CW];  // L2S: dW2 of outputs [CW q, CW q + CW)
        if constexpr (L2S) {
#pragma unroll
            for (int k = 0; k < CW; ++k) gq0[k] = gq1[k] = 0.f;
        } else {
#pragma unroll
            for (int n = 0; n < NP; ++n) {
                w2r0[n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + j0) : 0.f;
                w2r1[n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + j1) : 0.f;
                gw0[n] = gw1[n] = 0.f;
            }
        }
        float acc_hh[FA][16], acc_c[FA][16];  // dW1: dp_hi * x_hi | dp_hi * x_lo + dp_lo * x_hi
#pragma unroll
        for (int fa = 0; fa < FA; ++fa)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc_hh[fa][i] = acc_c[fa][i] = 0.f;
#pragma unroll
        for (int fa = 0; fa < FA; ++fa) tc::fence_acc(acc_hh[fa]), tc::fence_acc(acc_c[fa]);

        load(cta);
        for (int tile = cta, it = 0; tile < a.num_tiles; tile += ncta, ++it) {
            // ---- stage the tile: x row-major (B of GEMM1) and transposed (B of GEMM2), hi / lo; dz
            __syncthreads();  // every MMA that read the previous tile has retired
#pragma unroll
            for (int k = 0; k < kLd; ++k) {
                const int idx = tid + kThreads * k, r = idx / (8 * KA), c = idx % (8 * KA);
                float4 hi, lo;
                tc::split4(v[k], hi, lo);
                const uint32_t off = (c >> 3) * kXA + tc::sw128_offset(r, c & 7);
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
            if constexpr (L2S) {
                *reinterpret_cast<float4*>(dzs + (tid / NQ) * NPS + 4 * (tid % NQ)) = make_float4(z[0], z[1], z[2], z[3]);
                if (p == 0) {
#pragma unroll
                    for (int n = 0; n < 4; ++n) gb2[n] += z[n];
                }
            } else if (tid < RT) {
#pragma unroll
                for (int n = 0; n < NP; ++n) {
                    dzs[tid * NP + n] = z[n];
                    if (p == 0) gb2[n] += z[n];
                }
            }
            tc::fence_proxy_async();
            __syncthreads();
            load(tile + ncta);  // in flight during this tile's MMAs and epilogue

            // ---- GEMM1: PRE = W1_blk * X^T (N = 32 halves of the tile's batch rows)
            float d[NB][16];
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                for (int i = 0; i < 16; ++i) d[nb][i] = 0.f;
            // the zeroed accumulators are defined HERE, before the warpgroup fence: left alone, the compiler
            // sinks the moves behind the K-step guards, past the fence, and ptxas then serializes every wgmma
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) tc::fence_acc(d[nb]);
            tc::wgmma_fence();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t wo = (kk >> 2) * (64 * 128) + (kk & 3) * 32;
                        const uint32_t xo = (kk >> 2) * kXA + nb * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d[nb], tc::smem_desc_k_sw128(wa_lo, wo), tc::smem_desc_k_sw128(x_hi, xo), kk > 0);
                        tc::wgmma_n32_ss(d[nb], tc::smem_desc_k_sw128(wa_hi, wo), tc::smem_desc_k_sw128(x_lo, xo), true);
                    }
                }
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t wo = (kk >> 2) * (64 * 128) + (kk & 3) * 32;
                        const uint32_t xo = (kk >> 2) * kXA + nb * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d[nb], tc::smem_desc_k_sw128(wa_hi, wo), tc::smem_desc_k_sw128(x_hi, xo), true);
                    }
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) tc::fence_acc(d[nb]);

            // ---- epilogue: d <- DP in place (thread: hidden units j0 / j1, batch columns 8 i + 2 q + e)
            if constexpr (L2S) {
                const float* w2a = w2s + (64 * wg + 16 * warp + g) * NPS;  // unit j0 of the block
                const float* w2b = w2a + 8 * NPS;
                // d <- h in place: h > 0 exactly where the pre-activation is (relu'(0) = 0 as in torch), and
                // the dW2 chunks read h without holding a second copy of it
#pragma unroll
                for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                    for (int i = 0; i < 16; ++i) d[nb][i] = fmaxf(d[nb][i] + ((i & 2) ? bj1 : bj0), 0.f);
                if (l2) {
                    // dW2 in chunks of CW outputs: the quad's partial sums meet, lane q keeps chunk q
#pragma unroll
                    for (int cc = 0; cc < 4; ++cc) {
                        float s0[CW], s1[CW];
#pragma unroll
                        for (int k = 0; k < CW; ++k) s0[k] = s1[k] = 0.f;
#pragma unroll
                        for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                            for (int i = 0; i < 4; ++i)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const int m = 32 * nb + 8 * i + 2 * q + e;
                                    const float h0 = d[nb][4 * i + e], h1 = d[nb][4 * i + 2 + e];
                                    float4 zc[CW / 4];
#pragma unroll
                                    for (int u = 0; u < CW / 4; ++u)
                                        zc[u] = *reinterpret_cast<const float4*>(dzs + m * NPS + CW * cc + 4 * u);
#pragma unroll
                                    for (int k = 0; k < CW; ++k) {
                                        const float zk = f4(zc[k >> 2], k & 3);
                                        s0[k] = fmaf(zk, h0, s0[k]), s1[k] = fmaf(zk, h1, s1[k]);
                                    }
                                }
#pragma unroll
                        for (int k = 0; k < CW; ++k) {
                            s0[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s0[k], 1);
                            s1[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s1[k], 1);
                            s0[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s0[k], 2);
                            s1[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s1[k], 2);
                        }
                        if (q == cc) {
#pragma unroll
                            for (int k = 0; k < CW; ++k) gq0[k] += s0[k], gq1[k] += s1[k];
                        }
                    }
                }
#pragma unroll
                for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int m = 32 * nb + 8 * i + 2 * q + e;
                            const float h0 = d[nb][4 * i + e], h1 = d[nb][4 * i + 2 + e];
                            float dh0 = 0.f, dh1 = 0.f;
#pragma unroll
                            for (int n = 0; n < NP; n += 4) {
                                const float4 zv = *reinterpret_cast<const float4*>(dzs + m * NPS + n);
                                const float4 wa = *reinterpret_cast<const float4*>(w2a + n);
                                const float4 wb = *reinterpret_cast<const float4*>(w2b + n);
                                dh0 = fmaf(zv.x, wa.x, dh0), dh0 = fmaf(zv.y, wa.y, dh0);
                                dh0 = fmaf(zv.z, wa.z, dh0), dh0 = fmaf(zv.w, wa.w, dh0);
                                dh1 = fmaf(zv.x, wb.x, dh1), dh1 = fmaf(zv.y, wb.y, dh1);
                                dh1 = fmaf(zv.z, wb.z, dh1), dh1 = fmaf(zv.w, wb.w, dh1);
                            }
                            const float dp0 = h0 > 0.f ? dh0 : 0.f, dp1 = h1 > 0.f ? dh1 : 0.f;
                            gb10 += dp0, gb11 += dp1;
                            d[nb][4 * i + e] = dp0, d[nb][4 * i + 2 + e] = dp1;
                        }
            } else {
#pragma unroll
                for (int nb = 0; nb < NB; ++nb) {
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
                            if (!X4 || l2) {
#pragma unroll
                                for (int n = 0; n < NP; ++n) gw0[n] = fmaf(dz[n], h0, gw0[n]), gw1[n] = fmaf(dz[n], h1, gw1[n]);
                            }
                            const float dp0 = pre0 > 0.f ? dh0 : 0.f, dp1 = pre1 > 0.f ? dh1 : 0.f;
                            gb10 += dp0, gb11 += dp1;
                            d[nb][4 * i + e] = dp0, d[nb][4 * i + 2 + e] = dp1;
                        }
                    }
                }
            }

            // ---- GEMM2: dW1 += DP * X (A = DP from registers).  Phase 1: dp_lo * x_hi; phase 2 (DP
            // overwritten by dp_hi in place): dp_hi * x_lo, then dp_hi * x_hi into its own accumulator.
            // X4: round-to-nearest split (lo of either sign), so the tensor core's truncation of lo does not
            // pull every product of the longer K = 128 reductions towards zero
            uint32_t lo[NB][16];
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    if constexpr (X4) {
                        float hi, lof;
                        tc::split_tf32(d[nb][i], hi, lof);
                        lo[nb][i] = __float_as_uint(lof);
                        d[nb][i] = hi;
                    } else {
                        const float hi = __uint_as_float(__float_as_uint(d[nb][i]) & 0xffffe000u);
                        lo[nb][i] = __float_as_uint(d[nb][i] - hi);
                        d[nb][i] = hi;
                    }
                }
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4 * NB; ++kk) {
                const int nb = kk >> 2, i = kk & 3;
                const uint32_t al[4] = {lo[nb][4 * i], lo[nb][4 * i + 2], lo[nb][4 * i + 1], lo[nb][4 * i + 3]};
                const uint32_t ah[4] = {__float_as_uint(d[nb][4 * i]), __float_as_uint(d[nb][4 * i + 2]),
                                        __float_as_uint(d[nb][4 * i + 1]), __float_as_uint(d[nb][4 * i + 3])};
#pragma unroll
                for (int fa = 0; fa < FA; ++fa) {
                    const uint32_t xo = nb * kXtAtomBytes + (fa0 + fa) * 32 * 128 + i * 32;
                    tc::wgmma_n32_rs(acc_c[fa], al, tc::smem_desc_k_sw128(xt_hi, xo), true);
                    tc::wgmma_n32_rs(acc_c[fa], ah, tc::smem_desc_k_sw128(xt_lo, xo), true);
                    tc::wgmma_n32_rs(acc_hh[fa], ah, tc::smem_desc_k_sw128(xt_hi, xo), true);
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
            // the A registers are read asynchronously: keep them (and the accumulators) untouched until here
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
                tc::fence_acc(d[nb]);
#pragma unroll
                for (int i = 0; i < 16; ++i) asm volatile("" : "+r"(lo[nb][i])::"memory");
            }
#pragma unroll
            for (int fa = 0; fa < FA; ++fa) tc::fence_acc(acc_hh[fa]), tc::fence_acc(acc_c[fa]);
        }

        // ---- end of the pass: the quad's column sets meet (fixed order); dW1 / db1 / dW2 of the block
        if (!X4 || l2) {
#pragma unroll
            for (int s = 1; s <= 2; s <<= 1) {
                gb10 += __shfl_xor_sync(IMPALA_FULL_MASK, gb10, s);
                gb11 += __shfl_xor_sync(IMPALA_FULL_MASK, gb11, s);
#pragma unroll
                for (int n = 0; n < NPR; ++n) {
                    if constexpr (!L2S) {
                        gw0[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gw0[n], s);
                        gw1[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gw1[n], s);
                    }
                }
            }
            if (q == 0) {
                wsb[a.lay.ob1 + j0] = gb10;
                wsb[a.lay.ob1 + j1] = gb11;
                if constexpr (!L2S) {
#pragma unroll
                    for (int n = 0; n < NP; ++n)
                        if (n < a.N2) wsb[a.lay.oW2 + (size_t)n * H + j0] = gw0[n], wsb[a.lay.oW2 + (size_t)n * H + j1] = gw1[n];
                }
            }
            if constexpr (L2S) {
#pragma unroll
                for (int k = 0; k < CW; ++k) {
                    const int n = CW * q + k;
                    if (n < a.N2) wsb[a.lay.oW2 + (size_t)n * H + j0] = gq0[k], wsb[a.lay.oW2 + (size_t)n * H + j1] = gq1[k];
                }
            }
        }
#pragma unroll
        for (int fa = 0; fa < FA; ++fa) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int f = 32 * (fa0 + fa) + 8 * i + 2 * q;  // features f, f + 1 (O % 4 == 0: both or neither valid)
                if (f < O) {
                    *reinterpret_cast<float2*>(wsb + a.lay.oW1 + (size_t)j0 * O + f) =
                        make_float2(acc_hh[fa][4 * i] + acc_c[fa][4 * i], acc_hh[fa][4 * i + 1] + acc_c[fa][4 * i + 1]);
                    *reinterpret_cast<float2*>(wsb + a.lay.oW1 + (size_t)j1 * O + f) =
                        make_float2(acc_hh[fa][4 * i + 2] + acc_c[fa][4 * i + 2], acc_hh[fa][4 * i + 3] + acc_c[fa][4 * i + 3]);
                }
            }
        }
    }

    if constexpr (L2S) {
        // db2: thread t holds outputs 4 (t % NQ) .. + 3 of rows t / NQ (+ RT k); the lanes l ^ NQ,
        // l ^ 2 NQ, ... hold the same outputs, then the 8 warps meet through shared memory (fixed order)
#pragma unroll
        for (int n = 0; n < 4; ++n) {
#pragma unroll
            for (int off = NQ; off < 32; off <<= 1) gb2[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gb2[n], off);
        }
        if (lane < NQ) {
#pragma unroll
            for (int n = 0; n < 4; ++n) gb2x[(tid >> 5) * 32 + 4 * lane + n] = gb2[n];
        }
        __syncthreads();
        if (tid < a.N2) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) s += gb2x[w * 32 + tid];
            wsb[a.lay.ob2 + tid] = s;
        }
    } else {
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
    }
    __threadfence();  // this thread's partial-row stores are visible device-wide
    __syncthreads();
    return x_hi;
}

// ---- narrow shapes: one 64-unit hidden block per CTA, independent warpgroups
constexpr int kXtBytes = 2 * 32 * 128;  // x^T: 2 K atoms of 32 batch rows, 32 feature rows of 128 B
// one warpgroup's stage: x hi / lo, x^T hi / lo (1024-byte aligned), dz [64 rows][<= 4]
constexpr int kStageBytes = 2 * kXAtomBytes + 2 * kXtBytes + kRowsT * 4 * (int)sizeof(float);
// + the db2 exchange [4 dz-loading warps][4]
constexpr size_t kBlkSmemBytes = 1024 + (size_t)kWG * kStageBytes + 16 * sizeof(float);
static_assert(kStageBytes % 1024 == 0, "stages stay 1024-byte aligned");

// CTA `cta` of the `ncta` that take one network (a multiple of its H / 64 hidden blocks) belongs to
// group cta / (ncta / (H / 64)) - the group of a hidden block - and is CTA `r` = cta % (ncta / (H / 64))
// of it: it takes the tiles r, r + ncta / (H / 64), ... (warpgroups alternating) for its block and writes
// the block's entries of partial row r (dW1 rows, db1, dW2 columns; group 0 also db2 and the pads), so
// that the rows hold every entry exactly once each.  Returns >= 16 KiB of shared memory the caller may
// use as scratch.
template <int NP, bool SPLIT = false>
__device__ __forceinline__ uint8_t* bwd_blk_body(const BwdArgs<SPLIT>& a, const int cta, const int ncta) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    // the warpgroup index broadcast from lane 0: known warp-uniform, so the stage addresses and the
    // wgmma descriptors built from them stay in uniform registers
    const int wg = __shfl_sync(IMPALA_FULL_MASK, (int)threadIdx.x >> 7, 0);
    const int tid = threadIdx.x, lt = tid & 127, warp = lt >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int O = a.O, H = a.H, ochunks = O >> 2, ksteps = (O + 7) >> 3;
    const int cpg = ncta / (H / 64), grp = cta / cpg, r = cta - grp * cpg;
    uint8_t* x_hi = smem + wg * kStageBytes;
    uint8_t* x_lo = x_hi + kXAtomBytes;
    uint8_t* xt_hi = x_lo + kXAtomBytes;  // [2 K atoms][32 feature rows][128 B]
    uint8_t* xt_lo = xt_hi + kXtBytes;
    float* dzs = reinterpret_cast<float*>(xt_lo + kXtBytes);         // [64 rows][NP]
    float* gb2x = reinterpret_cast<float*>(smem + kWG * kStageBytes);  // [4 warps][4]
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;
    float* wsb = a.ws + (size_t)r * a.lay.total;

    if (grp == 0) {  // pads of the partial row
        const int64_t lo4[4] = {a.lay.oW1 + (int64_t)H * O, a.lay.ob1 + H, a.lay.oW2 + (int64_t)a.N2 * H,
                                a.lay.ob2 + a.N2};
        const int64_t hi4[4] = {a.lay.ob1, a.lay.oW2, a.lay.ob2, a.lay.total};
        for (int sgm = 0; sgm < 4; ++sgm)
            for (int64_t p = lo4[sgm] + tid; p < hi4[sgm]; p += kThreads) wsb[p] = 0.f;
    }

    // x rows of a tile -> registers: thread (warp, lane) holds row 16 warp + lane % 16, 16-byte chunks
    // 2 k + lane / 16 (a warp's transposed stores then hit 32 different banks, and chunk pairs GEMM1
    // never reads, k >= ksteps, are skipped by whole warps); dz row lt for lt < 64
    constexpr int kLd = kRowsT * 8 / 128;
    const int rr = 16 * warp + (lane & 15);
    float4 v[kLd];
    float z[NP];
    auto load = [&](int tile) {
#pragma unroll
        for (int k = 0; k < kLd; ++k) {
            const int c = 2 * k + (lane >> 4), row = tile * kRowsT + rr;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < ksteps && tile < a.num_tiles && row < a.M && c < ochunks)
                v[k] = __ldg(reinterpret_cast<const float4*>(a.x + (size_t)row * O) + c);
        }
        const int row = tile * kRowsT + lt;
#pragma unroll
        for (int n = 0; n < NP; ++n)
            z[n] = (lt < kRowsT && tile < a.num_tiles && row < a.M && n < a.N2) ? load_dz<SPLIT>(a, row, 0, n) : 0.f;
    };
    float gb2[NP];  // db2 = column sums of dout: this thread's dz values
#pragma unroll
    for (int n = 0; n < NP; ++n) gb2[n] = 0.f;

    // dz of the tile is the output of the kernel before this one (PDL, common.cuh)
    pdl_wait();
    // the thread's two hidden units; W1 hi / lo of both as GEMM1's A fragments (K step kk: feature
    // 8 kk + q + 4 (i >> 1) of unit i & 1 ? j1 : j0), for the whole launch
    const int j0 = 64 * grp + 16 * warp + g, j1 = j0 + 8;
    uint32_t wh[4][4], wl[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = 8 * kk + q + 4 * (i >> 1);
            float hi, lo;
            tc::split_tf32(f < O ? __ldg(W1 + (size_t)(i & 1 ? j1 : j0) * O + f) : 0.f, hi, lo);
            wh[kk][i] = __float_as_uint(hi), wl[kk][i] = __float_as_uint(lo);
        }
    const float bj0 = __ldg(b1 + j0), bj1 = __ldg(b1 + j1);
    float w2r0[NP], w2r1[NP], gw0[NP], gw1[NP], gb10 = 0.f, gb11 = 0.f;
#pragma unroll
    for (int n = 0; n < NP; ++n) {
        w2r0[n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + j0) : 0.f;
        w2r1[n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + j1) : 0.f;
        gw0[n] = gw1[n] = 0.f;
    }
    float acc_hh[16], acc_c[16];  // dW1: dp_hi * x_hi | dp_hi * x_lo + dp_lo * x_hi
#pragma unroll
    for (int i = 0; i < 16; ++i) acc_hh[i] = acc_c[i] = 0.f;
    tc::fence_acc(acc_hh), tc::fence_acc(acc_c);
    const uint64_t dx_hi = tc::smem_desc_k_sw128(x_hi, 0), dx_lo = tc::smem_desc_k_sw128(x_lo, 0);
    const uint64_t dxt_hi = tc::smem_desc_k_sw128(xt_hi, 0), dxt_lo = tc::smem_desc_k_sw128(xt_lo, 0);

    const int bar = 1 + wg, tstride = 2 * cpg;  // this warpgroup's named barrier and tile stride
    // Ping-pong: the warpgroups take turns to issue GEMM2, the larger of a tile's two MMA batches: warpgroup
    // 0's, warpgroup 1's, warpgroup 0's, ..., so that their GEMM2s reach the tensor pipe one after the other
    // instead of together, each while the other warpgroup runs its epilogue or staging.  Turn barrier 3 + w
    // (256 threads) is warpgroup w's: it syncs on its own before the issue and arrives on the other's after
    // the commit.  Warpgroup 0 takes n0 turns and warpgroup 1 as many (n0 - n1 <= 1: one empty turn after its
    // last tile), and every arrival is awaited: warpgroup 0 skips the sync of its first turn, warpgroup 1 the
    // arrival of its last, so both barriers are back at zero before the closing __syncthreads
    // (tests/test_pingpong_protocol_cpu.py models the sequence: bwd_ops there restates the three turn
    // conditions below - the G2 sync, the G2 arrival and the empty turn - and changes with them).  GEMM1
    // takes no turn: a token per GEMM measured the same step rate with twice the barriers (chosen by step rate,
    // not by the phase clocks).  Only the issue order changes, not the arithmetic.
    const int own = 3 + wg, other = 4 - wg;
    PHASE_BEGIN(wg);
    load(r + cpg * wg);
    for (int tile = r + cpg * wg; tile < a.num_tiles; tile += tstride) {
        PHASE_TILE(wg);
        // ---- stage the tile: x row-major (B of GEMM1) and transposed (B of GEMM2), hi / lo; dz
        tc::named_bar(bar, 128);  // every MMA of the warpgroup that read the previous tile has retired
        PHASE_MARK(wg, 0);
#pragma unroll
        for (int k = 0; k < kLd; ++k) {
            if (k >= ksteps) continue;  // features GEMM1 does not read; GEMM2's columns of them are dropped
            const int c = 2 * k + (lane >> 4);
            float4 hi, lo;
            tc::split4(v[k], hi, lo);
            const uint32_t off = tc::sw128_offset(rr, c);
            *reinterpret_cast<float4*>(x_hi + off) = hi;
            *reinterpret_cast<float4*>(x_lo + off) = lo;
            // batch row rr -> K atom rr / 32, position 8 kk + (qq >> 1) + 4 (qq & 1) with rr % 32 = 8 kk + qq
            const int r32 = rr & 31, pos = (r32 & ~7) + ((r32 & 7) >> 1) + 4 * (r32 & 1);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int f = 4 * c + e;
                const uint32_t toff = (rr >> 5) * (32 * 128) + (f >> 3) * 1024 + (f & 7) * 128 +
                                      (((pos >> 2) ^ (f & 7)) << 4) + (pos & 3) * 4;
                *reinterpret_cast<float*>(xt_hi + toff) = f4(hi, e);
                *reinterpret_cast<float*>(xt_lo + toff) = f4(lo, e);
            }
        }
        if (lt < kRowsT) {
#pragma unroll
            for (int n = 0; n < NP; ++n) dzs[lt * NP + n] = z[n], gb2[n] += z[n];
        }
        tc::fence_proxy_async();
        tc::named_bar(bar, 128);
        PHASE_MARK(wg, 1);

        // ---- GEMM1: PRE = W1_blk * X^T (one m64n64 MMA per product over the tile's 64 batch rows), A
        // from registers; descriptors = the stage's plus the operand's offset in 16-byte units (start
        // address field) (bases opaque per tile: hoisted out of the loop, every descriptor would hold two
        // registers)
        uint64_t bx_hi = dx_hi, bx_lo = dx_lo;
        asm volatile("" : "+l"(bx_hi), "+l"(bx_lo));
        float d[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) d[i] = 0.f;
        // zeroed accumulators defined before the warpgroup fence (see bwd_tc_body)
        tc::fence_acc(d);
        PHASE_GEMM_ON(wg);
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (kk < ksteps) {
                const uint32_t xo = (kk * 32) >> 4;
                tc::wgmma_n64_rs(d, wl[kk], bx_hi + xo, kk > 0);
                tc::wgmma_n64_rs(d, wh[kk], bx_lo + xo, true);
            }
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (kk < ksteps) tc::wgmma_n64_rs(d, wh[kk], bx_hi + ((kk * 32) >> 4), true);
        }
        tc::wgmma_commit();
        // the next tile's loads go out after GEMM1 is issued, not before: their address arithmetic and
        // bounds checks run while the MMAs execute instead of delaying the issue; they are in flight during
        // this tile's MMAs and epilogue
        load(tile + tstride);
        tc::wgmma_wait<0>();
        tc::fence_acc(d);
        PHASE_GEMM_OFF(wg);
        PHASE_MARK(wg, 2);

        // ---- epilogue: d <- DP in place (thread: hidden units j0 / j1, batch columns 8 i + 2 q + e)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int m = 8 * i + 2 * q + e;
                float dz[NP];
                if constexpr (NP == 4) {
                    const float4 t = *reinterpret_cast<const float4*>(dzs + 4 * m);
                    dz[0] = t.x, dz[1] = t.y, dz[2] = t.z, dz[3] = t.w;
                } else {
                    dz[0] = dzs[m];
                }
                // relu'(0) = 0 as in torch
                const float pre0 = d[4 * i + e] + bj0, pre1 = d[4 * i + 2 + e] + bj1;
                const float h0 = fmaxf(pre0, 0.f), h1 = fmaxf(pre1, 0.f);
                float dh0 = dz[0] * w2r0[0], dh1 = dz[0] * w2r1[0];
#pragma unroll
                for (int n = 1; n < NP; ++n) dh0 = fmaf(dz[n], w2r0[n], dh0), dh1 = fmaf(dz[n], w2r1[n], dh1);
#pragma unroll
                for (int n = 0; n < NP; ++n) gw0[n] = fmaf(dz[n], h0, gw0[n]), gw1[n] = fmaf(dz[n], h1, gw1[n]);
                const float dp0 = pre0 > 0.f ? dh0 : 0.f, dp1 = pre1 > 0.f ? dh1 : 0.f;
                gb10 += dp0, gb11 += dp1;
                d[4 * i + e] = dp0, d[4 * i + 2 + e] = dp1;
            }
        }

        // ---- GEMM2: dW1 += DP * X (A = DP from registers).  Phase 1: dp_lo * x_hi; phase 2 (DP
        // overwritten by dp_hi in place): dp_hi * x_lo, then dp_hi * x_hi into its own accumulator
        uint32_t lo[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float hi = __uint_as_float(__float_as_uint(d[i]) & 0xffffe000u);
            lo[i] = __float_as_uint(d[i] - hi);
            d[i] = hi;
        }
        uint64_t bxt_hi = dxt_hi, bxt_lo = dxt_lo;
        asm volatile("" : "+l"(bxt_hi), "+l"(bxt_lo));
        PHASE_MARK(wg, 3);
        tc::named_bar_if(wg == 1 || tile != r, own, 256);  // G2 turn
        PHASE_MARK(wg, 5);
        PHASE_GEMM_ON(wg);
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const uint32_t al[4] = {lo[4 * kk], lo[4 * kk + 2], lo[4 * kk + 1], lo[4 * kk + 3]};
            const uint32_t ah[4] = {__float_as_uint(d[4 * kk]), __float_as_uint(d[4 * kk + 2]),
                                    __float_as_uint(d[4 * kk + 1]), __float_as_uint(d[4 * kk + 3])};
            const uint32_t xo = ((kk >> 2) * 32 * 128 + (kk & 3) * 32) >> 4;
            tc::wgmma_n32_rs(acc_c, al, bxt_hi + xo, true);
            tc::wgmma_n32_rs(acc_c, ah, bxt_lo + xo, true);
            tc::wgmma_n32_rs(acc_hh, ah, bxt_hi + xo, true);
        }
        tc::wgmma_commit();
        tc::named_bar_arrive_if(wg == 0 || tile + cpg < a.num_tiles, other, 256);  // 1: warpgroup 0 has a next tile
        tc::wgmma_wait<0>();
        // the A registers are read asynchronously: keep them (and the accumulators) untouched until here
        tc::fence_acc(d);
#pragma unroll
        for (int i = 0; i < 32; ++i) asm volatile("" : "+r"(lo[i])::"memory");
        tc::fence_acc(acc_hh), tc::fence_acc(acc_c);
        PHASE_GEMM_OFF(wg);
        PHASE_MARK(wg, 4);
    }
    // an odd number of tiles in the CTA (r, r + cpg, ... alternate between the warpgroups): warpgroup 1 has
    // one fewer and takes the empty turn of warpgroup 0's last tile
    if (wg == 1 && (r < a.num_tiles ? (a.num_tiles - 1 - r) / cpg + 1 : 0) % 2 == 1) {
        tc::named_bar(own, 256);
    }

    // ---- end of the launch: the quad's column sets meet, then warpgroup 0 + warpgroup 1 (fixed order)
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
    float gwt[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) gwt[i] = acc_hh[i] + acc_c[i];
    // db2: fixed-order tree over each warp that loaded dz rows, then the 4 warps (below)
#pragma unroll
    for (int n = 0; n < NP; ++n) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) gb2[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gb2[n], off);
    }
    if (lt < kRowsT && lane == 0) {
#pragma unroll
        for (int n = 0; n < NP; ++n) gb2x[(2 * wg + warp) * 4 + n] = gb2[n];
    }
    // warpgroup 1's values -> its stage, laid out by thread (both warpgroups hold the same entries)
    float* xch = reinterpret_cast<float*>(smem + kStageBytes);
    __syncthreads();  // warpgroup 1's last MMAs have retired
    if (wg == 1) {
#pragma unroll
        for (int i = 0; i < 16; ++i) xch[i * 128 + lt] = gwt[i];
        xch[16 * 128 + lt] = gb10, xch[17 * 128 + lt] = gb11;
#pragma unroll
        for (int n = 0; n < NP; ++n) xch[(18 + n) * 128 + lt] = gw0[n], xch[(18 + NP + n) * 128 + lt] = gw1[n];
    }
    __syncthreads();
    if (wg == 0) {
#pragma unroll
        for (int i = 0; i < 16; ++i) gwt[i] += xch[i * 128 + lt];
        gb10 += xch[16 * 128 + lt], gb11 += xch[17 * 128 + lt];
#pragma unroll
        for (int n = 0; n < NP; ++n) gw0[n] += xch[(18 + n) * 128 + lt], gw1[n] += xch[(18 + NP + n) * 128 + lt];
        if (q == 0) {
            wsb[a.lay.ob1 + j0] = gb10;
            wsb[a.lay.ob1 + j1] = gb11;
#pragma unroll
            for (int n = 0; n < NP; ++n)
                if (n < a.N2) wsb[a.lay.oW2 + (size_t)n * H + j0] = gw0[n], wsb[a.lay.oW2 + (size_t)n * H + j1] = gw1[n];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = 8 * i + 2 * q;  // features f, f + 1 (O % 4 == 0: both or neither valid)
            if (f < O) {
                *reinterpret_cast<float2*>(wsb + a.lay.oW1 + (size_t)j0 * O + f) = make_float2(gwt[4 * i], gwt[4 * i + 1]);
                *reinterpret_cast<float2*>(wsb + a.lay.oW1 + (size_t)j1 * O + f) = make_float2(gwt[4 * i + 2], gwt[4 * i + 3]);
            }
        }
        // db2 from group 0 only: its CTAs see every tile once
        if (grp == 0 && tid == 0) {
#pragma unroll
            for (int n = 0; n < NP; ++n)
                if (n < a.N2) wsb[a.lay.ob2 + n] = (gb2x[n] + gb2x[4 + n]) + (gb2x[8 + n] + gb2x[12 + n]);
        }
    }
    __threadfence();  // this thread's partial-row stores are visible device-wide
    __syncthreads();
    PHASE_END(wg);
    return smem;
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

// grid = a multiple of the H / 64 hidden blocks; partial rows = CTAs per block
template <int NP>
__global__ void __launch_bounds__(kThreads, 1) mlp_bwd_tc_kernel(const __grid_constant__ BwdTcArgs a) {
    uint8_t* scratch = bwd_blk_body<NP>(a, blockIdx.x, gridDim.x);
    grid_arrive_and_wait(a.ctl);
    reduce_rows(a, gridDim.x / (a.H / 64), blockIdx.x, gridDim.x, reinterpret_cast<double*>(scratch));
    grid_depart(a.ctl);
}

// Its split-head twin (shared-torso networks, NP = 4 only), a kernel of its own name and arguments
__global__ void __launch_bounds__(kThreads, 1) mlp_bwd_tc_split_kernel(const __grid_constant__ BwdTcSplitArgs a) {
    uint8_t* scratch = bwd_blk_body<4, true>(a, blockIdx.x, gridDim.x);
    grid_arrive_and_wait(a.ctl);
    reduce_rows(a, gridDim.x / (a.H / 64), blockIdx.x, gridDim.x, reinterpret_cast<double*>(scratch));
    grid_depart(a.ctl);
}

// Policy and value network of one learner step in ONE launch: CTAs [0, n_pi) take the policy's
// tiles (partial rows 0 .. n_pi / (H_pi / 64) of its workspace), the rest the value function's.  After
// the grid barrier every CTA helps reduce both sets of rows (the value function's chunks are dealt from
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
    if ((int)blockIdx.x < n_pi) scratch = bwd_blk_body<4>(a_pi, blockIdx.x, n_pi);
    else scratch = bwd_blk_body<1>(a_vf, (int)blockIdx.x - n_pi, n_vf);
    grid_arrive_and_wait(a_pi.ctl);
    const PushArgs* pp = PUSH ? &push : nullptr;
    reduce_rows(a_pi, n_pi / (a_pi.H / 64), blockIdx.x, gridDim.x, reinterpret_cast<double*>(scratch), pp, 0);
    reduce_rows(a_vf, n_vf / (a_vf.H / 64), (int)gridDim.x - 1 - (int)blockIdx.x, gridDim.x,
                reinterpret_cast<double*>(scratch), pp, a_pi.lay.total);
    if (PUSH) {  // the extras, spread over the grid (observation normalization adds 2 O + 1 of them)
        const long long step = *push.seq + 1;
        const int64_t base = (step & 1) * push.buf_stride + (int64_t)push.rank * push.slot_stride + a_pi.lay.total +
                             a_vf.lay.total;
        for (int j = (int)(blockIdx.x * blockDim.x + threadIdx.x); j < n_extra; j += (int)(gridDim.x * blockDim.x)) {
            const double val = extra[j];
            for (int r = 0; r < push.world; ++r) ll_store(push.gather[r] + base + j, val, (unsigned)step);
        }
    }
    grid_depart(a_pi.ctl);
}

// Wide shapes: partial rows only (reduce_partials_kernel sums them)
template <int NP, int KA>
__global__ void __launch_bounds__(kThreads) mlp_bwd_tcw_kernel(const __grid_constant__ BwdTcArgs a) {
    bwd_tc_body<NP, KA>(a, blockIdx.x, gridDim.x);
}

// Its split-head twin (shared-torso networks, NP >= 4 only)
template <int NP, int KA>
__global__ void __launch_bounds__(kThreads) mlp_bwd_tcw_split_kernel(const __grid_constant__ BwdTcSplitArgs a) {
    bwd_tc_body<NP, KA, true>(a, blockIdx.x, gridDim.x);
}

static_assert(kWarps * 64 * sizeof(double) <= 2 * kXAtomBytes, "reduction scratch fits the x stage");

BwdTcArgs make_bwd_args(const float* x, const float* params, const float* dout, float* ws, double* grad,
                        unsigned int* ctl, int M, int O, int H, int N2) {
    BwdTcArgs a{};
    a.x = x, a.params = params, a.dout = dout, a.ws = ws, a.grad = grad, a.ctl = ctl;
    a.M = M, a.O = O, a.H = H, a.N2 = N2;
    a.num_tiles = (M + kRowsT - 1) / kRowsT;
    a.lay = impala_make_layout(O, H, N2);
    return a;
}

// impala_pair_split for networks that take whole sets of CTAs (one per hidden block: ga / gb CTAs):
// *na policy sets and *nb value-function sets, at most `grid` CTAs and no more sets than tiles, so
// that the slower side finishes earliest at per-tile cost wa / wb.  Needs ga + gb <= grid.
void split_sets(int tiles_a, int tiles_b, int grid, int ga, int gb, int64_t wa, int64_t wb, int* na, int* nb) {
    int64_t best_cost = INT64_MAX, best_sum = INT64_MAX;
    *na = *nb = 1;
    for (int sa = 1; sa <= tiles_a && sa * ga + gb <= grid; ++sa) {
        int sb = (grid - sa * ga) / gb;
        if (sb > tiles_b) sb = tiles_b;
        const int64_t ca = (int64_t)((tiles_a + sa - 1) / sa) * wa, cb = (int64_t)((tiles_b + sb - 1) / sb) * wb;
        const int64_t cost = ca > cb ? ca : cb, sum = ca + cb;
        if (cost < best_cost || (cost == best_cost && sum < best_sum)) *na = sa, *nb = sb, best_cost = cost, best_sum = sum;
    }
}

// Persistent grid of a Wide plan's backward: resident CTAs, at most one per tile and kMaxParts.
template <typename Args>
int launch_tcw(void (*kernel)(Args), const MlpPlan& p, const Args& a, cudaStream_t st, int* nparts) {
    const size_t smem = bwd_smem_bytes(p.ka, p.np);
    cudaError_t e;
    int sms = 0, per_sm = 0;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    if ((e = impala_resident_ctas((const void*)kernel, kThreads, smem, &per_sm)) != cudaSuccess) return (int)e;
    if (per_sm < 1) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    int grid = per_sm * sms;
    if (grid > a.num_tiles) grid = a.num_tiles;
    if (grid > kMaxParts) grid = kMaxParts;
    if ((e = impala_launch(kernel, grid, kThreads, smem, st, true, a)) != cudaSuccess) return (int)e;
    *nparts = grid;
    return impala_launch_status();
}

}  // namespace

// Per-CTA partial gradient rows go to ws (same layout as the FP32 kernel), their float64 sum to
// grad; ctl = two zeroed control words (see the grid barrier in the kernel).
int impala_mlp_bwd_tc(const float* x, const float* params, const float* dout, float* ws,
                      double* grad, unsigned int* ctl, int M, int O, int H, int N2, cudaStream_t st,
                      const float* dout_b, int M_a) {
    const BwdTcSplitArgs a{make_bwd_args(x, params, dout, ws, grad, ctl, M, O, H, N2), dout_b, M_a};
    const size_t smem = kBlkSmemBytes;
    cudaError_t e;
    int sms = 0;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    auto kernel = N2 == 1 ? mlp_bwd_tc_kernel<1> : mlp_bwd_tc_kernel<4>;
    const void* kfn = dout_b ? (const void*)mlp_bwd_tc_split_kernel : (const void*)kernel;  // split: N2 >= 2
    int per_sm = 0;  // unused: the cooperative launch fails when the grid cannot be resident
    if ((e = impala_resident_ctas(kfn, kThreads, smem, &per_sm)) != cudaSuccess) return (int)e;
    // every hidden block gets the same number of CTAs, no more than there are tiles (= partial rows the
    // workspace holds); grid <= SM count: the grid barrier needs residency
    const int nblk = H / 64;
    int cpg = (sms < kMaxParts ? sms : kMaxParts) / nblk;
    if (cpg > a.num_tiles) cpg = a.num_tiles;
    if (cpg < 1) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    e = dout_b ? impala_launch_ex(mlp_bwd_tc_split_kernel, nblk * cpg, kThreads, smem, st, true, true, a)
               : impala_launch_ex(kernel, nblk * cpg, kThreads, smem, st, true, true, static_cast<const BwdTcArgs&>(a));
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

// Both networks in one launch; the caller has routed each to a Narrow plan and checked 2 <= A <= 4.
// push != nullptr: data-parallel variant (see mlp_bwd_tc_pair_kernel).
int impala_mlp_bwd_tc_pair(const float* x, const float* params_pi, const float* params_vf,
                           const float* dlogits, const float* dv, float* ws_pi, float* ws_vf,
                           double* grad_pi, double* grad_vf, unsigned int* ctl, int M_pi, int M_vf, int O,
                           int H_pi, int H_vf, int A, cudaStream_t st, const PushArgs* push, const double* extra,
                           int n_extra) {
    const BwdTcArgs a_pi = make_bwd_args(x, params_pi, dlogits, ws_pi, grad_pi, ctl, M_pi, O, H_pi, A);
    const BwdTcArgs a_vf = make_bwd_args(x, params_vf, dv, ws_vf, grad_vf, ctl, M_vf, O, H_vf, 1);
    const size_t smem = kBlkSmemBytes;
    cudaError_t e;
    int sms = 0;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    int per_sm = 0;  // unused: the cooperative launch fails when the grid cannot be resident
    e = impala_resident_ctas(push ? (const void*)mlp_bwd_tc_pair_kernel<true> : (const void*)mlp_bwd_tc_pair_kernel<false>,
                             kThreads, smem, &per_sm);
    if (e != cudaSuccess) return (int)e;
    // a CTA does one hidden block of a tile whatever H is: the per-tile weights do not scale with H.  A
    // policy tile (4-output epilogue) costs about 1.25 value-function tiles (scripts/tune_pair_split.py)
    const int gp = H_pi / 64, gv = H_vf / 64;
    int grid = sms < kMaxParts ? sms : kMaxParts;  // <= SM count: the grid barrier needs residency
    if (grid < gp + gv) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    int sp = 1, sv = 1;
    split_sets(a_pi.num_tiles, a_vf.num_tiles, grid, gp, gv, impala_env_int("IMPALA_PAIR_W_BWD", 125), 100, &sp, &sv);
    grid = gp * sp + gv * sv;
    const int n_pi = gp * sp;
    // cooperative launch: the in-kernel grid barrier needs every CTA resident
    e = push ? impala_launch_ex(mlp_bwd_tc_pair_kernel<true>, grid, kThreads, smem, st, true, true, a_pi, a_vf, n_pi,
                                *push, extra, n_extra)
             : impala_launch_ex(mlp_bwd_tc_pair_kernel<false>, grid, kThreads, smem, st, true, true, a_pi, a_vf, n_pi,
                                PushArgs{}, (const double*)nullptr, 0);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

// Wide plans: per-CTA float32 partial gradient rows into ws (row stride = layout total); *nparts = rows
// written.  At four K atoms (GEMM2 in 64-feature halves) the tiles are 32 rows high.
int impala_mlp_bwd_tcw(const MlpPlan& p, const float* x, const float* params, const float* dout, float* ws, int M,
                       int O, int H, int N2, cudaStream_t st, int* nparts, const float* dout_b, int M_a) {
    BwdTcSplitArgs a{make_bwd_args(x, params, dout, ws, nullptr, nullptr, M, O, H, N2), dout_b, M_a};
    a.num_tiles = (M + p.rows - 1) / p.rows;
    const int np = p.np;
    if (dout_b) {  // split heads: N2 >= 2, so np >= 4
        auto kernel = p.ka == 1   ? (np == 4 ? mlp_bwd_tcw_split_kernel<4, 1> : mlp_bwd_tcw_split_kernel<16, 1>)
                      : p.ka == 2 ? (np == 4 ? mlp_bwd_tcw_split_kernel<4, 2> : mlp_bwd_tcw_split_kernel<16, 2>)
                                  : (np == 4 ? mlp_bwd_tcw_split_kernel<4, 4> : mlp_bwd_tcw_split_kernel<32, 4>);
        return launch_tcw(kernel, p, a, st, nparts);
    }
    auto kernel = p.ka == 1   ? (np == 1 ? mlp_bwd_tcw_kernel<1, 1> : np == 4 ? mlp_bwd_tcw_kernel<4, 1> : mlp_bwd_tcw_kernel<16, 1>)
                  : p.ka == 2 ? (np == 1 ? mlp_bwd_tcw_kernel<1, 2> : np == 4 ? mlp_bwd_tcw_kernel<4, 2> : mlp_bwd_tcw_kernel<16, 2>)
                              : (np == 1 ? mlp_bwd_tcw_kernel<1, 4> : np == 4 ? mlp_bwd_tcw_kernel<4, 4> : mlp_bwd_tcw_kernel<32, 4>);
    return launch_tcw(kernel, p, static_cast<const BwdTcArgs&>(a), st, nparts);
}

#ifdef IMPALA_PHASE_CLOCKS
IMPALA_PHASE_READER(impala_phase_read_bwd)

// The phase counters of the narrow backward body (out[0, kSlots)) and forward body (out[kSlots, 2 kSlots)),
// summed over every launch since the last reset; reset != 0 zeroes them after the copy.  Only in a build
// with IMPALA_PHASE_CLOCKS (scripts/phase_mlp.py).
extern "C" int impala_phase_read(unsigned long long* out, int reset) {
    const int e = impala_phase_read_bwd(out, reset);
    return e ? e : impala_phase_read_fwd(out + phase::kSlots, reset);
}
#endif
