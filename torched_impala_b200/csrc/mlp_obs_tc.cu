// MLP forward and backward on the Hopper tensor cores for wide observations (128 < O <= 1024, O % 4 == 0;
// stacked Atari RAM, flattened MinAtar), error-compensated 3xTF32 like the kernels of mlp_fwd_tc.cu /
// mlp_bwd_tc.cu.  Neither W1 (H x O) nor an x tile fits in shared memory at these widths, so every GEMM
// here STREAMS K in chunks of 32 (one 128-byte swizzle atom):
//
//   forward    OUT[64 rows, 64 hid]   = X[rows, O] * W1_blk[64 hid, O]^T,  K = O         then bias, ReLU, layer 2
//   backward 1 PRE[64 hid, 64 rows]   = W1_blk[64 hid, O] * X[rows, O]^T,   K = O         then DP, db1, dW2, db2
//   backward 2 dW1[64 hid, 64 feat]  += DP^T[64 hid, rows] * X[rows, 64 feat], K = batch rows
//
// One mainloop (kstream) serves all three: a CTA is one warpgroup; its A operand (64 rows of a
// K-contiguous matrix) is loaded from global memory straight into wgmma A fragments (16-byte loads,
// split into tf32 hi / lo in registers), its B operand (64 rows) is staged into a double-buffered,
// 128-byte-swizzled K-major shared-memory stage, K-contiguous (W1 rows, x rows) or transposed from x
// (backward 2).  The loads of chunk c + 1 are in flight while the MMAs of chunk c run.
//
// K order inside a chunk.  K is a sum, so the 32 positions of a chunk may hold its 32 features in any
// order as long as A and B agree.  Thread (g, q) of a warp owns A columns q and q + 4 of every K step;
// it takes features 16 j + 4 q .. + 3 (one 16-byte load per row and j) as (K step 2 j, column q),
// (2 j, q + 4), (2 j + 1, q), (2 j + 1, q + 4), and the B stage puts its features in the same positions.
//
// Numerics.  Every chunk has a FRESH accumulator: lo*hi + hi*lo of its 4 K steps first, hi*hi last
// (the accumulation order of the existing kernels within one chunk, at most 4 full-magnitude additions
// into an accumulator that the tensor core truncates), then it is added into a running fp32 sum in
// registers, round-to-nearest, in chunk order.  DP^T is split round-to-nearest (DESIGN §4: a truncated
// lo would bias the long batch-row reductions towards zero).
//
// Backward 1 writes DP^T [H][Mp] (hidden-major, batch rows contiguous; Mp = tiles x 64) to the
// workspace and per-CTA partial rows of db1 / dW2 / db2; backward 2 reads DP^T and writes per-CTA partial
// rows of dW1.  Each set of partial rows is summed in float64 in fixed order by reduce_partials_kernel
// (mlp.cu), so results are bitwise reproducible.  Every partial entry is written by every launch.
//
// Byte observations (uint8 x, Atari RAM / MinAtar planes).  Every kernel also exists with x as bytes
// (trailing template parameter XT = uint8_t).  An integer in 0..255 is exact in tf32: its split has lo = 0,
// so the MMAs with x_lo as an operand add nothing and are not issued (16 instead of 24 per chunk), x is
// loaded 4 features per 32-bit word and the lo buffer of an x stage is never filled.  The remaining MMAs
// keep their order and the first of a chunk takes over scale-d = 0, so each accumulator sees the same
// non-zero additions in the same order as the float kernels on the same values converted to float.
#include <algorithm>

#include "mlp_fwd_tc.cuh"
#include "tc_common.cuh"

namespace {

constexpr int kT = 128;              // threads per CTA: one warpgroup
constexpr int kBufBytes = 64 * 128;  // one B operand buffer (hi or lo): 64 rows x 32 tf32, swizzled
constexpr int kStageBytes = 4 * kBufBytes;  // [2 buffers][hi | lo]
constexpr int kHBlk = 64;            // hidden units per CTA (A rows in the backward, B rows in the forward)
constexpr int kFBlk = 64;            // features per CTA in backward 2

// A K-contiguous matrix [rows][ld]; entries with row >= rows are zero.
template <typename T>
struct Mat {
    const T* p;
    int64_t ld;
    int rows;
};

// Operand element types.  Raw = 4 consecutive entries as loaded (kept raw while the load is in flight);
// kExact: every value is exact in tf32 (the split's lo is zero).
template <typename T>
struct Elem;
template <>
struct Elem<float> {
    using Raw = float4;
    static constexpr bool kExact = false;
    __device__ static __forceinline__ Raw zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
    __device__ static __forceinline__ Raw load(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
    __device__ static __forceinline__ float4 widen(const Raw& r) { return r; }
};
template <>
struct Elem<uint8_t> {
    using Raw = uint32_t;
    static constexpr bool kExact = true;
    __device__ static __forceinline__ Raw zero() { return 0u; }
    __device__ static __forceinline__ Raw load(const uint8_t* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }
    __device__ static __forceinline__ float4 widen(const Raw& r) {
        return make_float4((float)(r & 255u), (float)((r >> 8) & 255u), (float)((r >> 16) & 255u), (float)(r >> 24));
    }
};

// position of feature k (0..31) of a chunk inside the chunk's 32 K positions (see the header)
__device__ __forceinline__ int kpos(int k) {
    return 16 * (k >> 4) + 8 * ((k & 3) >> 1) + ((k & 15) >> 2) + 4 * (k & 1);
}
__device__ __forceinline__ uint32_t stage_off(int n, int pos) { return tc::sw128_offset(n, pos >> 2) + (pos & 3) * 4; }
__device__ __forceinline__ float f4(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

// run[s][r] += sum over k in [kb, ke) of A[a0 + row(r)][k] * B[b0 + col(s, r)][k], in the accumulator
// layout of two m64n32 slices: row(r) = 16 warp + g + 8 ((r >> 1) & 1), col(s, r) = 32 s + 8 (r >> 2) + 2 q
// + (r & 1).  A entries with k >= ke are zero.  B: BT = false - Bm[b0 + n][k] (k >= ke zero); BT = true -
// Bm[k][b0 + n] (transposed: rows of Bm are K; n >= ncols zero).  kb is a multiple of 32.  The caller
// has a barrier between any earlier use of `stage` and this call; the call ends with one.
// TA / TB: element types of A and B.  An exact operand (bytes) has no lo part: the MMAs that would take
// it are not issued, and for B its lo buffer is left unwritten.
template <bool BT, typename TA, typename TB>
__device__ __forceinline__ void kstream(const Mat<TA>& A, int a0, const Mat<TB>& Bm, int b0, int ncols, int kb,
                                        int ke, uint8_t* stage, float (&run)[2][16]) {
    using EA = Elem<TA>;
    using EB = Elem<TB>;
    constexpr bool kLoA = !EA::kExact, kLoB = !EB::kExact;
    static_assert(kLoA || kLoB, "at most one operand is exact");
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    typename EA::Raw ra[4];           // raw A (row half h, 16-feature group j: ra[2 h + j]) of the next chunk
    typename EB::Raw rb[4];           // raw B of the next chunk
    uint32_t xh[4][4], xl[4][4];      // A fragments of the current chunk: [K step][slot] (xl unused if A is exact)
    auto load = [&](int kc) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int row = a0 + 16 * warp + g + 8 * h, k = kc + 16 * j + 4 * q;
                ra[2 * h + j] = EA::zero();
                if (row < A.rows && k < ke) ra[2 * h + j] = EA::load(A.p + row * A.ld + k);
            }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            rb[t] = EB::zero();
            if constexpr (!BT) {
                // thread -> (row n, 4-feature chunk u): a warp stores 4 rows x 8 chunks, conflict-free
                const int idx = tid + kT * t, n = idx >> 3, k = kc + 4 * (idx & 7);
                if (b0 + n < Bm.rows && k < ke) rb[t] = EB::load(Bm.p + (b0 + n) * Bm.ld + k);
            } else {
                // lane -> K position (batch row), warp -> 4 of the 64 columns: the transposed stores of a
                // warp hit 32 different banks
                const int col = b0 + 4 * (warp + 4 * t), k = kc + lane;
                if (k < Bm.rows && col < ncols) rb[t] = EB::load(Bm.p + k * Bm.ld + col);
            }
        }
    };
    auto stage_b = [&](uint8_t* hi, uint8_t* lo) {
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            float4 vh = EB::widen(rb[t]), vl;
            if constexpr (kLoB) tc::split4(EB::widen(rb[t]), vh, vl);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                uint32_t off;
                if constexpr (!BT) {
                    const int idx = tid + kT * t;
                    off = stage_off(idx >> 3, kpos(4 * (idx & 7) + e));
                } else {
                    off = stage_off(4 * (warp + 4 * t) + e, kpos(lane));
                }
                *reinterpret_cast<float*>(hi + off) = f4(vh, e);
                if constexpr (kLoB) *reinterpret_cast<float*>(lo + off) = f4(vl, e);
            }
        }
    };
    auto split_a = [&]() {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const float4 v = EA::widen(ra[2 * h + j]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float hi = f4(v, e), lo;
                    if constexpr (kLoA) tc::split_tf32(f4(v, e), hi, lo);
                    xh[2 * j + (e >> 1)][h + 2 * (e & 1)] = __float_as_uint(hi);
                    if constexpr (kLoA) xl[2 * j + (e >> 1)][h + 2 * (e & 1)] = __float_as_uint(lo);
                }
            }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            tc::fence_frag(xh[kk]);
            if constexpr (kLoA) tc::fence_frag(xl[kk]);
        }
    };

    const int nch = (ke - kb + 31) >> 5;
    load(kb);
    stage_b(stage, stage + kBufBytes);
    split_a();
    tc::fence_proxy_async();
    __syncthreads();
    for (int c = 0; c < nch; ++c) {
        // all 4 K steps even in a partial last chunk: its features are spread over them (see the header)
        const int kc = kb + 32 * c;
        const uint8_t* bhi = stage + (c & 1) * 2 * kBufBytes;
        uint64_t dh = tc::smem_desc_k_sw128(bhi, 0), dl = tc::smem_desc_k_sw128(bhi + kBufBytes, 0);
        asm volatile("" : "+l"(dh), "+l"(dl));  // opaque bases: no descriptor hoisted per MMA
        float d0[16], d1[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) d0[i] = 0.f, d1[i] = 0.f;
        tc::fence_acc(d0), tc::fence_acc(d1);  // zeroed before the warpgroup fence (see mlp_bwd_tc.cu)
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if constexpr (kLoA) {
                tc::wgmma_n32_rs(d0, xl[kk], dh + ((kk * 32) >> 4), kk > 0);
                tc::wgmma_n32_rs(d1, xl[kk], dh + ((32 * 128 + kk * 32) >> 4), kk > 0);
            }
            if constexpr (kLoB) {  // the first MMA of the chunk when A is exact
                tc::wgmma_n32_rs(d0, xh[kk], dl + ((kk * 32) >> 4), kLoA || kk > 0);
                tc::wgmma_n32_rs(d1, xh[kk], dl + ((32 * 128 + kk * 32) >> 4), kLoA || kk > 0);
            }
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            tc::wgmma_n32_rs(d0, xh[kk], dh + ((kk * 32) >> 4), true);
            tc::wgmma_n32_rs(d1, xh[kk], dh + ((32 * 128 + kk * 32) >> 4), true);
        }
        tc::wgmma_commit();
        if (c + 1 < nch) load(kc + 32);  // in flight during the MMAs
        tc::wgmma_wait<0>();
        tc::fence_acc(d0), tc::fence_acc(d1);
#pragma unroll
        for (int i = 0; i < 16; ++i) run[0][i] += d0[i], run[1][i] += d1[i];
        if (c + 1 < nch) {
            uint8_t* nhi = stage + ((c + 1) & 1) * 2 * kBufBytes;  // last read by chunk c - 1: retired
            stage_b(nhi, nhi + kBufBytes);
            split_a();
            tc::fence_proxy_async();
        }
        __syncthreads();
    }
}

__device__ __forceinline__ uint8_t* aligned_smem() {
    extern __shared__ uint8_t smem_raw[];
    return smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
}

// ------------------------------------------------------------------ forward
// CTA = one 64-row tile; the hidden layer is walked in 64-unit passes, out[row] = ((b2 + z_0) + z_1) + ...
// written by the thread that wrote the previous pass (write_rows).
// x: the observation rows (a.x is not read; it is the same address for XT = float).
template <int NP, typename XT>
__global__ void __launch_bounds__(kT) mlp_fwd_obs_kernel(const __grid_constant__ FwdTcArgs a, const XT* __restrict__ x) {
    constexpr int NPS = w2s_stride(NP);
    uint8_t* stage = aligned_smem();
    float* b1s = reinterpret_cast<float*>(stage + kStageBytes);  // [64]
    float* w2s = b1s + kHBlk;                                     // [64][NPS]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int tile = blockIdx.x;
    const Mat<XT> X{x, a.O, a.M};
    const Mat<float> W1{a.params + a.lay.oW1, a.O, a.H};
    for (int p = 0; p < a.H / kHBlk; ++p) {
        __syncthreads();  // the previous pass's epilogue is done with b1s / w2s
        for (int j = tid; j < kHBlk; j += kT) b1s[j] = __ldg(a.params + a.lay.ob1 + p * kHBlk + j);
        for (int idx = tid; idx < kHBlk * NP; idx += kT) {
            const int j = idx / NP, n = idx - j * NP;
            w2s[j * NPS + n] = n < a.N2 ? __ldg(a.params + a.lay.oW2 + (size_t)n * a.H + p * kHBlk + j) : 0.f;
        }
        float run[2][16] = {};
        kstream<false>(X, tile * kTileM, W1, p * kHBlk, 0, 0, a.O, stage, run);
        float p0[NP], p1[NP];
#pragma unroll
        for (int n = 0; n < NP; ++n) p0[n] = 0.f, p1[n] = 0.f;
        slice_epilogue<NP>(run[0], 0, q, b1s, w2s, p0, p1);
        slice_epilogue<NP>(run[1], 1, q, b1s, w2s, p0, p1);
        write_rows<NP>(a, p, tile, warp, g, q, p0, p1);
    }
}

// Its split-head twin (shared-torso networks, NP >= 4 only): the same body with the split-head write_rows, as a
// kernel of its own name and arguments.  The body is repeated, not shared through a device function: with the
// body in one, ptxas scheduled the dense kernel differently (other registers and instruction order).
template <int NP, typename XT>
__global__ void __launch_bounds__(kT) mlp_fwd_obs_split_kernel(const __grid_constant__ FwdTcSplitArgs a,
                                                               const XT* __restrict__ x) {
    constexpr int NPS = w2s_stride(NP);
    uint8_t* stage = aligned_smem();
    float* b1s = reinterpret_cast<float*>(stage + kStageBytes);  // [64]
    float* w2s = b1s + kHBlk;                                     // [64][NPS]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int tile = blockIdx.x;
    const Mat<XT> X{x, a.O, a.M};
    const Mat<float> W1{a.params + a.lay.oW1, a.O, a.H};
    for (int p = 0; p < a.H / kHBlk; ++p) {
        __syncthreads();  // the previous pass's epilogue is done with b1s / w2s
        for (int j = tid; j < kHBlk; j += kT) b1s[j] = __ldg(a.params + a.lay.ob1 + p * kHBlk + j);
        for (int idx = tid; idx < kHBlk * NP; idx += kT) {
            const int j = idx / NP, n = idx - j * NP;
            w2s[j * NPS + n] = n < a.N2 ? __ldg(a.params + a.lay.oW2 + (size_t)n * a.H + p * kHBlk + j) : 0.f;
        }
        float run[2][16] = {};
        kstream<false>(X, tile * kTileM, W1, p * kHBlk, 0, 0, a.O, stage, run);
        float p0[NP], p1[NP];
#pragma unroll
        for (int n = 0; n < NP; ++n) p0[n] = 0.f, p1[n] = 0.f;
        slice_epilogue<NP>(run[0], 0, q, b1s, w2s, p0, p1);
        slice_epilogue<NP>(run[1], 1, q, b1s, w2s, p0, p1);
        write_rows<NP, true>(a, p, tile, warp, g, q, p0, p1);
    }
}

// ------------------------------------------------------------------ backward
struct ObsBwdArgs {
    const void* x;  // float or uint8_t rows (the kernels' XT)
    const float* params;
    const float* dout;
    float* dpt;     // DP^T [H][mp]
    float* ws_r;    // partial rows [r1][lay.total - lay.ob1]: entries [ob1, total) (db1, dW2, db2, pads)
    float* ws_w;    // partial rows [p2][lay.ob1]: entries [0, ob1) (dW1, pads)
    int M, O, H, N2, num_tiles, mp, r1, p2;
    MlpLayout lay;
    const float* dout_b;  // SPLIT kernels: dout is head a, dout_b head b (split_dz)
    int M_a;
};

// Backward 1: CTA (r, blk) recomputes PRE of hidden block blk for tiles r, r + r1, ... and runs the
// CUDA-core epilogue on the accumulator (the thread's hidden units j0 = 16 warp + g and j0 + 8 of the
// block, 16 batch rows): h = relu(PRE + b1), dh = W2^T dz, dW2 += dz h, DP = PRE + b1 > 0 ? dh : 0,
// db1 += DP; DP goes to DP^T.  dW2 / db1 of the block (and db2 and the pads: blk 0) go to partial row r.
// NP = 32: dW2 in chunks of 8 outputs that the quad sums and lane q keeps (as bwd_tc_body).
template <int NP, typename XT, bool SPLIT = false>
__device__ __forceinline__ void bwd_obs_pre_body(const ObsBwdArgs& a) {
    constexpr bool L2S = NP > 4;
    constexpr int NPS = w2s_stride(NP);
    uint8_t* stage = aligned_smem();
    float* dzs = reinterpret_cast<float*>(stage + kStageBytes);  // [64 rows][NPS]
    float* w2s = dzs + kTileM * NPS;                              // [64 hidden][NPS]
    float* gb2x = w2s + kHBlk * NPS;                              // [4 warps][32]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int r = blockIdx.x, blk = blockIdx.y, H = a.H;
    const int64_t nr = a.lay.total - a.lay.ob1;
    float* wsr = a.ws_r + (size_t)r * nr;
    auto wsb = [&](int64_t e) -> float& { return wsr[e - a.lay.ob1]; };  // layout entry e >= ob1
    const float* __restrict__ W2 = a.params + a.lay.oW2;

    if (blk == 0) {
        const int64_t lo3[3] = {a.lay.ob1 + H, a.lay.oW2 + (int64_t)a.N2 * H, a.lay.ob2 + a.N2};
        const int64_t hi3[3] = {a.lay.oW2, a.lay.ob2, a.lay.total};
        for (int s = 0; s < 3; ++s)
            for (int64_t e = lo3[s] + tid; e < hi3[s]; e += kT) wsb(e) = 0.f;
    }
    for (int idx = tid; idx < kHBlk * NP; idx += kT) {
        const int j = idx / NP, n = idx - j * NP;
        w2s[j * NPS + n] = n < a.N2 ? __ldg(W2 + (size_t)n * H + blk * kHBlk + j) : 0.f;
    }
    const int j0 = blk * kHBlk + 16 * warp + g, j1 = j0 + 8;
    const float bj0 = __ldg(a.params + a.lay.ob1 + j0), bj1 = __ldg(a.params + a.lay.ob1 + j1);
    const float* w2a = w2s + (16 * warp + g) * NPS;  // W2 column of j0 (row of w2s)
    const float* w2b = w2a + 8 * NPS;
    constexpr int NG = L2S ? 8 : NP;
    float gw0[NG], gw1[NG], gb10 = 0.f, gb11 = 0.f, gb2 = 0.f;  // gb2: output tid % NP of this thread's dz entries
#pragma unroll
    for (int n = 0; n < NG; ++n) gw0[n] = gw1[n] = 0.f;

    const Mat<float> W1{a.params + a.lay.oW1, a.O, H};
    const Mat<XT> X{static_cast<const XT*>(a.x), a.O, a.M};
    for (int tile = r; tile < a.num_tiles; tile += a.r1) {
        __syncthreads();  // the previous tile's epilogue is done with dzs
        for (int idx = tid; idx < kTileM * NP; idx += kT) {
            const int m = idx / NP, n = idx - m * NP, row = tile * kTileM + m;
            float z;
            if constexpr (SPLIT) z = row < a.M && n < a.N2 ? split_dz(a.dout, a.dout_b, a.M_a, a.N2, row, n) : 0.f;
            else z = row < a.M && n < a.N2 ? __ldg(a.dout + (size_t)row * a.N2 + n) : 0.f;
            dzs[m * NPS + n] = z;
            gb2 += z;
        }
        float run[2][16] = {};
        kstream<false>(W1, blk * kHBlk, X, tile * kTileM, 0, 0, a.O, stage, run);

        if constexpr (L2S) {
#pragma unroll 1
            for (int cc = 0; cc < 4; ++cc) {
                float s0[8], s1[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) s0[k] = s1[k] = 0.f;
#pragma unroll
                for (int s = 0; s < 2; ++s)
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int m = 32 * s + 8 * i + 2 * q + e;
                            const float h0 = fmaxf(run[s][4 * i + e] + bj0, 0.f);
                            const float h1 = fmaxf(run[s][4 * i + 2 + e] + bj1, 0.f);
                            const float4 za = *reinterpret_cast<const float4*>(dzs + m * NPS + 8 * cc);
                            const float4 zb = *reinterpret_cast<const float4*>(dzs + m * NPS + 8 * cc + 4);
#pragma unroll
                            for (int k = 0; k < 8; ++k) {
                                const float zk = k < 4 ? f4(za, k) : f4(zb, k - 4);
                                s0[k] = fmaf(zk, h0, s0[k]), s1[k] = fmaf(zk, h1, s1[k]);
                            }
                        }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    s0[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s0[k], 1);
                    s1[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s1[k], 1);
                    s0[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s0[k], 2);
                    s1[k] += __shfl_xor_sync(IMPALA_FULL_MASK, s1[k], 2);
                }
                if (q == cc) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) gw0[k] += s0[k], gw1[k] += s1[k];
                }
            }
        }
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int m = 32 * s + 8 * i + 2 * q + e;
                    const float pre0 = run[s][4 * i + e] + bj0, pre1 = run[s][4 * i + 2 + e] + bj1;
                    float dh0 = 0.f, dh1 = 0.f;
                    if constexpr (NP % 4 == 0) {
#pragma unroll
                        for (int n = 0; n < NP; n += 4) {
                            const float4 zv = *reinterpret_cast<const float4*>(dzs + m * NPS + n);
                            const float4 wa = *reinterpret_cast<const float4*>(w2a + n);
                            const float4 wb = *reinterpret_cast<const float4*>(w2b + n);
                            dh0 = fmaf(zv.x, wa.x, dh0), dh0 = fmaf(zv.y, wa.y, dh0);
                            dh0 = fmaf(zv.z, wa.z, dh0), dh0 = fmaf(zv.w, wa.w, dh0);
                            dh1 = fmaf(zv.x, wb.x, dh1), dh1 = fmaf(zv.y, wb.y, dh1);
                            dh1 = fmaf(zv.z, wb.z, dh1), dh1 = fmaf(zv.w, wb.w, dh1);
                            if constexpr (!L2S) {
                                const float h0 = fmaxf(pre0, 0.f), h1 = fmaxf(pre1, 0.f);
#pragma unroll
                                for (int k = 0; k < 4; ++k)
                                    gw0[n + k] = fmaf(f4(zv, k), h0, gw0[n + k]), gw1[n + k] = fmaf(f4(zv, k), h1, gw1[n + k]);
                            }
                        }
                    } else {
                        const float z = dzs[m];
                        dh0 = z * w2a[0], dh1 = z * w2b[0];
                        gw0[0] = fmaf(z, fmaxf(pre0, 0.f), gw0[0]), gw1[0] = fmaf(z, fmaxf(pre1, 0.f), gw1[0]);
                    }
                    // relu'(0) = 0 as in torch
                    const float dp0 = pre0 > 0.f ? dh0 : 0.f, dp1 = pre1 > 0.f ? dh1 : 0.f;
                    gb10 += dp0, gb11 += dp1;
                    run[s][4 * i + e] = dp0, run[s][4 * i + 2 + e] = dp1;
                }
        // DP^T rows j0 / j1, batch columns 32 s + 8 i + 2 q, + 1
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const size_t col = (size_t)tile * kTileM + 32 * s + 8 * i + 2 * q;
                *reinterpret_cast<float2*>(a.dpt + (size_t)j0 * a.mp + col) = make_float2(run[s][4 * i], run[s][4 * i + 1]);
                *reinterpret_cast<float2*>(a.dpt + (size_t)j1 * a.mp + col) = make_float2(run[s][4 * i + 2], run[s][4 * i + 3]);
            }
    }

    // the quad's column sets meet (fixed order)
#pragma unroll
    for (int s = 1; s <= 2; s <<= 1) {
        gb10 += __shfl_xor_sync(IMPALA_FULL_MASK, gb10, s);
        gb11 += __shfl_xor_sync(IMPALA_FULL_MASK, gb11, s);
        if constexpr (!L2S) {
#pragma unroll
            for (int n = 0; n < NP; ++n) {
                gw0[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gw0[n], s);
                gw1[n] += __shfl_xor_sync(IMPALA_FULL_MASK, gw1[n], s);
            }
        }
    }
    if (q == 0) {
        wsb(a.lay.ob1 + j0) = gb10, wsb(a.lay.ob1 + j1) = gb11;
        if constexpr (!L2S) {
#pragma unroll
            for (int n = 0; n < NP; ++n)
                if (n < a.N2) wsb(a.lay.oW2 + (size_t)n * H + j0) = gw0[n], wsb(a.lay.oW2 + (size_t)n * H + j1) = gw1[n];
        }
    }
    if constexpr (L2S) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int n = 8 * q + k;
            if (n < a.N2) wsb(a.lay.oW2 + (size_t)n * H + j0) = gw0[k], wsb(a.lay.oW2 + (size_t)n * H + j1) = gw1[k];
        }
    }
    if (blk == 0) {
        // db2: thread t summed output t % NP; lanes of equal t % NP meet, then the 4 warps (fixed order)
#pragma unroll
        for (int off = NP; off < 32; off <<= 1) gb2 += __shfl_xor_sync(IMPALA_FULL_MASK, gb2, off);
        if (lane < NP) gb2x[warp * 32 + lane] = gb2;
        __syncthreads();
        if (tid < a.N2) wsb(a.lay.ob2 + tid) = ((gb2x[tid] + gb2x[32 + tid]) + gb2x[64 + tid]) + gb2x[96 + tid];
    }
}

template <int NP, typename XT>
__global__ void __launch_bounds__(kT) mlp_bwd_obs_pre_kernel(const __grid_constant__ ObsBwdArgs a) {
    bwd_obs_pre_body<NP, XT>(a);
}

// Its split-head twin (shared-torso networks, NP >= 4 only)
template <int NP, typename XT>
__global__ void __launch_bounds__(kT) mlp_bwd_obs_pre_split_kernel(const __grid_constant__ ObsBwdArgs a) {
    bwd_obs_pre_body<NP, XT, true>(a);
}

// Backward 2: CTA (r, fb, hb) forms dW1 of hidden block hb x feature block fb over the batch-row chunks
// [r nc / p2, (r + 1) nc / p2) (nc = mp / 32) and writes it (and, CTA (r, 0, 0), the W1 pads) to
// partial row r.
template <typename XT>
__global__ void __launch_bounds__(kT) mlp_bwd_obs_dw1_kernel(const __grid_constant__ ObsBwdArgs a) {
    uint8_t* stage = aligned_smem();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int r = blockIdx.x, fb = blockIdx.y, hb = blockIdx.z, O = a.O;
    float* wsb = a.ws_w + (size_t)r * a.lay.ob1;
    if (fb == 0 && hb == 0)
        for (int64_t e = (int64_t)a.H * O + tid; e < a.lay.ob1; e += kT) wsb[e] = 0.f;
    const int nc = a.mp / 32;
    const int c0 = (int)((int64_t)r * nc / a.p2), c1 = (int)((int64_t)(r + 1) * nc / a.p2);
    const Mat<float> DPt{a.dpt, a.mp, a.H};
    const Mat<XT> X{static_cast<const XT*>(a.x), O, a.M};
    float run[2][16] = {};
    kstream<true>(DPt, hb * kHBlk, X, fb * kFBlk, O, 32 * c0, 32 * c1, stage, run);
    const int j0 = hb * kHBlk + 16 * warp + g, j1 = j0 + 8;
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = fb * kFBlk + 32 * s + 8 * i + 2 * q;  // features f, f + 1 (O % 4 == 0: both or neither)
            if (f < O) {
                *reinterpret_cast<float2*>(wsb + (size_t)j0 * O + f) = make_float2(run[s][4 * i], run[s][4 * i + 1]);
                *reinterpret_cast<float2*>(wsb + (size_t)j1 * O + f) = make_float2(run[s][4 * i + 2], run[s][4 * i + 3]);
            }
        }
}

constexpr size_t kFwdSmem(int np) { return 1024 + kStageBytes + (size_t)kHBlk * (1 + w2s_stride(np)) * sizeof(float); }
constexpr size_t kPreSmem(int np) {
    return 1024 + kStageBytes + (size_t)(kTileM + kHBlk) * w2s_stride(np) * sizeof(float) + 4 * 32 * sizeof(float);
}
constexpr size_t kDw1Smem = 1024 + kStageBytes;

template <typename... KArgs, typename... Args>
int launch(void (*kernel)(KArgs...), dim3 grid, size_t smem, cudaStream_t st, Args&&... args) {
    int per_sm = 0;  // unused: the grid is one CTA per tile / block whatever the residency
    if (const cudaError_t e = impala_resident_ctas((const void*)kernel, kT, smem, &per_sm); e != cudaSuccess)
        return (int)e;
    kernel<<<grid, kT, smem, st>>>(static_cast<Args&&>(args)...);
    return impala_launch_status();
}

template <typename XT>
int fwd_obs(const MlpPlan& p, const XT* x, const float* params, float* out, int M, int O, int H, int N2,
            cudaStream_t st, float* out_b, int M_a) {
    FwdTcSplitArgs a{};
    a.x = sizeof(XT) == 4 ? reinterpret_cast<const float*>(x) : nullptr, a.params = params, a.out = out;
    a.M = M, a.O = O, a.H = H, a.N2 = N2;
    a.num_tiles = (M + kTileM - 1) / kTileM;
    a.hb = kHBlk;
    a.lay = impala_make_layout(O, H, N2);
    a.out_b = out_b, a.M_a = M_a;
    const dim3 grid(a.num_tiles);
    if (out_b)  // split heads: N2 >= 2, so np >= 4
        return p.np == 4 ? launch(mlp_fwd_obs_split_kernel<4, XT>, grid, kFwdSmem(4), st, a, x)
                         : launch(mlp_fwd_obs_split_kernel<32, XT>, grid, kFwdSmem(32), st, a, x);
    switch (p.np) {
        case 1: return launch(mlp_fwd_obs_kernel<1, XT>, grid, kFwdSmem(1), st, static_cast<const FwdTcArgs&>(a), x);
        case 4: return launch(mlp_fwd_obs_kernel<4, XT>, grid, kFwdSmem(4), st, static_cast<const FwdTcArgs&>(a), x);
        default: return launch(mlp_fwd_obs_kernel<32, XT>, grid, kFwdSmem(32), st, static_cast<const FwdTcArgs&>(a), x);
    }
}

template <typename XT>
int bwd_obs(const MlpPlan& p, const XT* x, const float* params, const float* dout, void* ws, const ObsBwdLayout& L,
            int M, int O, int H, int N2, cudaStream_t st, const float* dout_b, int M_a) {
    ObsBwdArgs a{};
    a.x = x, a.params = params, a.dout = dout;
    a.dpt = reinterpret_cast<float*>(static_cast<char*>(ws) + L.dpt_off);
    a.ws_r = reinterpret_cast<float*>(static_cast<char*>(ws) + L.rest_off);
    a.ws_w = reinterpret_cast<float*>(static_cast<char*>(ws) + L.w1_off);
    a.M = M, a.O = O, a.H = H, a.N2 = N2;
    a.num_tiles = (M + kTileM - 1) / kTileM;
    a.mp = L.mp, a.r1 = L.r1, a.p2 = L.p2;
    a.lay = impala_make_layout(O, H, N2);
    a.dout_b = dout_b, a.M_a = M_a;
    const dim3 g1(L.r1, H / kHBlk);
    int rc;
    if (dout_b)  // split heads: N2 >= 2, so np >= 4
        rc = p.np == 4 ? launch(mlp_bwd_obs_pre_split_kernel<4, XT>, g1, kPreSmem(4), st, a)
                       : launch(mlp_bwd_obs_pre_split_kernel<32, XT>, g1, kPreSmem(32), st, a);
    else switch (p.np) {
        case 1: rc = launch(mlp_bwd_obs_pre_kernel<1, XT>, g1, kPreSmem(1), st, a); break;
        case 4: rc = launch(mlp_bwd_obs_pre_kernel<4, XT>, g1, kPreSmem(4), st, a); break;
        default: rc = launch(mlp_bwd_obs_pre_kernel<32, XT>, g1, kPreSmem(32), st, a); break;
    }
    if (rc != IMPALA_OK) return rc;
    return launch(mlp_bwd_obs_dw1_kernel<XT>, dim3(L.p2, (O + kFBlk - 1) / kFBlk, H / kHBlk), kDw1Smem, st, a);
}

}  // namespace

int impala_mlp_fwd_obs(const MlpPlan& p, const float* x, const float* params, float* out, int M, int O, int H, int N2,
                       cudaStream_t st, float* out_b, int M_a) {
    return fwd_obs(p, x, params, out, M, O, H, N2, st, out_b, M_a);
}
int impala_mlp_fwd_obs(const MlpPlan& p, const uint8_t* x, const float* params, float* out, int M, int O, int H,
                       int N2, cudaStream_t st, float* out_b, int M_a) {
    return fwd_obs(p, x, params, out, M, O, H, N2, st, out_b, M_a);
}

// Workspace past the control header: DP^T [H][mp] | r1 partial rows of [ob1, total) | p2 partial rows of
// [0, ob1), each region 256-byte aligned.  r1 (backward-1 CTAs per hidden block) and p2 (batch-row ranges
// of backward 2) depend on the shape only: about 512 CTAs per phase, so the partial rows stay small next
// to DP^T.
ObsBwdLayout impala_mlp_obs_bwd_layout(int M, int O, int H, int N2) {
    ObsBwdLayout L;
    const MlpLayout lay = impala_make_layout(O, H, N2);
    const int tiles = (M + kTileM - 1) / kTileM, nblk = H / kHBlk, nfb = (O + kFBlk - 1) / kFBlk;
    const int nc = tiles * kTileM / 32;
    L.mp = tiles * kTileM;
    L.r1 = std::min(tiles, (512 + nblk - 1) / nblk);
    L.p2 = std::min(nc, std::max(1, 512 / (nblk * nfb)));
    L.dpt_off = 0;
    L.rest_off = impala_round_up((int64_t)H * L.mp * (int64_t)sizeof(float), 256);
    L.w1_off = L.rest_off + impala_round_up((int64_t)L.r1 * (lay.total - lay.ob1) * (int64_t)sizeof(float), 256);
    L.bytes = L.w1_off + (int64_t)L.p2 * lay.ob1 * (int64_t)sizeof(float);
    return L;
}

int impala_mlp_bwd_obs(const MlpPlan& p, const float* x, const float* params, const float* dout, void* ws,
                       const ObsBwdLayout& L, int M, int O, int H, int N2, cudaStream_t st, const float* dout_b,
                       int M_a) {
    return bwd_obs(p, x, params, dout, ws, L, M, O, H, N2, st, dout_b, M_a);
}
int impala_mlp_bwd_obs(const MlpPlan& p, const uint8_t* x, const float* params, const float* dout, void* ws,
                       const ObsBwdLayout& L, int M, int O, int H, int N2, cudaStream_t st, const float* dout_b,
                       int M_a) {
    return bwd_obs(p, x, params, dout, ws, L, M, O, H, N2, st, dout_b, M_a);
}
