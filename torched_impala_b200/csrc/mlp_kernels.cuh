// Kernel templates of the FP32 MLP forward / backward (see mlp.cu for the design notes).
// Included by mlp_inst.cu, which is compiled once per padded observation width
// (-DIMPALA_OP=..) and direction (-DIMPALA_BWD=0/1) so the instantiations build in parallel.
#pragma once

#include <type_traits>

#include "common.cuh"

struct MlpArgs {
    const float* x;
    const float* params;
    const float* dout;
    float* out;
    float* ws;
    int M, O, H, N2;
    int num_tiles;
    MlpLayout lay;
};

// The arguments of the FP32 split-head twins (SPLIT kernels): out / dout is head a, out_b / dout_b head b (see
// split_out).  A struct of its own, so the kernels of the interleaved layout keep their parameter space.
struct MlpSplitArgs : MlpArgs {
    float* out_b;
    const float* dout_b;
    int M_a;
};
template <bool SPLIT>
using MlpArgsT = std::conditional_t<SPLIT, MlpSplitArgs, MlpArgs>;

// Split heads of a shared-torso network (impala_mlp_forward_shared / impala_mlp_backward_shared): the
// N2 = N + 1 outputs of M rows are head a, columns [0, N) of rows [0, M_a) at `a` (row stride N), and head b,
// column N of every row at `b` (stride 1).  Rows >= M_a of head a are not written and read as 0.  The
// kernels take this as a compile-time SPLIT flag, instantiated for N2 >= 2 only; SPLIT = false is the
// interleaved (M, N2) layout, unchanged.
__device__ __forceinline__ float* split_out(float* a, float* b, int M_a, int N2, int row, int n) {
    return n == N2 - 1 ? b + row : row < M_a ? a + (size_t)row * (N2 - 1) + n : nullptr;
}
__device__ __forceinline__ float split_dz(const float* a, const float* b, int M_a, int N2, int row, int n) {
    return n == N2 - 1 ? __ldg(b + row) : row < M_a ? __ldg(a + (size_t)row * (N2 - 1) + n) : 0.f;
}

struct MlpConfig {
    int jpt, maxt, op, np, threads, slices;
    int ks;  // backward: threads per hidden unit (2 / 4 = the observation features are split over a lane pair / quad)
};

constexpr int kRows = 32;        // rows per staged tile
constexpr int kGroup = 8;        // rows per register block
constexpr int kMaxParts = 1024;  // upper bound on persistent CTAs (= per-CTA partials)

// Defined in mlp.cu: caches occupancy per (kernel, device, block, smem) and launches a
// persistent grid of min(tiles, resident CTAs) x slices blocks.
int impala_mlp_launch(void (*kernel)(MlpArgs), const MlpArgs& a, const MlpConfig& c, size_t smem,
                      cudaStream_t st, int* grid_out);
int impala_mlp_launch(void (*kernel)(MlpSplitArgs), const MlpSplitArgs& a, const MlpConfig& c, size_t smem,
                      cudaStream_t st, int* grid_out);

// Which kernels run one MLP call: decided by the route in mlp.cu, carried out by the launchers below.
enum class MlpKernel {
    Fp32,    // FP32 CUDA-core kernels (mlp_kernels.cuh / mlp_inst.cu), configuration `fp32`
    Narrow,  // tensor-core block kernels: forward mlp_fwd_tc_kernel<NP, 1>, backward mlp_bwd_tc_kernel<NP>
    Wide,    // tensor-core pass kernels: mlp_fwd_tc_kernel<NP, KA>, mlp_bwd_tcw_kernel<NP, KA>
    Obs,     // K-streamed tensor-core kernels for O > 128 (mlp_obs_tc.cu)
};
struct MlpPlan {
    MlpKernel kernel;
    int np, ka;             // template parameters <NP, KA> (padded outputs, 32-feature K atoms)
    int hb;                 // forward: hidden units per pass
    int rows;               // backward: batch rows per tile
    bool reduce_in_kernel;  // backward: the kernel sums its partial rows into grad itself
    int64_t ws;             // backward: workspace bytes the call needs
    MlpConfig fp32;         // the FP32 kernels' configuration (backward: always, it sizes the workspace)
};

// Tensor-core (wgmma, 3xTF32) forward of the Narrow and Wide plans, defined in mlp_fwd_tc.cu.
// out_b != nullptr: split heads (out = head a, out_b = head b, see split_out), the SPLIT kernels.
int impala_mlp_fwd_tc(const MlpPlan& p, const float* x, const float* params, float* out, int M, int O, int H, int N2,
                      cudaStream_t st, float* out_b = nullptr, int M_a = 0);

// Policy + value network in one launch (CTA ranges per network); A in 2..4, both nets on Narrow plans.
int impala_mlp_fwd_tc_pair(const float* x, const float* params_pi, const float* params_vf, float* logits,
                           float* values, int M_pi, int M_vf, int O, int H_pi, int H_vf, int A,
                           cudaStream_t st);

// Tensor-core backward of a Narrow plan (mlp_bwd_tc.cu): per-CTA partial rows into ws, reduced in-kernel to grad.
// dout_b != nullptr (here and below): split heads (dout = head a, dout_b = head b, see split_dz).
int impala_mlp_bwd_tc(const float* x, const float* params, const float* dout, float* ws,
                      double* grad, unsigned int* ctl, int M, int O, int H, int N2, cudaStream_t st,
                      const float* dout_b = nullptr, int M_a = 0);

int impala_mlp_bwd_tc_pair(const float* x, const float* params_pi, const float* params_vf,
                           const float* dlogits, const float* dv, float* ws_pi, float* ws_vf,
                           double* grad_pi, double* grad_vf, unsigned int* ctl, int M_pi, int M_vf, int O,
                           int H_pi, int H_vf, int A, cudaStream_t st, const PushArgs* push = nullptr,
                           const double* extra = nullptr, int n_extra = 0);

// Tensor-core backward of a Wide plan (mlp_bwd_tc.cu): *nparts float32 partial rows in ws for
// reduce_partials_kernel.
int impala_mlp_bwd_tcw(const MlpPlan& p, const float* x, const float* params, const float* dout, float* ws, int M,
                       int O, int H, int N2, cudaStream_t st, int* nparts, const float* dout_b = nullptr,
                       int M_a = 0);

// Obs plans (mlp_obs_tc.cu): 128 < O <= 1024, K streamed.  Byte observations (values 0..255) enter the
// network as they are.
int impala_mlp_fwd_obs(const MlpPlan& p, const float* x, const float* params, float* out, int M, int O, int H, int N2,
                       cudaStream_t st, float* out_b = nullptr, int M_a = 0);
int impala_mlp_fwd_obs(const MlpPlan& p, const uint8_t* x, const float* params, float* out, int M, int O, int H,
                       int N2, cudaStream_t st, float* out_b = nullptr, int M_a = 0);
// Backward workspace past the control header: byte offsets of DP^T and of the two sets of float32 partial
// rows (r1 rows of layout entries [ob1, total), p2 rows of [0, ob1)) for reduce_partials_kernel.
struct ObsBwdLayout {
    int64_t dpt_off, rest_off, w1_off, bytes;
    int mp, r1, p2;
};
ObsBwdLayout impala_mlp_obs_bwd_layout(int M, int O, int H, int N2);
int impala_mlp_bwd_obs(const MlpPlan& p, const float* x, const float* params, const float* dout, void* ws,
                       const ObsBwdLayout& L, int M, int O, int H, int N2, cudaStream_t st,
                       const float* dout_b = nullptr, int M_a = 0);
int impala_mlp_bwd_obs(const MlpPlan& p, const uint8_t* x, const float* params, const float* dout, void* ws,
                       const ObsBwdLayout& L, int M, int O, int H, int N2, cudaStream_t st,
                       const float* dout_b = nullptr, int M_a = 0);

// One per padded observation width / direction, defined in mlp_inst.cu; out_b / dout_b != nullptr selects the
// split-head twin.
#define IMPALA_DECL_DISPATCH(OPV)                                                             \
    int impala_mlp_fwd_op##OPV(const MlpSplitArgs&, const MlpConfig&, size_t, cudaStream_t, int*); \
    int impala_mlp_bwd_op##OPV(const MlpSplitArgs&, const MlpConfig&, size_t, cudaStream_t, int*);
IMPALA_DECL_DISPATCH(8)
IMPALA_DECL_DISPATCH(24)
IMPALA_DECL_DISPATCH(32)
IMPALA_DECL_DISPATCH(64)
IMPALA_DECL_DISPATCH(128)

namespace impala_mlp {

template <int R, int OP>
__device__ __forceinline__ void stage_x(float* xs, const float* __restrict__ x, int row0, int M,
                                        int O) {
    for (int idx = threadIdx.x; idx < R * OP; idx += blockDim.x) {
        const int r = idx / OP, k = idx - r * OP;
        const int row = row0 + r;
        xs[idx] = (row < M && k < O) ? __ldg(x + (size_t)row * O + k) : 0.f;
    }
}

// W1 rows of this thread's hidden units, kept in registers for the CTA's lifetime.
template <int JPT, int OP>
__device__ __forceinline__ void load_w1(float (&w)[JPT][OP], const float* __restrict__ W1, int j0,
                                        int jstride, int H, int O) {
#pragma unroll
    for (int q = 0; q < JPT; ++q) {
        const int j = j0 + q * jstride;
#pragma unroll
        for (int k = 0; k < OP; ++k) w[q][k] = (j < H && k < O) ? __ldg(W1 + (size_t)j * O + k) : 0.f;
    }
}

// acc[q][r] = b1[j_q] + sum_k W1[j_q][k] * x[r][k] for the kGroup rows at xg
template <int JPT, int OP>
__device__ __forceinline__ void layer1(float (&acc)[JPT][kGroup], const float (&w)[JPT][OP],
                                       const float* xg, const float (&b1r)[JPT]) {
#pragma unroll
    for (int q = 0; q < JPT; ++q)
#pragma unroll
        for (int r = 0; r < kGroup; ++r) acc[q][r] = b1r[q];
#pragma unroll
    for (int k4 = 0; k4 < OP / 4; ++k4) {
#pragma unroll
        for (int r = 0; r < kGroup; ++r) {
            const float4 xv = *reinterpret_cast<const float4*>(xg + r * OP + 4 * k4);  // broadcast
#pragma unroll
            for (int q = 0; q < JPT; ++q) {
                acc[q][r] = fmaf(w[q][4 * k4 + 0], xv.x, acc[q][r]);
                acc[q][r] = fmaf(w[q][4 * k4 + 1], xv.y, acc[q][r]);
                acc[q][r] = fmaf(w[q][4 * k4 + 2], xv.z, acc[q][r]);
                acc[q][r] = fmaf(w[q][4 * k4 + 3], xv.w, acc[q][r]);
            }
        }
    }
}

// p ? x : y as an opaque selp: the plain select of two elements of the butterfly's value array is turned
// into a dynamically indexed load by the compiler, which sends the array to local memory.
__device__ __forceinline__ float selp_f32(bool p, float x, float y) {
    float d;
    asm("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %3, 0;\n\tselp.f32 %0, %1, %2, q;\n\t}" : "=f"(d) : "f"(x), "f"(y), "r"((int)p));
    return d;
}

// One step of the transposing butterfly with compile-time indices: lanes exchange HALF values with the
// lane HALF away and keep the half of the set their lane bit selects.
template <int HALF>
__device__ __forceinline__ void bfly_step(float (&vals)[32], int lane) {
    const bool hi = (lane & HALF) != 0;
#pragma unroll
    for (int i = 0; i < HALF; ++i) {
        const float send = selp_f32(hi, vals[i], vals[i + HALF]);
        const float keep = selp_f32(hi, vals[i + HALF], vals[i]);
        vals[i] = keep + __shfl_xor_sync(IMPALA_FULL_MASK, send, HALF);
    }
}

// The wide-shape instantiations ask for one resident CTA per SM: without it ptxas caps the OP = 64,
// NP = 32 kernel at 128 registers and spills.
// SPLIT: the split-head twin (shared-torso networks, NP >= 4 only)
template <int JPT, int OP, int NP, int MAXT, bool SPLIT = false>
__global__ void __launch_bounds__(MAXT, (OP == 128 || NP == 32) ? 1 : 0) mlp_fwd_kernel(MlpArgsT<SPLIT> a) {
    static_assert(kGroup * NP == 32 || NP != 4, "butterfly chunk must be 32 values");
    // the instantiations of the wide shapes (O > 64 or N2 > 16) keep the butterfly in registers
    constexpr bool kSelp = OP == 128 || NP == 32;
    extern __shared__ __align__(16) float smem[];
    const int nt = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nwarps = nt >> 5;
    float* xs = smem;                // [kRows][OP]
    float* part = xs + kRows * OP;   // [nwarps][kRows*NP]
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;
    const float* __restrict__ b2 = a.params + a.lay.ob2;

    float w[JPT][OP], b1r[JPT], w2r[JPT][NP];
    load_w1<JPT, OP>(w, W1, tid, nt, a.H, a.O);
#pragma unroll
    for (int q = 0; q < JPT; ++q) {
        const int j = tid + q * nt;
        b1r[q] = j < a.H ? __ldg(b1 + j) : 0.f;
#pragma unroll
        for (int n = 0; n < NP; ++n)
            w2r[q][n] = (j < a.H && n < a.N2) ? __ldg(W2 + (size_t)n * a.H + j) : 0.f;
    }

    // rows per 32-value butterfly chunk; a register block of kGroup rows holds kGroup*NP values
    constexpr int VALS = kGroup * NP;            // 8, 32 or 128
    constexpr int CH = VALS >= 32 ? VALS / 32 : 1;  // butterfly chunks per register block
    for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
        const int row0 = tile * kRows;
        __syncthreads();  // previous tile's readers of xs / part are done
        stage_x<kRows, OP>(xs, a.x, row0, a.M, a.O);
        __syncthreads();
#pragma unroll 1
        for (int g = 0; g < kRows / kGroup; ++g) {
            float acc[JPT][kGroup];
            layer1<JPT, OP>(acc, w, xs + g * kGroup * OP, b1r);
            if constexpr (VALS >= 32) {
#pragma unroll
                for (int c = 0; c < CH; ++c) {
                    float vals[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) {
                        const int v = c * 32 + i, r = v / NP, n = v % NP;
                        float s = 0.f;
#pragma unroll
                        for (int q = 0; q < JPT; ++q) s = fmaf(fmaxf(acc[q][r], 0.f), w2r[q][n], s);
                        vals[i] = s;
                    }
                    // transposing butterfly: 32 values x 32 lanes -> lane i holds warp-sum of value i
                    if constexpr (kSelp) {
                        bfly_step<16>(vals, lane), bfly_step<8>(vals, lane), bfly_step<4>(vals, lane);
                        bfly_step<2>(vals, lane), bfly_step<1>(vals, lane);
                    } else {
#pragma unroll
                        for (int s = 0; s < 5; ++s) {
                            const int half = 16 >> s;
                            const bool hi = (lane & half) != 0;
#pragma unroll
                            for (int i = 0; i < half; ++i) {
                                const float send = hi ? vals[i] : vals[i + half];
                                const float keep = hi ? vals[i + half] : vals[i];
                                vals[i] = keep + __shfl_xor_sync(IMPALA_FULL_MASK, send, half);
                            }
                        }
                    }
                    part[warp * (kRows * NP) + g * VALS + c * 32 + lane] = vals[0];
                }
            } else {
                // VALS == 8 (NP == 1): 8 values per lane; 3 transposing steps then 2 plain ones
                float vals[kGroup];
#pragma unroll
                for (int r = 0; r < kGroup; ++r) {
                    float s = 0.f;
#pragma unroll
                    for (int q = 0; q < JPT; ++q) s = fmaf(fmaxf(acc[q][r], 0.f), w2r[q][0], s);
                    vals[r] = s;
                }
#pragma unroll
                for (int s = 0; s < 3; ++s) {
                    const int half = 4 >> s;         // values kept after this step
                    const int off = 16 >> s;         // lane distance
                    const bool hi = (lane & off) != 0;
#pragma unroll
                    for (int i = 0; i < half; ++i) {
                        const float send = hi ? vals[i] : vals[i + half];
                        const float keep = hi ? vals[i + half] : vals[i];
                        vals[i] = keep + __shfl_xor_sync(IMPALA_FULL_MASK, send, off);
                    }
                }
                vals[0] += __shfl_xor_sync(IMPALA_FULL_MASK, vals[0], 2);
                vals[0] += __shfl_xor_sync(IMPALA_FULL_MASK, vals[0], 1);
                // value index held by this lane: bit4 -> 4, bit3 -> 2, bit2 -> 1
                if ((lane & 3) == 0) part[warp * (kRows * NP) + g * VALS + (lane >> 2)] = vals[0];
            }
        }
        __syncthreads();
        for (int idx = tid; idx < kRows * NP; idx += nt) {
            const int r = idx / NP, n = idx - r * NP;
            const int row = row0 + r;
            if (n < a.N2 && row < a.M) {
                float s = __ldg(b2 + n);
                for (int ww = 0; ww < nwarps; ++ww) s += part[ww * (kRows * NP) + idx];
                if constexpr (SPLIT) {
                    if (float* o = split_out(a.out, a.out_b, a.M_a, a.N2, row, n)) *o = s;
                } else {
                    a.out[(size_t)row * a.N2 + n] = s;
                }
            }
        }
    }
}

__device__ __forceinline__ void zero_range(float* p, int64_t lo, int64_t hi) {
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) p[i] = 0.f;
}

// grid = (persistent row-tile CTAs, hidden slices): CTA (bx, by) owns hidden units
// [by * (nt / KS) * JPT, (by+1) * (nt / KS) * JPT) and writes that part of partial row bx.
// KS = 2 (wide observations, OP = 64): a hidden unit is shared by a lane pair, each lane keeps HALF of
// its W1 row and of its dW1 row in registers (2 x 32 instead of 2 x 64 - the one-thread-per-unit
// form spilled ~1.5 KB per thread at this width); the two partial dot products of the recompute
// meet through one shuffle per row, everything downstream of the pre-activation is computed by
// both lanes and stored by the even one.
// KS = 4 (wide shapes, OP = 64 / 128): the same over a lane quad, OP / 4 features per lane; the quad's
// features are interleaved in 16-byte chunks (lane `half` holds chunks half, half + 4, ...) so that the
// four broadcast loads of a row hit four different bank groups.
// NP = 32 (and NP = 16 at KS = 4): the W2 column of a unit and its gradient are split over the KS lanes
// as well (NP / KS outputs per lane); the partial dh of the lanes meet through log2(KS) shuffles per row.
template <int JPT, int OP, int NP, int MAXT, int KS = 1, bool SPLIT = false>
__global__ void __launch_bounds__(MAXT) mlp_bwd_kernel(MlpArgsT<SPLIT> a) {
    extern __shared__ __align__(16) float smem[];
    constexpr int OPH = OP / KS;  // features held by this thread
    constexpr bool SPLITN = NP > 16 || (KS == 4 && NP == 16);
    constexpr int NPL = SPLITN ? NP / KS : NP;  // W2 outputs held by this thread
    static_assert(!SPLITN || KS > 1, "the NP = 32 backward splits W2 over a lane group");
    constexpr int XSTEP = KS == 4 ? 4 * KS : 4;  // feature distance of this thread's 16-byte chunks
    const int nt = blockDim.x, tid = threadIdx.x;
    const int half = KS == 2 ? (tid & 1) : (KS == 4 ? (tid & 3) : 0);
    const int ju = KS == 2 ? (tid >> 1) : (KS == 4 ? (tid >> 2) : tid), nu = nt / KS;
    const int j0 = blockIdx.y * nu * JPT + ju;
    const int koff = KS == 4 ? 4 * half : half * OPH;  // first feature of this thread
    const int n0 = SPLITN ? half * NPL : 0;             // first W2 output of this thread
    float* xs = smem;               // [kRows][OP]
    float* dzs = xs + kRows * OP;   // [kRows][NP]
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;

    float w[JPT][OPH], b1r[JPT], w2r[JPT][NPL];
    float gw1[JPT][OPH], gb1[JPT], gw2[JPT][NPL], gb2 = 0.f;
#pragma unroll
    for (int q = 0; q < JPT; ++q) {
        const int j = j0 + q * nu;
#pragma unroll
        for (int k = 0; k < OPH; ++k) {
            const int f = KS == 4 ? koff + XSTEP * (k >> 2) + (k & 3) : koff + k;  // feature of w[q][k]
            w[q][k] = (j < a.H && f < a.O) ? __ldg(W1 + (size_t)j * a.O + f) : 0.f;
        }
        b1r[q] = (j < a.H && half == 0) ? __ldg(b1 + j) : 0.f;  // added once per unit
        gb1[q] = 0.f;
#pragma unroll
        for (int n = 0; n < NPL; ++n) {
            w2r[q][n] = (j < a.H && n0 + n < a.N2) ? __ldg(W2 + (size_t)(n0 + n) * a.H + j) : 0.f;
            gw2[q][n] = 0.f;
        }
#pragma unroll
        for (int k = 0; k < OPH; ++k) gw1[q][k] = 0.f;
    }

    for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
        const int row0 = tile * kRows;
        __syncthreads();
        stage_x<kRows, OP>(xs, a.x, row0, a.M, a.O);
        for (int idx = tid; idx < kRows * NP; idx += nt) {
            const int r = idx / NP, n = idx - r * NP;
            const int row = row0 + r;
            if constexpr (SPLIT)
                dzs[idx] = (row < a.M && n < a.N2) ? split_dz(a.dout, a.dout_b, a.M_a, a.N2, row, n) : 0.f;
            else
                dzs[idx] = (row < a.M && n < a.N2) ? __ldg(a.dout + (size_t)row * a.N2 + n) : 0.f;
        }
        __syncthreads();
#pragma unroll 1
        for (int g = 0; g < kRows / kGroup; ++g) {
            const float* xg = xs + g * kGroup * OP + koff;
            const float* dzg = dzs + g * kGroup * NP;
            float acc[JPT][kGroup];
            // recompute pre-activations (this thread's features; row stride of the tile stays OP)
#pragma unroll
            for (int q = 0; q < JPT; ++q)
#pragma unroll
                for (int r = 0; r < kGroup; ++r) acc[q][r] = b1r[q];
#pragma unroll
            for (int k4 = 0; k4 < OPH / 4; ++k4) {
#pragma unroll
                for (int r = 0; r < kGroup; ++r) {
                    const float4 xv = *reinterpret_cast<const float4*>(xg + r * OP + XSTEP * k4);
#pragma unroll
                    for (int q = 0; q < JPT; ++q) {
                        acc[q][r] = fmaf(w[q][4 * k4 + 0], xv.x, acc[q][r]);
                        acc[q][r] = fmaf(w[q][4 * k4 + 1], xv.y, acc[q][r]);
                        acc[q][r] = fmaf(w[q][4 * k4 + 2], xv.z, acc[q][r]);
                        acc[q][r] = fmaf(w[q][4 * k4 + 3], xv.w, acc[q][r]);
                    }
                }
            }
#pragma unroll
            for (int m = 1; m < KS; m <<= 1)
#pragma unroll
                for (int q = 0; q < JPT; ++q)
#pragma unroll
                    for (int r = 0; r < kGroup; ++r) acc[q][r] += __shfl_xor_sync(IMPALA_FULL_MASK, acc[q][r], m);
#pragma unroll
            for (int r = 0; r < kGroup; ++r) {
                float dz[NPL];
                const float* dzr = dzg + r * NP + n0;
                if constexpr (NPL % 4 == 0) {
#pragma unroll
                    for (int n4 = 0; n4 < NPL / 4; ++n4) {
                        const float4 t = *reinterpret_cast<const float4*>(dzr + 4 * n4);
                        dz[4 * n4] = t.x, dz[4 * n4 + 1] = t.y, dz[4 * n4 + 2] = t.z, dz[4 * n4 + 3] = t.w;
                    }
                } else {
#pragma unroll
                    for (int n = 0; n < NPL; ++n) dz[n] = dzr[n];
                }
#pragma unroll
                for (int q = 0; q < JPT; ++q) {
                    const float pre = acc[q][r];
                    const float h = fmaxf(pre, 0.f);
                    float dh = 0.f;
#pragma unroll
                    for (int n = 0; n < NPL; ++n) {
                        dh = fmaf(dz[n], w2r[q][n], dh);
                        gw2[q][n] = fmaf(dz[n], h, gw2[q][n]);
                    }
                    if constexpr (SPLITN) {
#pragma unroll
                        for (int m = 1; m < KS; m <<= 1) dh += __shfl_xor_sync(IMPALA_FULL_MASK, dh, m);
                    }
                    const float dp = pre > 0.f ? dh : 0.f;  // relu'(0) = 0 as in torch
                    acc[q][r] = dp;
                    gb1[q] += dp;
                }
            }
#pragma unroll
            for (int k4 = 0; k4 < OPH / 4; ++k4) {
#pragma unroll
                for (int r = 0; r < kGroup; ++r) {
                    const float4 xv = *reinterpret_cast<const float4*>(xg + r * OP + XSTEP * k4);
#pragma unroll
                    for (int q = 0; q < JPT; ++q) {
                        gw1[q][4 * k4 + 0] = fmaf(acc[q][r], xv.x, gw1[q][4 * k4 + 0]);
                        gw1[q][4 * k4 + 1] = fmaf(acc[q][r], xv.y, gw1[q][4 * k4 + 1]);
                        gw1[q][4 * k4 + 2] = fmaf(acc[q][r], xv.z, gw1[q][4 * k4 + 2]);
                        gw1[q][4 * k4 + 3] = fmaf(acc[q][r], xv.w, gw1[q][4 * k4 + 3]);
                    }
                }
            }
        }
        if (blockIdx.y == 0 && tid < a.N2) {
            for (int r = 0; r < kRows; ++r) gb2 += dzs[r * NP + tid];
        }
    }

    // this CTA's slice of partial-gradient row blockIdx.x (parameter-block layout)
    float* wsb = a.ws + (size_t)blockIdx.x * a.lay.total;
#pragma unroll
    for (int q = 0; q < JPT; ++q) {
        const int j = j0 + q * nu;
        if (j < a.H) {
#pragma unroll
            for (int k = 0; k < OPH; ++k) {
                const int f = KS == 4 ? koff + XSTEP * (k >> 2) + (k & 3) : koff + k;
                if (f < a.O) wsb[a.lay.oW1 + (size_t)j * a.O + f] = gw1[q][k];
            }
            if (half == 0) {
                wsb[a.lay.ob1 + j] = gb1[q];
                if constexpr (!SPLITN) {
#pragma unroll
                    for (int n = 0; n < NP; ++n)
                        if (n < a.N2) wsb[a.lay.oW2 + (size_t)n * a.H + j] = gw2[q][n];
                }
            }
            if constexpr (SPLITN) {
#pragma unroll
                for (int n = 0; n < NPL; ++n)
                    if (n0 + n < a.N2) wsb[a.lay.oW2 + (size_t)(n0 + n) * a.H + j] = gw2[q][n];
            }
        }
    }
    if (blockIdx.y == 0) {
        if (tid < a.N2) wsb[a.lay.ob2 + tid] = gb2;
        zero_range(wsb, a.lay.oW1 + (int64_t)a.H * a.O, a.lay.ob1);
        zero_range(wsb, a.lay.ob1 + a.H, a.lay.oW2);
        zero_range(wsb, a.lay.oW2 + (int64_t)a.N2 * a.H, a.lay.ob2);
        zero_range(wsb, a.lay.ob2 + a.N2, a.lay.total);
    }
}

}  // namespace impala_mlp
