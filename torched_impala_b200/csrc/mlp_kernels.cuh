// Kernel templates of the FP32 MLP forward / backward (see mlp.cu for the design notes).
// Included by mlp_inst.cu, which is compiled once per padded observation width
// (-DIMPALA_OP=..) and direction (-DIMPALA_BWD=0/1) so the instantiations build in parallel.
#pragma once

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

struct MlpConfig {
    int jpt, maxt, op, np, threads, slices;
    int ks;  // backward: threads per hidden unit (2 = the observation features are split over a lane pair)
};

constexpr int kRows = 32;        // rows per staged tile
constexpr int kGroup = 8;        // rows per register block
constexpr int kMaxParts = 1024;  // upper bound on persistent CTAs (= per-CTA partials)

// Defined in mlp.cu: caches occupancy per (kernel, device, block, smem) and launches a
// persistent grid of min(tiles, resident CTAs) x slices blocks.
int impala_mlp_launch(void (*kernel)(MlpArgs), const MlpArgs& a, const MlpConfig& c, size_t smem,
                      cudaStream_t st, int* grid_out);

// Tensor-core (wgmma, 3xTF32) forward for GEMM-shaped layers, defined in mlp_fwd_tc.cu.
bool impala_mlp_fwd_tc_eligible(const float* x, int M, int O, int H, int N2);
int impala_mlp_fwd_tc(const float* x, const float* params, float* out, int M, int O, int H, int N2,
                      cudaStream_t st);

// Policy + value network in one launch (CTA ranges per network); A in 2..4, both nets eligible.
int impala_mlp_fwd_tc_pair(const float* x, const float* params_pi, const float* params_vf, float* logits,
                           float* values, int M_pi, int M_vf, int O, int H_pi, int H_vf, int A,
                           cudaStream_t st);

// Tensor-core backward (mlp_bwd_tc.cu): per-CTA partial rows into ws, reduced in-kernel to grad.
bool impala_mlp_bwd_tc_eligible(const float* x, const float* dout, int M, int O, int H, int N2);
int impala_mlp_bwd_tc(const float* x, const float* params, const float* dout, float* ws,
                      double* grad, unsigned int* ctl, int M, int O, int H, int N2, cudaStream_t st);

int impala_mlp_bwd_tc_pair(const float* x, const float* params_pi, const float* params_vf,
                           const float* dlogits, const float* dv, float* ws_pi, float* ws_vf,
                           double* grad_pi, double* grad_vf, unsigned int* ctl, int M_pi, int M_vf, int O,
                           int H_pi, int H_vf, int A, cudaStream_t st, const PushArgs* push = nullptr,
                           const double* extra = nullptr, int n_extra = 0);

// Wide tensor-core kernels (forward in mlp_fwd_tc.cu, backward in mlp_bwd_tc.cu): O <= 64, H a multiple
// of 128 (BASELINE c5: O = 64, H = 512).  The forward needs no workspace; the backward leaves *nparts float32 partial rows in ws for
// reduce_partials_kernel.  IMPALA_MLP_TCW=0 disables them.
bool impala_mlp_tcw_eligible(const float* x, int M, int O, int H, int N2);
int impala_mlp_fwd_tcw(const float* x, const float* params, float* out, int M, int O, int H, int N2,
                       cudaStream_t st);
int impala_mlp_bwd_tcw(const float* x, const float* params, const float* dout, float* ws, int M, int O, int H,
                       int N2, cudaStream_t st, int* nparts);

// One per padded observation width / direction, defined in mlp_inst.cu.
#define IMPALA_DECL_DISPATCH(OPV)                                                             \
    int impala_mlp_fwd_op##OPV(const MlpArgs&, const MlpConfig&, size_t, cudaStream_t, int*); \
    int impala_mlp_bwd_op##OPV(const MlpArgs&, const MlpConfig&, size_t, cudaStream_t, int*);
IMPALA_DECL_DISPATCH(8)
IMPALA_DECL_DISPATCH(24)
IMPALA_DECL_DISPATCH(32)
IMPALA_DECL_DISPATCH(64)

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

template <int JPT, int OP, int NP, int MAXT>
__global__ void __launch_bounds__(MAXT) mlp_fwd_kernel(MlpArgs a) {
    static_assert(kGroup * NP == 32 || NP != 4, "butterfly chunk must be 32 values");
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
                a.out[(size_t)row * a.N2 + n] = s;
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
template <int JPT, int OP, int NP, int MAXT, int KS = 1>
__global__ void __launch_bounds__(MAXT) mlp_bwd_kernel(MlpArgs a) {
    extern __shared__ __align__(16) float smem[];
    constexpr int OPH = OP / KS;  // features held by this thread
    const int nt = blockDim.x, tid = threadIdx.x;
    const int half = KS == 2 ? (tid & 1) : 0, ju = KS == 2 ? (tid >> 1) : tid, nu = nt / KS;
    const int j0 = blockIdx.y * nu * JPT + ju;
    const int koff = half * OPH;
    float* xs = smem;               // [kRows][OP]
    float* dzs = xs + kRows * OP;   // [kRows][NP]
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;

    float w[JPT][OPH], b1r[JPT], w2r[JPT][NP];
    float gw1[JPT][OPH], gb1[JPT], gw2[JPT][NP], gb2 = 0.f;
#pragma unroll
    for (int q = 0; q < JPT; ++q) {
        const int j = j0 + q * nu;
#pragma unroll
        for (int k = 0; k < OPH; ++k)
            w[q][k] = (j < a.H && koff + k < a.O) ? __ldg(W1 + (size_t)j * a.O + koff + k) : 0.f;
        b1r[q] = (j < a.H && half == 0) ? __ldg(b1 + j) : 0.f;  // added once per unit
        gb1[q] = 0.f;
#pragma unroll
        for (int n = 0; n < NP; ++n) {
            w2r[q][n] = (j < a.H && n < a.N2) ? __ldg(W2 + (size_t)n * a.H + j) : 0.f;
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
                    const float4 xv = *reinterpret_cast<const float4*>(xg + r * OP + 4 * k4);
#pragma unroll
                    for (int q = 0; q < JPT; ++q) {
                        acc[q][r] = fmaf(w[q][4 * k4 + 0], xv.x, acc[q][r]);
                        acc[q][r] = fmaf(w[q][4 * k4 + 1], xv.y, acc[q][r]);
                        acc[q][r] = fmaf(w[q][4 * k4 + 2], xv.z, acc[q][r]);
                        acc[q][r] = fmaf(w[q][4 * k4 + 3], xv.w, acc[q][r]);
                    }
                }
            }
            if constexpr (KS == 2) {
#pragma unroll
                for (int q = 0; q < JPT; ++q)
#pragma unroll
                    for (int r = 0; r < kGroup; ++r) acc[q][r] += __shfl_xor_sync(IMPALA_FULL_MASK, acc[q][r], 1);
            }
#pragma unroll
            for (int r = 0; r < kGroup; ++r) {
                float dz[NP];
                if constexpr (NP % 4 == 0) {
#pragma unroll
                    for (int n4 = 0; n4 < NP / 4; ++n4) {
                        const float4 t = *reinterpret_cast<const float4*>(dzg + r * NP + 4 * n4);
                        dz[4 * n4] = t.x, dz[4 * n4 + 1] = t.y, dz[4 * n4 + 2] = t.z, dz[4 * n4 + 3] = t.w;
                    }
                } else {
#pragma unroll
                    for (int n = 0; n < NP; ++n) dz[n] = dzg[r * NP + n];
                }
#pragma unroll
                for (int q = 0; q < JPT; ++q) {
                    const float pre = acc[q][r];
                    const float h = fmaxf(pre, 0.f);
                    float dh = 0.f;
#pragma unroll
                    for (int n = 0; n < NP; ++n) {
                        dh = fmaf(dz[n], w2r[q][n], dh);
                        gw2[q][n] = fmaf(dz[n], h, gw2[q][n]);
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
                    const float4 xv = *reinterpret_cast<const float4*>(xg + r * OP + 4 * k4);
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
            for (int k = 0; k < OPH; ++k)
                if (koff + k < a.O) wsb[a.lay.oW1 + (size_t)j * a.O + koff + k] = gw1[q][k];
            if (half == 0) {
                wsb[a.lay.ob1 + j] = gb1[q];
#pragma unroll
                for (int n = 0; n < NP; ++n)
                    if (n < a.N2) wsb[a.lay.oW2 + (size_t)n * a.H + j] = gw2[q][n];
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
