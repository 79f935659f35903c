// Epilogue of the tensor-core MLP forwards (mlp_fwd_tc.cu, mlp_obs_tc.cu): bias, ReLU and the second
// layer on the fp32 accumulator of a 32-unit hidden slice, and the pass rule that writes an output row.
#pragma once

#include <type_traits>

#include "mlp_kernels.cuh"

namespace {

constexpr int kTileM = 64;  // rows per tile (wgmma M)

struct FwdTcArgs {
    const float* x;
    const float* params;
    float* out;
    int M, O, H, N2, num_tiles;
    int hb;  // hidden units per pass (multiple of 32, <= 256, divides H)
    MlpLayout lay;
};

// The arguments of the split-head twins (SPLIT kernels): out is head a, out_b head b (split_out).  A
// struct of its own, so the kernels of the interleaved layout keep their parameter space.
struct FwdTcSplitArgs : FwdTcArgs {
    float* out_b;
    int M_a;
};
template <bool SPLIT>
using FwdArgs = std::conditional_t<SPLIT, FwdTcSplitArgs, FwdTcArgs>;

// W2 rows in shared memory are padded to NP + 4 at NP = 16 and 32: the lanes of a quad read hidden units
// two apart, and with 64- or 128-byte rows their 16-byte loads would fall into one bank group
__host__ __device__ constexpr int w2s_stride(int np) { return np > 4 ? np + 4 : np; }

// Epilogue of the 32-unit slices nc, nc + 1, ... held in one accumulator (16 registers per slice: an
// m64n32 accumulator, or the halves of an m64n64 one), slice by slice: bias, ReLU, second layer on this
// thread's 2 rows x 8 units of the slice, added into the partial sums p0 / p1 of rows 16 warp + g and + 8
template <int NP, int ND>
__device__ __forceinline__ void slice_epilogue(const float (&d)[ND], int nc, int q, const float* b1s, const float* w2s,
                                               float (&p0)[NP], float (&p1)[NP]) {
    constexpr int NPS = w2s_stride(NP);
    static_assert(ND % 16 == 0, "whole 32-unit slices");
#pragma unroll
    for (int i = 0; i < ND / 4; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int j = nc * 32 + 8 * i + 2 * q + e;
            const float bj = b1s[j];
            const float h0 = fmaxf(d[4 * i + e] + bj, 0.f);
            const float h1 = fmaxf(d[4 * i + 2 + e] + bj, 0.f);
            if constexpr (NP % 4 == 0) {
#pragma unroll
                for (int n = 0; n < NP; n += 4) {
                    const float4 w = *reinterpret_cast<const float4*>(w2s + NPS * j + n);
                    p0[n] = fmaf(h0, w.x, p0[n]), p0[n + 1] = fmaf(h0, w.y, p0[n + 1]);
                    p0[n + 2] = fmaf(h0, w.z, p0[n + 2]), p0[n + 3] = fmaf(h0, w.w, p0[n + 3]);
                    p1[n] = fmaf(h1, w.x, p1[n]), p1[n + 1] = fmaf(h1, w.y, p1[n + 1]);
                    p1[n + 2] = fmaf(h1, w.z, p1[n + 2]), p1[n + 3] = fmaf(h1, w.w, p1[n + 3]);
                }
            } else {
                const float w = w2s[j];
                p0[0] = fmaf(h0, w, p0[0]), p1[0] = fmaf(h1, w, p1[0]);
            }
        }
    }
}

// The quad's four column sets meet (fixed order), lane q == 0 writes (pass 0: b2 + z_0) or adds to
// what it wrote in the previous pass the two rows of this tile (SPLIT: at the split-head addresses)
template <int NP, bool SPLIT = false>
__device__ __forceinline__ void write_rows(const FwdArgs<SPLIT>& a, int p, int tile, int warp, int g, int q, float (&p0)[NP],
                                           float (&p1)[NP]) {
    const float* __restrict__ b2 = a.params + a.lay.ob2;
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
                if constexpr (SPLIT) {
#pragma unroll
                    for (int n = 0; n < NP; ++n) {
                        float* o = n < a.N2 ? split_out(a.out, a.out_b, a.M_a, a.N2, row, n) : nullptr;
                        if (o) *o = (p == 0 ? __ldg(b2 + n) : *o) + (h ? p1[n] : p0[n]);
                    }
                } else {
                    float* o = a.out + (size_t)row * a.N2;
#pragma unroll
                    for (int n = 0; n < NP; ++n)
                        if (n < a.N2) o[n] = (p == 0 ? __ldg(b2 + n) : o[n]) + (h ? p1[n] : p0[n]);
                }
            }
        }
    }
}

}  // namespace
