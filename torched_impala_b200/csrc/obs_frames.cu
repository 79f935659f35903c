// Frame-stacked observations: the slab carries each frame once, (T+k, B, F); one launch per step
// rebuilds the dense (T+1, B, k F) observation rows the MLP kernels read.
#include <algorithm>

#include "common.cuh"

namespace {

// One vector of V elements: frame element -> observation element, converted.  V = 16 bytes of input
// for uint8 frames (16 bytes out as uint8, 64 bytes as float32), 16 bytes (4 floats) for float32 frames;
// V = 1 is the scalar path for frame widths the vectors do not divide.
template <typename In, typename Out, int V>
__device__ __forceinline__ void copy_vec(const In* __restrict__ src, Out* __restrict__ dst) {
    if constexpr (V == 1) {
        *dst = (Out)__ldg(src);
    } else if constexpr (sizeof(In) == sizeof(Out)) {
        *reinterpret_cast<uint4*>(dst) = __ldg(reinterpret_cast<const uint4*>(src));
    } else {  // uint8 -> float32: one 16-byte load, four 16-byte stores
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(src));
        const unsigned words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
            reinterpret_cast<float4*>(dst)[q] = make_float4((float)(words[q] & 255u), (float)((words[q] >> 8) & 255u),
                                                            (float)((words[q] >> 16) & 255u), (float)(words[q] >> 24));
    }
}

// out vector i = (r k + j) Fv + f  <-  frames vector (r + j B) Fv + f, for output row r = t B + b < rows,
// frame slot j < k and vector f < Fv of the frame.  The output is walked contiguously; (r, j, f) follow
// the grid stride as a mixed-radix counter, so no element pays a division.
template <typename In, typename Out, int V>
__global__ void __launch_bounds__(256) obs_unstack_kernel(const In* __restrict__ in, Out* __restrict__ out,
                                                          int64_t rows, int64_t B, int Fv, int k) {
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t kFv = (int64_t)k * Fv;
    int64_t r = i0 / kFv;
    const int c = (int)(i0 - r * kFv);
    int j = c / Fv, f = c - j * Fv;
    const int64_t dr = stride / kFv;
    const int dc = (int)(stride - dr * kFv), dj = dc / Fv, df = dc - dj * Fv;
    for (int64_t i = i0; r < rows; i += stride) {
        copy_vec<In, Out, V>(in + ((r + j * B) * Fv + f) * V, out + i * V);
        f += df, j += dj, r += dr;
        if (f >= Fv) f -= Fv, ++j;
        if (j >= k) j -= k, ++r;
    }
}

template <typename In, typename Out>
int launch_unstack(const void* frames, void* out, int64_t rows, int B, int F, int k, cudaStream_t st) {
    constexpr int V = sizeof(In) == 1 ? 16 : 4;  // 16 bytes of frame data per vector
    const bool vec = F % V == 0 && ((reinterpret_cast<uintptr_t>(frames) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const int Fv = vec ? F / V : F;
    int sms = 0;
    if (const cudaError_t e = impala_sm_count(&sms); e != cudaSuccess) return (int)e;
    const int64_t work = rows * k * Fv;
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((work + 255) / 256, (int64_t)sms * 16));
    const In* x = static_cast<const In*>(frames);
    Out* y = static_cast<Out*>(out);
    if (vec)
        obs_unstack_kernel<In, Out, V><<<grid, 256, 0, st>>>(x, y, rows, B, Fv, k);
    else
        obs_unstack_kernel<In, Out, 1><<<grid, 256, 0, st>>>(x, y, rows, B, Fv, k);
    return impala_launch_status();
}

}  // namespace

extern "C" int impala_obs_unstack(const void* frames, int in_dtype, void* out, int out_dtype, int R, int B, int F,
                                  int k, void* stream) {
    if (!frames || !out || R < 1 || B < 1 || F < 1 || k < 1) return IMPALA_ERR_BAD_ARG;
    const int64_t rows = (int64_t)R * B;
    cudaStream_t st = (cudaStream_t)stream;
    if (in_dtype == IMPALA_OBS_U8 && out_dtype == IMPALA_OBS_U8)
        return launch_unstack<uint8_t, uint8_t>(frames, out, rows, B, F, k, st);
    if (in_dtype == IMPALA_OBS_U8 && out_dtype == IMPALA_OBS_F32)
        return launch_unstack<uint8_t, float>(frames, out, rows, B, F, k, st);
    if (in_dtype == IMPALA_OBS_F32 && out_dtype == IMPALA_OBS_F32)
        return launch_unstack<float, float>(frames, out, rows, B, F, k, st);
    return IMPALA_ERR_BAD_ARG;
}
