// Inline-PTX wrappers for the sm_90a tensor-core path: warpgroup MMA (`wgmma.mma_async`, kind
// tf32, fp32 accumulators in registers) with K-major, 128-byte-swizzled shared-memory operands,
// and the 3xTF32 operand split.
//
// Descriptor bit layout follows the PTX ISA "Matrix Descriptor Format" table for wgmma (the same
// fields CuTe's GMMA::DescriptorIterator encodes).  Fragment layouts (PTX ISA, "Register
// Fragments" of wgmma .m64nNk8 with .tf32 inputs), for thread t of a warpgroup, warp w = t / 32,
// g = (t % 32) / 4, q = t % 4:
//   accumulator d[r]: row 16 w + g + 8 ((r >> 1) & 1), column 8 (r >> 2) + 2 q + (r & 1)
//   A operand a[i]:   row 16 w + g + 8 (i & 1),        column q + 4 (i >> 1)
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// named barrier over `nthreads` threads (multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void named_bar(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ wgmma
// K-major operand tile, rows of 128 bytes (32 tf32), SWIZZLE_128B, 8-row groups 1024 B apart.
// `byte_off` selects the K step inside the 128-byte row (32 bytes per K = 8 step) or a later
// 8-row group (multiples of 1024).  Tiles are 1024-byte aligned (base offset field 0).
__device__ __forceinline__ uint64_t smem_desc_k_sw128(const void* tile, uint32_t byte_off) {
    const uint32_t addr = smem_u32(tile) + byte_off;
    uint64_t d = 0;
    d |= static_cast<uint64_t>((addr >> 4) & 0x3fff);  // start address          [0,14)
    d |= static_cast<uint64_t>(1) << 16;               // leading byte offset (unused for swizzled K-major)
    d |= static_cast<uint64_t>(1024 >> 4) << 32;       // stride byte offset: next 8-row group
    d |= static_cast<uint64_t>(1) << 62;               // SWIZZLE_128B
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// the accumulator registers are not touched by the compiler across an in-flight wgmma
__device__ __forceinline__ void fence_acc(float (&d)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define IMPALA_WG_D16                                                                                   \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}"
#define IMPALA_WG_D16_OPS(d)                                                                            \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),     \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]),        \
        "+f"(d[15])

// D[64, 32] (+)= A[64, 8] * B[32, 8]^T, both operands from shared memory (warpgroup-collective)
__device__ __forceinline__ void wgmma_n32_ss(float (&d)[16], uint64_t a_desc, uint64_t b_desc, bool accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 " IMPALA_WG_D16 ", %16, %17, p, 1, 1;\n\t"
        "}\n"
        : IMPALA_WG_D16_OPS(d)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate ? 1 : 0));
}
// the same with A from registers (fragment layout in the header comment)
__device__ __forceinline__ void wgmma_n32_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b_desc,
                                             bool accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 " IMPALA_WG_D16 ", {%16, %17, %18, %19}, %20, p, 1, 1;\n\t"
        "}\n"
        : IMPALA_WG_D16_OPS(d)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate ? 1 : 0));
}
#undef IMPALA_WG_D16
#undef IMPALA_WG_D16_OPS

// ------------------------------------------------------------------ 3xTF32 operand split
// hi = round-to-nearest tf32 of x (what the tensor core will see exactly), lo = x - hi (exact in
// fp32; the tensor core truncates it to tf32, an error of 2^-21 relative to x).
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    uint32_t h;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
    hi = __uint_as_float(h);
    lo = x - hi;
}
__device__ __forceinline__ void split4(const float4& v, float4& hi, float4& lo) {
    split_tf32(v.x, hi.x, lo.x);
    split_tf32(v.y, hi.y, lo.y);
    split_tf32(v.z, hi.z, lo.z);
    split_tf32(v.w, hi.w, lo.w);
}

// byte offset of 16-byte chunk `c16` (0..7) of row `r` inside a K-major SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_offset(uint32_t r, uint32_t c16) {
    return (r >> 3) * 1024u + (r & 7u) * 128u + ((c16 ^ (r & 7u)) << 4);
}

}  // namespace tc
