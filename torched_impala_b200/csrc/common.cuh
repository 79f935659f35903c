// Shared helpers for the sm_90a learner kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/impala_b200.h"

#define IMPALA_FULL_MASK 0xffffffffu

static inline int64_t impala_round_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

struct MlpLayout {
    int64_t oW1, ob1, oW2, ob2, total;
};

static inline MlpLayout impala_make_layout(int O, int H, int N2) {
    MlpLayout l;
    const int64_t al = IMPALA_PARAM_ALIGN;
    l.oW1 = 0;
    l.ob1 = impala_round_up(l.oW1 + (int64_t)H * O, al);
    l.oW2 = impala_round_up(l.ob1 + H, al);
    l.ob2 = impala_round_up(l.oW2 + (int64_t)N2 * H, al);
    l.total = impala_round_up(l.ob2 + N2, al);
    return l;
}

// Kernels this library has launched (or recorded into a capturing stream) since it was loaded;
// defined in abi.cu, read through impala_launch_count().
extern long long g_impala_launches;

// Called once after every kernel launch of the library.
static inline int impala_launch_status() {
    __atomic_fetch_add(&g_impala_launches, 1, __ATOMIC_RELAXED);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

// SM count of the current device (cached per device).
static inline cudaError_t impala_sm_count(int* out) {
    static int cached[64] = {0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64 || !cached[dev]) {
        int n = 0;
        if ((e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
        if (dev < 0 || dev >= 64) return *out = n, cudaSuccess;
        cached[dev] = n;
    }
    *out = cached[dev];
    return cudaSuccess;
}

static inline int impala_env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

// A persistent launch of `grid` CTAs shared by two tile lists (policy / value network): how many
// CTAs take list A so that the slower side finishes earliest, for per-tile cost weights wa, wb.
static inline int impala_pair_split(int tiles_a, int tiles_b, int grid, int64_t wa, int64_t wb) {
    int best = 1;
    int64_t best_cost = INT64_MAX, best_sum = INT64_MAX;
    for (int na = 1; na < grid; ++na) {
        const int nb = grid - na;
        if (na > tiles_a || nb > tiles_b) continue;
        const int64_t ca = (int64_t)((tiles_a + na - 1) / na) * wa, cb = (int64_t)((tiles_b + nb - 1) / nb) * wb;
        const int64_t cost = ca > cb ? ca : cb, sum = ca + cb;
        if (cost < best_cost || (cost == best_cost && sum < best_sum)) best = na, best_cost = cost, best_sum = sum;
    }
    return best;
}

__device__ __forceinline__ double warp_sum_f64(double x) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(IMPALA_FULL_MASK, x, off);
    return x;
}

// ---- programmatic dependent launch (PDL): kernels 2..4 of a learner step are launched with the
// programmatic-stream-serialization attribute and call pdl_wait() before the first access to
// anything their predecessor produces.  No kernel triggers early (no griddepcontrol.launch_dependents):
// the trigger is the implicit one at the exit of each predecessor CTA, i.e. every write of the
// predecessor precedes it, so the successor's CTAs are merely pre-staged - they occupy SMs as the
// predecessor's CTAs drain and run their own prologue (weight staging, optimizer-state loads) while
// the last predecessor CTAs finish - and pdl_wait() returns once the predecessor grid is complete and flushed.  (An early trigger at kernel start
// was measured first: the optimizer then read gradients the backward's reduction phase had not
// written yet - tests/test_gpu_fullsize.py caught it - so the wait must not be relied on to cover
// writes issued after a trigger.)  Inside a captured CUDA graph these launches become programmatic
// edges.  Without an early trigger there is little left to overlap, so the attribute is OFF by default
// (IMPALA_PDL=1 enables it; the waits are no-ops on plain launches).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// cluster_x > 1: launch as thread-block clusters of that many CTAs along x (grid.x a multiple of it).
template <typename... KArgs, typename... Args>
static inline cudaError_t impala_launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                           cudaStream_t st, bool dependent, bool cooperative, Args&&... args) {
    return impala_launch_cl(kernel, grid, block, smem, st, dependent, cooperative, 1, static_cast<Args&&>(args)...);
}

template <typename... KArgs, typename... Args>
static inline cudaError_t impala_launch_cl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                           cudaStream_t st, bool dependent, bool cooperative, int cluster_x,
                                           Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = st;
    cudaLaunchAttribute attr[3];
    unsigned n = 0;
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = (unsigned)cluster_x, attr[n].val.clusterDim.y = 1, attr[n].val.clusterDim.z = 1;
        ++n;
    }
    if (dependent && impala_env_int("IMPALA_PDL", 0) != 0) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cooperative) {
        attr[n].id = cudaLaunchAttributeCooperative;
        attr[n].val.cooperative = 1;
        ++n;
    }
    cfg.attrs = attr, cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// cooperative: the kernel contains a grid-wide barrier - the launch then FAILS (instead of the barrier
// hanging) when the CTAs cannot all be resident, e.g. under an MPS SM limit or in a green context.
template <typename... KArgs, typename... Args>
static inline cudaError_t impala_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                        cudaStream_t st, bool dependent, Args&&... args) {
    return impala_launch_ex(kernel, grid, block, smem, st, dependent, false, static_cast<Args&&>(args)...);
}

// ---- push-model all-reduce over peer memory, LL ("low latency") format (protocol: see optim.cu)
// One float64 travels as 16 bytes  [lo32 | step32 | hi32 | step32] : each 8-byte half carries the
// step number it belongs to, 8-byte stores are single NVLink transactions, so a reader that sees
// both halves tagged with the step it is waiting for has the value - no fence, no separate flag,
// no acknowledgement on the data path.
struct PushArgs {
    ulonglong2* const* gather;  // device array [world]: every rank's gather buffer (peer-mapped)
    const long long* seq;       // this rank's step counter (device, 1 word); the step in flight is *seq + 1
    int64_t slot_stride;        // LL elements between two ranks' slots
    int64_t buf_stride;         // LL elements between the two parity buffers
    int rank, world;
};
__device__ __forceinline__ void ll_store(ulonglong2* dst, double v, unsigned step) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
    const unsigned long long tag = (unsigned long long)step << 32;
    const unsigned long long lo = (bits & 0xffffffffull) | tag, hi = (bits >> 32) | tag;
    // plain (weak) 16-byte store: LL needs no ordering between elements, only that each 8-byte half
    // lands whole - which any aligned 8-byte store does
    asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(lo), "l"(hi) : "memory");
}
__device__ __forceinline__ ulonglong2 ll_load(const ulonglong2* src) {
    ulonglong2 w;
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w.x), "=l"(w.y) : "l"(src) : "memory");
    return w;
}
__device__ __forceinline__ bool ll_ready(const ulonglong2& w, unsigned step) {
    return (unsigned)(w.x >> 32) == step && (unsigned)(w.y >> 32) == step;
}
__device__ __forceinline__ double ll_value(const ulonglong2& w) {
    return __longlong_as_double((long long)((w.x & 0xffffffffull) | (w.y << 32)));
}
