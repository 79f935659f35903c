// Phase clocks of the narrow tensor-core MLP kernels (bwd_blk_body, fwd_rs_body): where a warpgroup's
// cycles go, per phase of its tile loop.  Compiled in only with -DIMPALA_PHASE_CLOCKS (`IMPALA_PHASE_CLOCKS=1
// IMPALA_LIB_DIR=<dir> python -m torched_impala_b200.build`, read by scripts/phase_mlp.py); without it every
// macro below is empty, so the library's kernels and ABI are those of a build without the header.
//
// One thread per warpgroup (thread 0 of the warpgroup) keeps its last clock64() reading in shared memory and
// adds the delta since then to the phase sum a mark names, so the hot loop holds no extra live register.  A
// GEMM window is issue -> wait return; a window that opens while the other warpgroup of the CTA is inside
// one counts as an overlap (the convoy measure: two warpgroups whose MMAs queue behind each other).  At the
// end of the body the sums of every warpgroup go to the translation unit's __device__ buffer, with the CTA's
// %globaltimer span (tail and imbalance).
#pragma once

#include <stdint.h>

namespace phase {
constexpr int kPhases = 8;  // phase sums [0, 8): meaning per kernel (scripts/phase_mlp.py)
// counters after the phase sums
enum : int {
    kTiles = kPhases,  // warpgroup-tiles
    kOverlap,          // GEMM windows opened while the other warpgroup was inside one
    kWindows,          // GEMM windows
    kWgCycles,         // clock64 from body start to end, summed over warpgroups
    kCtaNs,            // %globaltimer span of each CTA, summed
    kCtas,
    kFirstNs,          // earliest CTA start, latest CTA end (%globaltimer)
    kLastNs,
    kSlots
};
}  // namespace phase

#ifdef IMPALA_PHASE_CLOCKS

namespace phase {
__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
}  // namespace phase

// the buffer of this translation unit's instrumented body: zeroed on load and by the reader's reset
static __device__ unsigned long long impala_phase_buf[phase::kSlots];

// pc_s[wg]: [0, kPhases) sums, then tiles, overlaps, windows, last clock, body start clock, in-window flag.
// Both rows are zeroed before a __syncthreads, so the other warpgroup's in-window flag is never read
// uninitialised (called where every thread of the CTA passes).
#define PHASE_BEGIN(wg)                                                                                     \
    __shared__ unsigned long long pc_s[2][16];                                                              \
    __shared__ unsigned long long pc_ns0;                                                                   \
    const bool pc_on = (threadIdx.x & 127) == 0;                                                            \
    if (threadIdx.x < 32) pc_s[threadIdx.x >> 4][threadIdx.x & 15] = 0ull;                                  \
    __syncthreads();                                                                                        \
    if (pc_on) {                                                                                            \
        pc_s[wg][11] = pc_s[wg][12] = (unsigned long long)clock64();                                        \
        if (threadIdx.x == 0) pc_ns0 = phase::globaltimer();                                                \
    }
// the cycles since the previous mark go to phase k
#define PHASE_MARK(wg, k)                                                                                   \
    if (pc_on) {                                                                                            \
        const unsigned long long t_ = (unsigned long long)clock64();                                        \
        pc_s[wg][k] += t_ - pc_s[wg][11];                                                                   \
        pc_s[wg][11] = t_;                                                                                  \
    }
#define PHASE_GEMM_ON(wg)                                                                                   \
    if (pc_on) {                                                                                            \
        pc_s[wg][10] += 1ull;                                                                               \
        pc_s[wg][9] += *(volatile unsigned long long*)&pc_s[(wg) ^ 1][13] != 0ull;                          \
        *(volatile unsigned long long*)&pc_s[wg][13] = 1ull;                                                \
    }
#define PHASE_GEMM_OFF(wg)                                                                                  \
    if (pc_on) *(volatile unsigned long long*)&pc_s[wg][13] = 0ull;
#define PHASE_TILE(wg)                                                                                      \
    if (pc_on) pc_s[wg][8] += 1ull;
// a body without a closing __syncthreads of its own: every warpgroup is done before the CTA's end time
#define PHASE_SYNC() __syncthreads()
// after the body's closing __syncthreads
#define PHASE_END(wg)                                                                                       \
    if (pc_on) {                                                                                            \
        for (int i_ = 0; i_ < phase::kPhases; ++i_) atomicAdd(&impala_phase_buf[i_], pc_s[wg][i_]);         \
        atomicAdd(&impala_phase_buf[phase::kTiles], pc_s[wg][8]);                                           \
        atomicAdd(&impala_phase_buf[phase::kOverlap], pc_s[wg][9]);                                         \
        atomicAdd(&impala_phase_buf[phase::kWindows], pc_s[wg][10]);                                        \
        atomicAdd(&impala_phase_buf[phase::kWgCycles], (unsigned long long)clock64() - pc_s[wg][12]);       \
        if (threadIdx.x == 0) {                                                                             \
            const unsigned long long e_ = phase::globaltimer();                                             \
            atomicAdd(&impala_phase_buf[phase::kCtaNs], e_ - pc_ns0);                                       \
            atomicAdd(&impala_phase_buf[phase::kCtas], 1ull);                                               \
            atomicMin(&impala_phase_buf[phase::kFirstNs], pc_ns0);                                          \
            atomicMax(&impala_phase_buf[phase::kLastNs], e_);                                               \
        }                                                                                                   \
    }
// host reader of this translation unit's buffer: copies kSlots counters to `out`, then optionally re-arms
#define IMPALA_PHASE_READER(name)                                                                           \
    int name(unsigned long long* out, int reset) {                                                          \
        if (cudaMemcpyFromSymbol(out, impala_phase_buf, sizeof(impala_phase_buf)) != cudaSuccess) return -1; \
        if (reset) {                                                                                        \
            unsigned long long z[phase::kSlots] = {};                                                       \
            z[phase::kFirstNs] = ~0ull;                                                                     \
            if (cudaMemcpyToSymbol(impala_phase_buf, z, sizeof(z)) != cudaSuccess) return -1;               \
        }                                                                                                   \
        return 0;                                                                                           \
    }
int impala_phase_read_bwd(unsigned long long* out, int reset);
int impala_phase_read_fwd(unsigned long long* out, int reset);

#else

#define PHASE_BEGIN(wg)
#define PHASE_MARK(wg, k)
#define PHASE_GEMM_ON(wg)
#define PHASE_GEMM_OFF(wg)
#define PHASE_TILE(wg)
#define PHASE_SYNC()
#define PHASE_END(wg)

#endif
