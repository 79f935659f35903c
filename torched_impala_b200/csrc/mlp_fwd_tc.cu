// MLP forward on the Hopper tensor cores (wgmma, fp32 accumulators in registers), error-compensated
// 3xTF32.
//
//   out[m,:] = relu(x[m,:] W1^T + b1) W2^T + b2          (models.py:23-25 / :51-52, eval mode)
//
// Layer 1 is the GEMM: per 64-row tile  D[64, HB] = X[64, K] * W1_blk[HB, K]^T  with K = the
// observation width padded to 32 (one 128-byte swizzle atom, narrow kernels) or 64 (two atoms:
// BASELINE config c5, obs = 64).  To stay within 1e-5 of the float64 reference, every fp32 operand
// is split into a tf32 "hi" (round-to-nearest) and a "lo" remainder and three MMAs are accumulated
// per K step: lo*hi + hi*lo first, hi*hi last (the dropped lo*lo term is ~2^-22 relative; the
// small terms go first so that only the last additions into the accumulator are full-magnitude).
//
// The accumulator of a 32-unit slice of the hidden layer is 16 registers per thread, so the CUDA
// cores see each hidden activation exactly once, in the registers wgmma left it in: bias, ReLU and
// the small second layer (<= 32 outputs) run on the thread's two rows and eight columns, and the four
// threads of a quad that share a row combine their partial sums with two shuffles (fixed order).
//
// One CTA = kWG independent warpgroups, each owning its own 64-row tiles; the weights W1 hi / lo of
// up to 256 hidden units (a "block") sit in shared memory and are shared.  At one K atom (O <= 32)
// the x tile is wgmma's A operand straight from registers: each thread loads the x elements of its
// own fragment slots from global memory and splits them, so nothing is staged and the tile loop has
// no barrier but the ping-pong turns of the two warpgroups' MMA batches (fwd_rs_body).  With two or
// four K atoms the tile is split into per-warpgroup hi / lo stages in shared memory instead
// (fwd_ss_body).  While one
// warpgroup runs its epilogue the other warpgroups' MMAs keep the tensor cores busy, and every
// warpgroup has the next tile's x in flight in registers while it computes the current one.  Wider hidden
// layers walk their blocks in passes: out[row] = ((b2 + z_0) + z_1) + ...  where the thread that
// owns a row adds the block's partial second-layer sum to what the SAME thread wrote in the
// previous pass (fixed order, bitwise reproducible, no workspace).
#include "mlp_fwd_tc.cuh"
#include "phase_clocks.cuh"
#include "tc_common.cuh"

namespace {

constexpr int kWG = 2;                      // warpgroups per CTA
constexpr int kThreads = kWG * 128;
constexpr int kXAtomBytes = kTileM * 128;   // 8 KiB: 64 rows x 32 floats

// At one K atom the x tile is the wgmma A operand straight from registers; with more atoms the tile is
// staged in shared memory (at two atoms the register path held 185 registers and took 12 % longer at
// BASELINE c5; at four the fragments alone would take 128 registers).
__host__ __device__ constexpr bool x_in_regs(int ka) { return ka == 1; }

__host__ __device__ constexpr size_t fwd_smem_bytes(int hb, int ka, int np) {
    return 1024 /*alignment slack*/ + (size_t)2 * ka * hb * 128 +
           (x_in_regs(ka) ? 0 : (size_t)kWG * 2 * ka * kXAtomBytes) + (size_t)hb * (w2s_stride(np) + 1) * sizeof(float);
}

// Stage one pass's W1 rows (hi / lo swizzled K-major tiles), b1 and W2 (transposed, rows padded to NPS).
// The weights are read L2-cold at the start of a step, so each thread keeps kStageLd loads in flight
// before it stores any of them (one dependent load per loop trip would put every one of them on the
// launch's critical path).
constexpr int kStageLd = 8;

template <int NP, int KA>
__device__ __forceinline__ void stage_weights(const FwdTcArgs& a, int p, uint8_t* w_hi, uint8_t* w_lo, float* b1s,
                                              float* w2s) {
    constexpr int NPS = w2s_stride(NP);
    const int HB = a.hb, ochunks = a.O >> 2, tid = threadIdx.x;
    const float* __restrict__ W1 = a.params + a.lay.oW1;
    const float* __restrict__ b1 = a.params + a.lay.ob1;
    const float* __restrict__ W2 = a.params + a.lay.oW2;
    const int n_w1 = HB * 8 * KA, n_w2 = HB * NP;
    for (int base = tid; base < n_w1; base += kStageLd * kThreads) {
        float4 w[kStageLd];
#pragma unroll
        for (int u = 0; u < kStageLd; ++u) {
            const int idx = base + u * kThreads, r = idx / (8 * KA), c = idx % (8 * KA);
            w[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (idx < n_w1 && c < ochunks) w[u] = __ldg(reinterpret_cast<const float4*>(W1 + (size_t)(p * HB + r) * a.O) + c);
        }
#pragma unroll
        for (int u = 0; u < kStageLd; ++u) {
            const int idx = base + u * kThreads, r = idx / (8 * KA), c = idx % (8 * KA);
            if (idx < n_w1) {
                float4 hi, lo;
                tc::split4(w[u], hi, lo);
                const uint32_t off = (c >> 3) * (HB * 128) + tc::sw128_offset(r, c & 7);
                *reinterpret_cast<float4*>(w_hi + off) = hi;
                *reinterpret_cast<float4*>(w_lo + off) = lo;
            }
        }
    }
    for (int idx = tid; idx < HB; idx += kThreads) b1s[idx] = __ldg(b1 + p * HB + idx);
    for (int base = tid; base < n_w2; base += kStageLd * kThreads) {
        float w[kStageLd];
#pragma unroll
        for (int u = 0; u < kStageLd; ++u) {
            const int idx = base + u * kThreads, j = idx / NP, n = idx - j * NP;
            w[u] = idx < n_w2 && n < a.N2 ? __ldg(W2 + (size_t)n * a.H + p * HB + j) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < kStageLd; ++u) {
            const int idx = base + u * kThreads, j = idx / NP, n = idx - j * NP;
            if (idx < n_w2) w2s[j * NPS + n] = w[u];
        }
    }
}

// One CTA's share of a network: CTA `cta` of `ncta`; warpgroup w takes tiles u, u + ncta * kWG, ...
// with u = cta * kWG + w (a launch may give different CTA ranges to different networks).
//
// x fragments in registers (one K atom).  Thread (warp, g, q) owns rows 16 warp + g and + 8
// of the tile in both the A fragment and the accumulator, so it loads its own features 8 kk + q and
// 8 kk + q + 4 of those two rows straight from global memory: nothing is staged, and a warpgroup
// waits for the other only for its turn to issue.  The next tile's raw values are in flight in xr while
// the current tile computes; they are split into hi / lo after the tile's last MMA batch has retired.  Only W1
// is read from shared memory (1 KB per MMA instead of 3 KB), and the tile loop has no barrier but the
// ping-pong turns below.
// The 32-unit slices go to the tensor cores two at a time, as one m64n64 MMA chain into one
// 32-register accumulator (see `issue`): a tile waits on 4 batches instead of 8, and issues 9 MMAs per
// batch instead of 18.
template <int NP, int KA, bool SPLIT = false>
__device__ __forceinline__ void fwd_rs_body(const FwdArgs<SPLIT>& a, const int cta, const int ncta) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const int HB = a.hb;
    uint8_t* w_hi = smem;  // [KA atoms][HB rows][128 B]
    uint8_t* w_lo = w_hi + KA * HB * 128;
    float* b1s = reinterpret_cast<float*>(smem + 2 * KA * HB * 128);  // [HB]
    float* w2s = b1s + HB;                                             // [HB][NPS]
    // the warpgroup index broadcast from lane 0: known warp-uniform, or ptxas takes the turn barriers for
    // divergent code and serializes every wgmma (C7520)
    const int wg = __shfl_sync(IMPALA_FULL_MASK, (int)threadIdx.x >> 7, 0);
    const int tid = threadIdx.x, warp = (tid >> 5) & 3, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int O = a.O, ksteps = (O + 7) >> 3, nslices = HB / 32;
    const int unit = cta * kWG + wg, nunits = ncta * kWG;

    constexpr int KS = 4 * KA;  // K steps of 8 features
    float xr[KS][4];            // next tile, raw: A fragment slot i = row + 8 (i & 1), feature 8 kk + q + 4 (i >> 1)
    uint32_t xh[KS][4], xl[KS][4];
    auto load = [&](int tile) {
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = tile * kTileM + 16 * warp + g + 8 * (i & 1), f = 8 * kk + q + 4 * (i >> 1);
                xr[kk][i] = 0.f;
                if (kk < ksteps && tile < a.num_tiles && row < a.M && f < O) xr[kk][i] = __ldg(a.x + (size_t)row * O + f);
            }
        }
    };
    // One MMA batch over the slices from nc on that the accumulator holds: two (32 registers, one
    // m64n64 MMA per product, B = W1 rows [32 nc, 32 nc + 64), contiguous in the swizzled tile) or one
    // (the odd slice, m64n32); lo * hi + hi * lo over all K steps first, hi * hi last (see the header).
    // The MMAs form one dependent chain.  Descriptors = W1 hi / lo's plus the operand's offset in 16-byte
    // units (start address field); the bases are opaque per batch, or every descriptor is hoisted
    // into a register pair of its own.
    const uint64_t dw_hi = tc::smem_desc_k_sw128(w_hi, 0), dw_lo = tc::smem_desc_k_sw128(w_lo, 0);
    auto issue = [&](auto& d, int nc) {
        constexpr int ND = sizeof(d) / sizeof(float);
        auto mma = [&](const uint32_t(&x)[4], uint64_t bw, bool acc) {
            if constexpr (ND == 32) tc::wgmma_n64_rs(d, x, bw, acc);
            else tc::wgmma_n32_rs(d, x, bw, acc);
        };
        uint64_t bw_hi = dw_hi, bw_lo = dw_lo;
        asm volatile("" : "+l"(bw_hi), "+l"(bw_lo));
        auto wo = [&](int kk) -> uint32_t { return ((kk >> 2) * (HB * 128) + nc * 32 * 128 + (kk & 3) * 32) >> 4; };
#pragma unroll
        for (int i = 0; i < ND; ++i) d[i] = 0.f;
        tc::fence_acc(d);  // zeroed before the warpgroup fence (see mlp_bwd_tc.cu)
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
            if (kk < ksteps) {
                mma(xl[kk], bw_hi + wo(kk), kk > 0);
                mma(xh[kk], bw_lo + wo(kk), true);
            }
        }
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
            if (kk < ksteps) mma(xh[kk], bw_hi + wo(kk), true);
        }
        tc::wgmma_commit();
    };

    // Ping-pong: the warpgroups take turns to issue an MMA batch, batch 0 of warpgroup 0, batch 0 of
    // warpgroup 1, batch 1 of 0, ..., so that one warpgroup's epilogue runs while the other's MMAs execute.
    // Turn barrier 3 + w (256 threads) is warpgroup w's: it syncs on its own before the issue and arrives on
    // the other's after the commit.  Within a pass warpgroup 0 takes nb turns per tile and warpgroup 1 as many
    // (one tile fewer: it takes that tile's nb turns empty); warpgroup 0 skips the sync of its first turn,
    // warpgroup 1 the arrival of its last, so both barriers are back at zero at the pass's closing
    // __syncthreads (tests/test_pingpong_protocol_cpu.py models the sequence: fwd_ops there restates `turn`,
    // `pass_turn` and the empty turns after the tile loop, and changes with them).
    const int nb = (nslices + 1) / 2;  // MMA batches per tile
    auto turn = [&](bool first) { tc::named_bar_if(wg == 1 || !first, 3 + wg, 256); };
    auto pass_turn = [&](bool last, int tile) {  // after the commit; last: the tile's last batch
        tc::named_bar_arrive_if(wg == 0 || !last || tile - 1 + nunits < a.num_tiles, 4 - wg, 256);
    };
    PHASE_BEGIN(wg);
    const int npass = a.H / HB;
    for (int p = 0; p < npass; ++p) {
        load(unit);       // in flight during the weight staging
        __syncthreads();  // the previous pass is done with the weights
        stage_weights<NP, KA>(a, p, w_hi, w_lo, b1s, w2s);
        tc::fence_proxy_async();
        __syncthreads();
        PHASE_MARK(wg, 5);

        int tile = unit;
        for (; tile < a.num_tiles; tile += nunits) {
            PHASE_TILE(wg);
            // the previous tile's MMAs have all retired: its fragments may be overwritten
#pragma unroll
            for (int kk = 0; kk < KS; ++kk) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float hi, lo;
                    tc::split_tf32(xr[kk][i], hi, lo);
                    xh[kk][i] = __float_as_uint(hi), xl[kk][i] = __float_as_uint(lo);
                }
                tc::fence_frag(xh[kk]);
                tc::fence_frag(xl[kk]);
            }
            load(tile + nunits);  // in flight during this tile's MMAs and epilogue
            PHASE_MARK(wg, 2);

            float p0[NP], p1[NP];
#pragma unroll
            for (int n = 0; n < NP; ++n) p0[n] = 0.f, p1[n] = 0.f;
            int nc = 0;
            for (; nc + 2 <= nslices; nc += 2) {
                float d[32];
                turn(tile == unit && nc == 0);
                PHASE_MARK(wg, 4);
                PHASE_GEMM_ON(wg);
                issue(d, nc);
                pass_turn(nc + 2 >= nslices, tile);
                tc::wgmma_wait<0>();
                tc::fence_acc(d);
                PHASE_GEMM_OFF(wg);
                PHASE_MARK(wg, 0);
                slice_epilogue<NP>(d, nc, q, b1s, w2s, p0, p1);
                PHASE_MARK(wg, 1);
            }
            if (nc < nslices) {  // odd number of slices (H = 32, 96, 160, 224)
                float d[16];
                turn(tile == unit && nc == 0);
                PHASE_MARK(wg, 4);
                PHASE_GEMM_ON(wg);
                issue(d, nc);
                pass_turn(true, tile);
                tc::wgmma_wait<0>();
                tc::fence_acc(d);
                PHASE_GEMM_OFF(wg);
                PHASE_MARK(wg, 0);
                slice_epilogue<NP>(d, nc, q, b1s, w2s, p0, p1);
                PHASE_MARK(wg, 1);
            }
            write_rows<NP, SPLIT>(a, p, tile, warp, g, q, p0, p1);
            PHASE_MARK(wg, 3);
        }
        // warpgroup 1 with one tile fewer in the pass (tile - 1: warpgroup 0's next): its empty turns
        if (wg == 1 && tile - 1 < a.num_tiles) {
            for (int b = 0; b < nb; ++b) {
                tc::named_bar(4, 256);
                if (b + 1 < nb) tc::named_bar_arrive(3, 256);
            }
        }
    }
    PHASE_SYNC();
    PHASE_END(wg);
}

// x tile staged in shared memory (four K atoms): each warpgroup splits it into its own hi / lo
// swizzled tiles, and every slice waits for its MMAs before its epilogue.
template <int NP, int KA, bool SPLIT = false>
__device__ __forceinline__ void fwd_ss_body(const FwdArgs<SPLIT>& a, const int cta, const int ncta) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment (SWIZZLE_128B atoms) by OFFSETTING the __shared__ array
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const int HB = a.hb;
    uint8_t* w_hi = smem;                          // [KA atoms][HB rows][128 B]
    uint8_t* w_lo = w_hi + KA * HB * 128;
    const int tid = threadIdx.x, wg = tid >> 7, lt = tid & 127, warp = lt >> 5, lane = tid & 31;
    uint8_t* x_hi = w_lo + KA * HB * 128 + wg * 2 * KA * kXAtomBytes;  // this warpgroup's [KA][64 rows][128 B]
    uint8_t* x_lo = x_hi + KA * kXAtomBytes;
    float* b1s = reinterpret_cast<float*>(smem + 2 * KA * HB * 128 + kWG * 2 * KA * kXAtomBytes);  // [HB]
    float* w2s = b1s + HB;                                                                         // [HB][NPS]

    const int O = a.O, ochunks = O >> 2, ksteps = (O + 7) >> 3;
    const int unit = cta * kWG + wg, nunits = ncta * kWG;
    const int g = lane >> 2, q = lane & 3;

    // x rows of a tile -> registers: chunk idx = lt + 128 k is (row idx / (8 KA), 16-byte chunk idx % (8 KA))
    constexpr int kLd = 4 * KA;
    float4 v[kLd];
    auto load = [&](int tile) {
#pragma unroll
        for (int k = 0; k < kLd; ++k) {
            const int idx = lt + 128 * k, r = idx / (8 * KA), c = idx % (8 * KA);
            const int row = tile * kTileM + r;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tile < a.num_tiles && row < a.M && c < ochunks)
                v[k] = __ldg(reinterpret_cast<const float4*>(a.x + (size_t)row * O) + c);
        }
    };

    const int npass = a.H / HB;
    for (int p = 0; p < npass; ++p) {
        load(unit);       // in flight during the weight staging
        __syncthreads();  // the previous pass is done with the weights
        stage_weights<NP, KA>(a, p, w_hi, w_lo, b1s, w2s);
        tc::fence_proxy_async();
        __syncthreads();

        for (int tile = unit; tile < a.num_tiles; tile += nunits) {
            // ---- x tile -> hi / lo swizzled tiles (the warpgroup's previous MMAs have all retired)
            tc::named_bar(1 + wg, 128);
#pragma unroll
            for (int k = 0; k < kLd; ++k) {
                const int idx = lt + 128 * k, r = idx / (8 * KA), c = idx % (8 * KA);
                float4 hi, lo;
                tc::split4(v[k], hi, lo);
                const uint32_t off = (c >> 3) * kXAtomBytes + tc::sw128_offset(r, c & 7);
                *reinterpret_cast<float4*>(x_hi + off) = hi;
                *reinterpret_cast<float4*>(x_lo + off) = lo;
            }
            tc::fence_proxy_async();
            tc::named_bar(1 + wg, 128);
            load(tile + nunits);  // in flight during this tile's MMAs and epilogue

            float p0[NP], p1[NP];  // partial second-layer sums of rows 16 warp + g and + 8
#pragma unroll
            for (int n = 0; n < NP; ++n) p0[n] = 0.f, p1[n] = 0.f;
            for (int nc = 0; nc < HB / 32; ++nc) {
                float d[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) d[i] = 0.f;
                tc::fence_acc(d);  // zeroed before the warpgroup fence (see mlp_bwd_tc.cu)
                tc::wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t xo = (kk >> 2) * kXAtomBytes + (kk & 3) * 32;
                        const uint32_t wo = (kk >> 2) * (HB * 128) + nc * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d, tc::smem_desc_k_sw128(x_lo, xo), tc::smem_desc_k_sw128(w_hi, wo), kk > 0);
                        tc::wgmma_n32_ss(d, tc::smem_desc_k_sw128(x_hi, xo), tc::smem_desc_k_sw128(w_lo, wo), true);
                    }
                }
#pragma unroll
                for (int kk = 0; kk < 4 * KA; ++kk) {
                    if (kk < ksteps) {
                        const uint32_t xo = (kk >> 2) * kXAtomBytes + (kk & 3) * 32;
                        const uint32_t wo = (kk >> 2) * (HB * 128) + nc * 32 * 128 + (kk & 3) * 32;
                        tc::wgmma_n32_ss(d, tc::smem_desc_k_sw128(x_hi, xo), tc::smem_desc_k_sw128(w_hi, wo), true);
                    }
                }
                tc::wgmma_commit();
                tc::wgmma_wait<0>();
                tc::fence_acc(d);
                slice_epilogue<NP>(d, nc, q, b1s, w2s, p0, p1);
            }
            write_rows<NP, SPLIT>(a, p, tile, warp, g, q, p0, p1);
        }
    }
}

template <int NP, int KA>
__global__ void __launch_bounds__(kThreads) mlp_fwd_tc_kernel(const __grid_constant__ FwdTcArgs a) {
    if constexpr (x_in_regs(KA)) fwd_rs_body<NP, KA>(a, blockIdx.x, gridDim.x);
    else fwd_ss_body<NP, KA>(a, blockIdx.x, gridDim.x);
}

// Its split-head twin (shared-torso networks, NP >= 4 only): a kernel of its own name and arguments, so the
// kernels of the interleaved layout keep theirs
template <int NP, int KA>
__global__ void __launch_bounds__(kThreads) mlp_fwd_tc_split_kernel(const __grid_constant__ FwdTcSplitArgs a) {
    if constexpr (x_in_regs(KA)) fwd_rs_body<NP, KA, true>(a, blockIdx.x, gridDim.x);
    else fwd_ss_body<NP, KA, true>(a, blockIdx.x, gridDim.x);
}

// Policy and value network of one learner step in ONE launch: CTAs [0, n_pi) run the policy
// tiles, the rest the value-function tiles.  Both read the same observations; one launch means
// one weight staging per CTA and a finer tile quantisation than two launches.  Both networks run
// through ONE body instantiation (NP = 4; the value function's W2 rows are zero-padded to 4 outputs,
// and its output 0 takes exactly the FMAs, in the same order, of the one-output epilogue): with a
// branch on the network around two instantiations, or around the epilogue form, ptxas serializes
// every wgmma of the kernel (C7520, a compiler-inserted warpgroup arrive in a divergent path).  The
// arguments are selected field by field for the same reason.
__global__ void __launch_bounds__(kThreads)
mlp_fwd_tc_pair_kernel(const __grid_constant__ FwdTcArgs a_pi, const __grid_constant__ FwdTcArgs a_vf,
                       const int n_pi) {
    const bool pi = (int)blockIdx.x < n_pi;
    FwdTcArgs a = a_pi;
    a.params = pi ? a_pi.params : a_vf.params, a.out = pi ? a_pi.out : a_vf.out;
    a.M = pi ? a_pi.M : a_vf.M, a.H = pi ? a_pi.H : a_vf.H, a.N2 = pi ? a_pi.N2 : a_vf.N2;
    a.num_tiles = pi ? a_pi.num_tiles : a_vf.num_tiles, a.hb = pi ? a_pi.hb : a_vf.hb;
    a.lay.oW1 = pi ? a_pi.lay.oW1 : a_vf.lay.oW1, a.lay.ob1 = pi ? a_pi.lay.ob1 : a_vf.lay.ob1;
    a.lay.oW2 = pi ? a_pi.lay.oW2 : a_vf.lay.oW2, a.lay.ob2 = pi ? a_pi.lay.ob2 : a_vf.lay.ob2;
    fwd_rs_body<4, 1>(a, pi ? (int)blockIdx.x : (int)blockIdx.x - n_pi, pi ? n_pi : (int)gridDim.x - n_pi);
}

FwdTcArgs make_fwd_args(const float* x, const float* params, float* out, int M, int O, int H, int N2, int hb) {
    FwdTcArgs a{};
    a.x = x, a.params = params, a.out = out;
    a.M = M, a.O = O, a.H = H, a.N2 = N2;
    a.num_tiles = (M + kTileM - 1) / kTileM;
    a.hb = hb;
    a.lay = impala_make_layout(O, H, N2);
    return a;
}

// Resident CTAs of `kernel` on the whole device at `smem` bytes.
int resident_grid(const void* kernel, size_t smem, int* grid) {
    int per_sm = 0, sms = 0;
    cudaError_t e;
    if ((e = impala_resident_ctas(kernel, kThreads, smem, &per_sm)) != cudaSuccess) return (int)e;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    if (per_sm < 1) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    *grid = per_sm * sms;
    return IMPALA_OK;
}

template <int NP, int KA, bool SPLIT = false>
int launch_fwd(const FwdArgs<SPLIT>& a, cudaStream_t st) {
    const size_t smem = fwd_smem_bytes(a.hb, KA, NP);
    const void* kernel;
    if constexpr (SPLIT) kernel = (const void*)mlp_fwd_tc_split_kernel<NP, KA>;
    else kernel = (const void*)mlp_fwd_tc_kernel<NP, KA>;
    int grid = 0;
    const int rc = resident_grid(kernel, smem, &grid);
    if (rc != IMPALA_OK) return rc;
    const int want = (a.num_tiles + kWG - 1) / kWG;
    if constexpr (SPLIT) mlp_fwd_tc_split_kernel<NP, KA><<<want < grid ? want : grid, kThreads, smem, st>>>(a);
    else mlp_fwd_tc_kernel<NP, KA><<<want < grid ? want : grid, kThreads, smem, st>>>(a);
    return impala_launch_status();
}

template <int KA>
int launch_fwd_ka(int np, const FwdTcSplitArgs& a, cudaStream_t st) {
    if (a.out_b)  // split heads: N2 >= 2, so np >= 4
        return np == 4 ? launch_fwd<4, KA, true>(a, st) : np == 16 ? launch_fwd<16, KA, true>(a, st)
                                                        : launch_fwd<32, KA, true>(a, st);
    return np == 1 ? launch_fwd<1, KA>(a, st) : np == 4 ? launch_fwd<4, KA>(a, st)
                   : np == 16 ? launch_fwd<16, KA>(a, st) : launch_fwd<32, KA>(a, st);
}

}  // namespace

int impala_mlp_fwd_tc(const MlpPlan& p, const float* x, const float* params, float* out, int M, int O, int H, int N2,
                      cudaStream_t st, float* out_b, int M_a) {
    const FwdTcSplitArgs a{make_fwd_args(x, params, out, M, O, H, N2, p.hb), out_b, M_a};
    return p.ka == 1 ? launch_fwd_ka<1>(p.np, a, st) : p.ka == 2 ? launch_fwd_ka<2>(p.np, a, st)
                                                     : launch_fwd_ka<4>(p.np, a, st);
}

// Both networks in one launch (policy: 2..4 outputs, value fn: 1 output); the caller has routed each
// to a Narrow plan, which holds the whole hidden layer in one pass.  Per-tile cost weights split the
// CTAs between the two tile lists; both networks run the same MMAs and the same 4-output epilogue per
// tile, so the default weighs a policy tile as one value-function tile.
int impala_mlp_fwd_tc_pair(const float* x, const float* params_pi, const float* params_vf, float* logits,
                           float* values, int M_pi, int M_vf, int O, int H_pi, int H_vf, int A,
                           cudaStream_t st) {
    const FwdTcArgs a_pi = make_fwd_args(x, params_pi, logits, M_pi, O, H_pi, A, H_pi);
    const FwdTcArgs a_vf = make_fwd_args(x, params_vf, values, M_vf, O, H_vf, 1, H_vf);
    // both networks stage W2 in the 4-output layout (one body instantiation, see the kernel)
    const size_t s_pi = fwd_smem_bytes(a_pi.hb, 1, 4), s_vf = fwd_smem_bytes(a_vf.hb, 1, 4);
    const size_t smem = s_pi > s_vf ? s_pi : s_vf;
    int grid = 0;
    const int rc = resident_grid((const void*)mlp_fwd_tc_pair_kernel, smem, &grid);
    if (rc != IMPALA_OK) return rc;
    const int units_pi = (a_pi.num_tiles + kWG - 1) / kWG, units_vf = (a_vf.num_tiles + kWG - 1) / kWG;
    if (grid > units_pi + units_vf) grid = units_pi + units_vf;
    const int n_pi = impala_pair_split(units_pi, units_vf, grid,
                                       impala_env_int("IMPALA_PAIR_W_FWD", 100) * (H_pi / 32),
                                       100 * (H_vf / 32));
    mlp_fwd_tc_pair_kernel<<<grid, kThreads, smem, st>>>(a_pi, a_vf, n_pi);
    return impala_launch_status();
}

#ifdef IMPALA_PHASE_CLOCKS
IMPALA_PHASE_READER(impala_phase_read_fwd)
#endif
