// V-trace targets, the three losses and their closed-form backward
// (reference learner.py:116-162 + helpers :298-321 + the non-MLP part of :175).
//
// The kernel body and its launcher; vtrace_loss.cu holds the entry points of the plain, diag and PopArt
// kernels, vtrace_loss_rclip.cu those of the reward-clipping ones and vtrace_loss_gauss.cu those of the
// diagonal-Gaussian policies, vtrace_loss_md.cu those of the multi-discrete ones and vtrace_loss_mask.cu those of
// the masked categorical and multi-discrete ones (separate translation units, so the parallel build compiles the
// sets of instantiations side by side).
//
// Lane = trajectory, warp = time segment (vtrace_lane_kernel below): every tensor of the
// time-major (T, B[, A]) batch is read and written as fully coalesced row segments straight from /
// to global memory (128-bit accesses for the logits), the T-step recurrence is split over the
// warps of a CTA as composed affine maps (one barrier per chunk), and everything else stays in
// registers.
//
// Transcendentals use the hardware approximations (ex2/lg2.approx.ftz, relative error ~2^-22) in
// the base-2 domain: the arguments are differences from the row maximum (<= 0) and sums in
// [1, A], so the absolute error stays ~1e-7, far inside the 1e-5 parity budget, at a fraction of
// the instruction count of expf/logf.
//
// Reference quirks reproduced in IMPALA_MODE_REFERENCE (SURVEY.md section 0.2):
//   delta_t = rho_t (r_t + gamma v_{t+1} - v_0)                  learner.py:126  (v[:1])
//   acc_i   = delta_i + disc_i c_i (acc_{i+1} - v_{i+1})          learner.py:130
//   vs = acc + v (:131);  pg_t = rho_t (r_t + disc_t vs_{t+1} - v_t)   (:135)
// i.e. the affine map F_i(x) = (delta_i - g_i v_{i+1}) + g_i x with g_i = disc_i c_i.
#pragma once
#include <cooperative_groups.h>
#include <math.h>

#include <cstdlib>
#include <type_traits>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace {

// ex2 / lg2 hardware approximations with flush-to-zero (no denormal fix-up code): relative error
// ~2^-22.  Softmax is evaluated in the base-2 domain: zs = z * log2(e), p_k = 2^(zs_k - lse2).
__device__ __forceinline__ float ex2f(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float lg2f(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
// p ? x : y as an opaque selp: a plain C++ select chain over the logits of a step ("the logit of the
// taken action") is turned into a dynamically indexed load by the compiler, which sends the whole
// register array to local memory.
__device__ __forceinline__ float selp_f32(bool p, float x, float y) {
    float d;
    asm("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %3, 0;\n\tselp.f32 %0, %1, %2, q;\n\t}" : "=f"(d) : "f"(x), "f"(y), "r"((int)p));
    return d;
}

// MASK: a step's legal word with the bits >= A dropped; no legal bit makes the whole row legal (padded steps, the
// empty columns of replay)
__device__ __forceinline__ unsigned legal_row(unsigned w, int A) {
    const unsigned all = A >= 32 ? ~0u : (1u << A) - 1u;
    w &= all;
    return w ? w : all;
}

// MASK: the illegal entries of a row (lg: legal_row) set to -inf by selects, so that whatever the row held there (raw
// logits, -inf, NaN) is gone: the maximum and log-sum-exp of the legal entries follow with the unmasked arithmetic
// (2^-inf = 0 adds exactly zero), and every later use tests the entry against -inf.  With every bit set nothing changes.
template <int AP>
__device__ __forceinline__ void mask_row(unsigned lg, float (&z)[AP]) {
#pragma unroll
    for (int k = 0; k < AP; ++k) z[k] = ((lg >> k) & 1u) ? z[k] : -INFINITY;
}
// legal entry test of a masked row (log2 pi or a shifted logit: -inf exactly where mask_row put it)
__device__ __forceinline__ bool is_legal(float x) { return x != -INFINITY; }

constexpr int kMaxSeg = 32;  // time segments (= warps) per CTA

struct VtArgs {
    const float* cur_logits;
    const float* beh_logits;
    const int32_t* actions;
    const float* rewards;
    const uint8_t* done;
    const int32_t* lens;
    const float* v;
    float* vs;
    float* pg_adv;
    float* dlogits;
    float* dv;
    double* scalars;
    double* partials;        // [gridDim.x][4] per-CTA loss sums ([12] with the off-policy sums; workspace)
    unsigned int* counter;   // CTA arrival counter (workspace; zero on entry, zero on exit)
    int T, B, A, mode;
    float gamma, rho_bar, c_bar, v_loss_c, policy_loss_c, entropy_c, inv_batch;
};
// DIAG instantiations take the off-policy sums' destination as well (the others keep VtArgs, so their
// parameter block and code are those of the plain loss kernel).
struct VtDiagArgs : VtArgs {
    double* diag;  // [8] sums over the valid steps, see impala_vtrace_loss_diag
};
// POPART instantiations (on top of DIAG) read the value statistics as well: v is the normalized output.
struct VtPopArgs : VtDiagArgs {
    const double* popart;  // {mu, nu, sigma, ...}, see impala_vtrace_loss_popart
};
// RCLIP instantiations (on top of any of the three) take the reward transform as well.
template <class Base>
struct VtClipArgs : Base {
    int reward_clip;  // IMPALA_REWARD_CLIP_*
};
template <bool DIAG, bool POPART = false>
using VtArgsB = typename std::conditional<POPART, VtPopArgs,
                                          typename std::conditional<DIAG, VtDiagArgs, VtArgs>::type>::type;
template <bool DIAG, bool POPART = false, bool RCLIP = false>
using VtArgsT = typename std::conditional<RCLIP, VtClipArgs<VtArgsB<DIAG, POPART>>, VtArgsB<DIAG, POPART>>::type;
// MD instantiations (on top of any of the above) take the multi-discrete heads as well, by value.
template <class Base>
struct VtMdArgs : Base {
    unsigned head_mask;  // bit j set: policy output j is the first of a head (bit 0 always set)
};
template <bool DIAG, bool POPART = false, bool RCLIP = false, bool MD = false>
using VtArgsM = typename std::conditional<MD, VtMdArgs<VtArgsT<DIAG, POPART, RCLIP>>, VtArgsT<DIAG, POPART, RCLIP>>::type;

// The reward transform of the RCLIP instantiations (DeepMind's IMPALA `reward_clipping`), with compares and
// selects rather than fminf / fmaxf so that a NaN reward stays NaN (as torch.clamp keeps it): abs_one is
// clip(r, -1, 1); soft_asymmetric is 5 tanh(r / 5) for r >= 0 and 1.5 tanh(r / 5) for r < 0 (full-precision
// tanhf).  +-inf saturates: +-1, and 5 / -1.5.
__device__ __forceinline__ float clip_reward(float r, int mode) {
    if (mode == IMPALA_REWARD_CLIP_ABS_ONE) {
        r = r > 1.f ? 1.f : r;
        return r < -1.f ? -1.f : r;
    }
    const float t = tanhf(r * 0.2f);
    return r < 0.f ? 1.5f * t : 5.f * t;
}

// Row loads / stores of the (T, B, A) logits: lane = trajectory, so a warp reads 32 * A consecutive
// floats of a time step.  VEC (A == AP, 16-byte aligned bases): one 128-bit (A = 4), one 64-bit
// (A = 2) or AP/4 128-bit accesses per lane, i.e. 512 contiguous bytes per warp instruction at A = 4.
template <int AP, bool VEC>
__device__ __forceinline__ void load_logits(const float* __restrict__ p, unsigned elem, int A, float (&z)[AP]) {
    if constexpr (VEC && AP == 2) {
        const float2 q = __ldg(reinterpret_cast<const float2*>(p + elem * 2));
        z[0] = q.x, z[1] = q.y;
    } else if constexpr (VEC) {
#pragma unroll
        for (int k = 0; k < AP; k += 4) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(p + elem * AP + k));
            z[k] = q.x, z[k + 1] = q.y, z[k + 2] = q.z, z[k + 3] = q.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < AP; ++k) z[k] = k < A ? __ldg(p + elem * A + k) : 0.f;
    }
}
template <int AP, bool VEC>
__device__ __forceinline__ void store_logits(float* __restrict__ p, unsigned elem, int A, const float (&z)[AP]) {
    if constexpr (VEC && AP == 2) {
        *reinterpret_cast<float2*>(p + elem * 2) = make_float2(z[0], z[1]);
    } else if constexpr (VEC) {
#pragma unroll
        for (int k = 0; k < AP; k += 4)
            *reinterpret_cast<float4*>(p + elem * AP + k) = make_float4(z[k], z[k + 1], z[k + 2], z[k + 3]);
    } else {
#pragma unroll
        for (int k = 0; k < AP; ++k)
            if (k < A) p[elem * A + k] = z[k];
    }
}

// Streaming log-softmax of one (T, B, A) row for the wide action sets (AP > 16), where the
// whole-row register arrays of the other instantiations no longer fit: the row is loaded, reduced
// and dropped.  Returns the base-2 shift -max * log2(e) and lse2 = log2 sum_k 2^(z_k log2(e) - max
// log2(e)), so log2 pi(k) = fmaf(z_k, log2(e), shift) - lse2; *za is the shifted logit of `act`.
// MASK: over the entries of the legal word lg only (mask_row: the illegal ones are -inf, 2^-inf adds exactly 0).
template <int AP, bool VEC, bool MASK = false>
__device__ __forceinline__ void row_lse2(const float* __restrict__ p, unsigned elem, int A, int act, float* shift,
                                         float* lse2, float* za, unsigned lg = 0u) {
    float z[AP];
    load_logits<AP, VEC>(p, elem, A, z);
    if constexpr (MASK) mask_row<AP>(lg, z);
    float mx = z[0];
#pragma unroll
    for (int k = 1; k < AP; ++k)
        if (k < A) mx = fmaxf(mx, z[k]);
    const float sh = -mx * kLog2e;
    float se = 0.f, z_a = fmaf(z[0], kLog2e, sh);
#pragma unroll
    for (int k = 0; k < AP; ++k) {
        const float zs = fmaf(z[k], kLog2e, sh);
        if (k < A) se += ex2f(zs);
        if (k > 0) z_a = selp_f32(k == act, zs, z_a);
    }
    *shift = sh, *lse2 = lg2f(se), *za = z_a;
}

// KL(mu || pi) / ln 2 of one streaming row pair (VEC rows), from the shifts and log-sum-exps row_lse2 returned:
// both rows are read again four logits at a time (L1 / L2 hits), so no whole row is held.  MASK: the legal entries only.
template <int AP, bool MASK = false>
__device__ __forceinline__ float row_kl2(const float* __restrict__ pc, const float* __restrict__ pb, unsigned elem,
                                         float shc, float lsec, float shb, float lseb, unsigned lg = 0u) {
    float kl = 0.f;
#pragma unroll
    for (int k = 0; k < AP; k += 4) {
        const float4 qc = __ldg(reinterpret_cast<const float4*>(pc + elem * AP + k));
        const float4 qb = __ldg(reinterpret_cast<const float4*>(pb + elem * AP + k));
        const float zc[4] = {qc.x, qc.y, qc.z, qc.w}, zb[4] = {qb.x, qb.y, qb.z, qb.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float lpi = fmaf(zc[j], kLog2e, shc) - lsec, lmu = fmaf(zb[j], kLog2e, shb) - lseb;
            if (!MASK || ((lg >> (k + j)) & 1u)) kl = fmaf(ex2f(lmu), lmu - lpi, kl);
        }
    }
    return kl;
}

// ---- GAUSS: diagonal Gaussian policies.  A step's policy outputs are [m | s], 2A floats (means, then log
// standard deviations, sigma = e^s), its action the unsquashed sample, A floats.  VEC (A == AP, 16-byte aligned
// bases): 128-bit loads and stores (64-bit for the AP = 2 action row); otherwise element accesses, and the
// entries k >= A are zero, which adds exactly zero to every term below (u = 0, s = 0, sigma ratio 1).
constexpr float kHalfLog2Pi = 0.9189385332046727f;    // 1/2 log(2 pi)
constexpr float kHalfLog2PiE = 1.4189385332046727f;   // 1/2 (1 + log(2 pi)): entropy per dimension minus s_k
template <int AP, bool VEC>
__device__ __forceinline__ void load_gauss(const float* __restrict__ p, unsigned elem, int A, float (&m)[AP],
                                           float (&s)[AP]) {
    if constexpr (VEC) {
        float z[2 * AP];
        load_logits<2 * AP, true>(p, elem, 2 * AP, z);
#pragma unroll
        for (int k = 0; k < AP; ++k) m[k] = z[k], s[k] = z[AP + k];
    } else {
#pragma unroll
        for (int k = 0; k < AP; ++k) {
            m[k] = k < A ? __ldg(p + elem * 2 * A + k) : 0.f;
            s[k] = k < A ? __ldg(p + elem * 2 * A + A + k) : 0.f;
        }
    }
}
template <int AP, bool VEC>
__device__ __forceinline__ void store_gauss(float* __restrict__ p, unsigned elem, int A, const float (&dz)[2 * AP]) {
    if constexpr (VEC) {
        store_logits<2 * AP, true>(p, elem, 2 * AP, dz);
    } else {
#pragma unroll
        for (int k = 0; k < AP; ++k)
            if (k < A) p[elem * 2 * A + k] = dz[k], p[elem * 2 * A + A + k] = dz[AP + k];
    }
}
// Step 2 of one Gaussian step, reduced as the three rows load (base 2, like the categorical terms):
//   *lp2 = log2 pi(a) = log2(e) sum_k [-u_k^2 / 2 - s_k - log(2 pi) / 2],  u_k = (a_k - m_k) / sigma_k
//   *lr2 = log2 pi(a) - log2 mu(a), summed from the per-dimension differences (the constants cancel)
//   *kl2 (DIAG) = KL(mu || pi) / ln 2 = log2(e) sum_k [s_k - sb_k + (sigma_b,k^2 + (mb_k - m_k)^2) / (2 sigma_k^2) - 1/2]
template <int AP, bool VEC, bool DIAG>
__device__ __forceinline__ void gauss_terms(const float* __restrict__ pc, const float* __restrict__ pb,
                                            const float* __restrict__ pa, unsigned elem, int A, float* lp2, float* lr2,
                                            float* kl2) {
    float m[AP], s[AP], mb[AP], sb[AP], x[AP];
    load_gauss<AP, VEC>(pc, elem, A, m, s);
    load_gauss<AP, VEC>(pb, elem, A, mb, sb);
    load_logits<AP, VEC>(pa, elem, A, x);
    float q = 0.f, dq = 0.f, ss = 0.f, ds = 0.f, kl = 0.f;
#pragma unroll
    for (int k = 0; k < AP; ++k) {
        const float ic = expf(-s[k]), ib = expf(-sb[k]);  // 1 / sigma, full precision: u^2 reaches ~10
        const float u = (x[k] - m[k]) * ic, ub = (x[k] - mb[k]) * ib;
        q = fmaf(u, u, q), dq = fmaf(u - ub, u + ub, dq);  // u^2 - ub^2 per term: no cancellation of the sums
        ss += s[k], ds += sb[k] - s[k];
        if constexpr (DIAG) {
            const float r = ex2f((sb[k] - s[k]) * kLog2e), d = (mb[k] - m[k]) * ic;  // sigma_b / sigma, offset / sigma
            kl += (s[k] - sb[k]) + 0.5f * (fmaf(r, r, d * d) - 1.f);
        }
    }
    *lp2 = (fmaf(-0.5f, q, -ss) - (float)A * kHalfLog2Pi) * kLog2e;
    *lr2 = fmaf(-0.5f, dq, ds) * kLog2e;
    *kl2 = kl * kLog2e;
}

// ---- MD: multi-discrete (factorised categorical) policies.  Head k owns the policy outputs [s_k, s_k + n_k) of a
// step's A = N outputs (bit s_k of the head mask hm), its action row holds K = popc(hm) indices a_k.  Head boundaries
// are runtime values, so every sweep below walks the unrolled entries j with the head mask as a predicate (uniform
// over the grid) and never indexes a register array with a runtime value: a head's log-sum-exp is an online one,
// reset at the head's first entry, and the per-head values come back to the head's entries through a sweep in the
// other direction.  Each head is shifted by its own first logit, x_j = z_j log2(e) - z_s log2(e) (one rounding), and
// the shift cancels in log2 p_j = x_j - lse_k; the online maximum keeps every 2^(x - m) in (0, 1].  The sweeps read
// the rows four logits at a time (md_chunk; step 4's second sweep re-reads, an L1 hit).  At AP = 32 the kernel is
// bounded at 256 threads (255 registers): under the 512-thread bound of the other widths it spills.
template <int AP, bool VEC>
__device__ __forceinline__ void md_chunk(const float* __restrict__ p, unsigned elem, int A, int j0,
                                         float (&q)[AP < 4 ? AP : 4]) {
    if constexpr (VEC && AP == 2) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(p + elem * 2));
        q[0] = v.x, q[1] = v.y;
    } else if constexpr (VEC) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(p + elem * AP + j0));
        q[0] = v.x, q[1] = v.y, q[2] = v.z, q[3] = v.w;
    } else {
#pragma unroll
        for (int u = 0; u < (AP < 4 ? AP : 4); ++u) q[u] = j0 + u < A ? __ldg(p + elem * A + j0 + u) : 0.f;
    }
}
// one entry x of a head's online log-sum-exp (base 2): m the running maximum, s = sum 2^(x_i - m); returns the
// factor 2^-|x - m| and whether the maximum moved (the KL weight of the behaviour row rescales with them)
__device__ __forceinline__ bool md_online(float x, float& m, float& s, float* e) {
    const float d = x - m;
    *e = ex2f(-fabsf(d));
    const bool up = d > 0.f;
    s = up ? fmaf(s, *e, 1.f) : s + *e, m = fmaxf(m, x);
    return up;
}
// Step 2, reduced as the two rows and the K indices load (base 2, like the categorical terms):
//   *lp2 = log2 pi(a) = sum_k (x_{s_k + a_k} - lse_k),
//   *lr2 = log2 pi(a) - log2 mu(a) = sum_k [d_{s_k + a_k} - log2 sum_j mu_j 2^d_j],
//   *kl2 (DIAG) = sum_k KL_k / ln 2 = sum_k [log2 sum_j mu_j 2^d_j - sum_j mu_j d_j],
// with d_j = ((z_j - zb_j) - (z_s - zb_s)) log2(e) measured from the head's first entry s (both terms are invariant to
// it): a head the current policy shifts as a whole against the behaviour (softmax-invariant) gives d = 0, so 2^d
// overflows only where the logit differences within one head spread over ~88 nats.
// The ratio and KL come from the per-entry differences d_j (the behaviour perturbs the policy by little, so they are
// small and exact to a rounding of their own size), not from two log-sum-exps of shifted logits of magnitude ~10 per
// head: K heads of those would add K such roundings to the log ratio.  The sums over a head are online ones under the
// behaviour row's maximum; a closed head folds into a product (each sum in [1, n_k] or near 1), so a row costs few lg2.
// Returns the taken mask: bit s_k + a_k for every head (an index outside its head sets no bit).
constexpr int kMaxHeads = 16;
template <int AP, bool VEC, bool DIAG>
__device__ __forceinline__ unsigned md_terms(const float* __restrict__ pc, const float* __restrict__ pb,
                                             const int32_t* __restrict__ pa, unsigned elem, int A, unsigned hm,
                                             float* lp2, float* lr2, float* kl2) {
    constexpr int W = AP < 4 ? AP : 4;
    const int K = __popc(hm);
    unsigned taken = 0u, rest = hm;
#pragma unroll
    for (int k = 0; k < kMaxHeads; ++k) {
        if (k < K) {
            const int ak = __ldg(pa + elem * (unsigned)K + k), s = __ffs(rest) - 1;
            rest &= rest - 1u;
            const int n = (rest ? __ffs(rest) - 1 : A) - s;
            if ((unsigned)ak < (unsigned)n) taken |= 1u << (s + ak);
        }
    }
    // current row: shift sh, maximum m, sum s; behaviour row: shb, mb, sb; ub = sum 2^(xb - mb) 2^d,
    // wb = sum 2^(xb - mb) (-d).  Closed heads: msc = sum of the maxima, prc / prb / pru = products of the sums
    float shc = 0.f, shb = 0.f, rs = 0.f, mc = 0.f, sc = 1.f, mb = 0.f, sb = 1.f, ub = 1.f, wb = 0.f;
    float msc = 0.f, prc = 1.f, prb = 1.f, pru = 1.f, klw = 0.f, za = 0.f, da = 0.f;
#pragma unroll
    for (int j0 = 0; j0 < AP; j0 += W) {
        float zc[W], zb[W];
        md_chunk<AP, VEC>(pc, elem, A, j0, zc);
        md_chunk<AP, VEC>(pb, elem, A, j0, zb);
#pragma unroll
        for (int u = 0; u < W; ++u) {
            const int j = j0 + u;
            if (j < A) {
                const bool st = (hm >> j) & 1u;
                if (st) {
                    if (j > 0) {  // close the previous head
                        msc += mc, prc *= sc, prb *= sb, pru *= ub;
                        if constexpr (DIAG) klw += __fdividef(wb, sb);
                    }
                    shc = -zc[u] * kLog2e, shb = -zb[u] * kLog2e, rs = zc[u] - zb[u];
                }
                const float xc = fmaf(zc[u], kLog2e, shc), xb = fmaf(zb[u], kLog2e, shb);
                const float d = ((zc[u] - zb[u]) - rs) * kLog2e, ed = ex2f(d);
                if (st) {
                    mc = xc, sc = 1.f, mb = xb, sb = 1.f, ub = ed, wb = -d;
                } else {
                    float ec, eb;
                    md_online(xc, mc, sc, &ec);
                    const bool up = md_online(xb, mb, sb, &eb);
                    ub = up ? fmaf(ub, eb, ed) : fmaf(eb, ed, ub);
                    if constexpr (DIAG) wb = up ? fmaf(wb, eb, -d) : fmaf(eb, -d, wb);
                }
                if ((taken >> j) & 1u) za += xc, da += d;
            }
        }
    }
    msc += mc, prc *= sc, prb *= sb, pru *= ub;
    if constexpr (DIAG) klw += __fdividef(wb, sb);
    const float lrs = lg2f(pru / prb);  // sum_k log2 sum_j mu_j 2^d_j
    *lp2 = za - (msc + lg2f(prc));
    *lr2 = da - lrs;
    *kl2 = klw + lrs;
    return taken;
}
// Step 4: the current row re-read into its entropy sum_k H_k (returned) and the N gradients
//   dz_j = inv_batch [cp (p_j - [j taken]) + entropy_c p_j (ln p_j + H_k)],  cp = policy_loss_c pg_adv, zero if !valid,
// in two sweeps that each read the row and keep only dz:
//   forward:  each head's online lse and t = sum_j 2^(x_j - m) x_j, so that H_k / ln 2 = lse_k - t / s; its offset
//             c_k = sh_k - lse_k (log2 p_j = z_j log2(e) + c_k, one rounding) is left at its last entry and H_k at the
//             entry before (n_k >= 2);
//   backward: the gradient, with c_k and H_k picked up at the head's last entry.
template <int AP, bool VEC>
__device__ __forceinline__ float md_grad(const float* __restrict__ pc, unsigned elem, int A, unsigned hm,
                                         unsigned taken, bool valid, float cp, float entropy_c, float inv_batch,
                                         float (&dz)[AP]) {
    constexpr int W = AP < 4 ? AP : 4;
    const unsigned em = (hm >> 1) | (1u << (A - 1));  // bit j: output j is the last of its head
    float sh = 0.f, m = 0.f, s = 1.f, t = 0.f, ent = 0.f;
#pragma unroll
    for (int j0 = 0; j0 < AP; j0 += W) {
        float z[W];
        md_chunk<AP, VEC>(pc, elem, A, j0, z);
#pragma unroll
        for (int u = 0; u < W; ++u) {
            const int j = j0 + u;
            if (j < A) {
                const bool st = (hm >> j) & 1u;
                if (st) sh = -z[u] * kLog2e;
                const float x = fmaf(z[u], kLog2e, sh);
                if (st) {
                    m = x, s = 1.f, t = x;
                } else {
                    float e;
                    t = md_online(x, m, s, &e) ? fmaf(t, e, x) : fmaf(e, x, t);
                }
                if ((em >> j) & 1u) {
                    const float lse = m + lg2f(s), h = (lse - __fdividef(t, s)) * kLn2;
                    ent += h;
                    dz[j] = sh - lse;
                    if (j > 0) dz[j > 0 ? j - 1 : 0] = h;
                }
            }
        }
    }
    float c = 0.f, H = 0.f;
#pragma unroll
    for (int j0 = AP - W; j0 >= 0; j0 -= W) {
        float z[W];
        md_chunk<AP, VEC>(pc, elem, A, j0, z);
#pragma unroll
        for (int u = W - 1; u >= 0; --u) {
            const int j = j0 + u;
            if (j < A) {
                if ((em >> j) & 1u) {
                    c = dz[j];
                    if (j > 0) H = dz[j > 0 ? j - 1 : 0];
                }
                const float lp = fmaf(z[u], kLog2e, c), p = ex2f(lp);  // log2 p_j, p_j
                const float onehot = ((taken >> j) & 1u) ? 1.f : 0.f;
                const float d = inv_batch * (cp * (p - onehot) + entropy_c * p * (lp * kLn2 + H));
                dz[j] = valid ? d : 0.f;
            } else {
                dz[j] = 0.f;
            }
        }
    }
    return ent;
}

// md_terms for MASK (the unmasked kernels keep md_terms above, and its code): the action row is [a_0 .. a_{K-1}, legal];
// *lgo receives the legal word (legal_row, then every head without a legal bit made all-legal).  The sweep skips the
// illegal entries: a head's differences d_j and online sums start at its first legal entry, which takes the place of
// s_k.  With every bit set it is md_terms, operation for operation.
template <int AP, bool VEC, bool DIAG>
__device__ __forceinline__ unsigned md_terms_masked(const float* __restrict__ pc, const float* __restrict__ pb,
                                             const int32_t* __restrict__ pa, unsigned elem, int A, unsigned hm,
                                             float* lp2, float* lr2, float* kl2, unsigned* lgo) {
    constexpr int W = AP < 4 ? AP : 4;
    const int K = __popc(hm);
    const unsigned KW = (unsigned)K + 1u;  // int32 per action row: the K indices, the legal word
    const unsigned lg0 = legal_row((unsigned)__ldg(pa + elem * KW + K), A);
    unsigned taken = 0u, rest = hm, lg = lg0;
#pragma unroll
    for (int k = 0; k < kMaxHeads; ++k) {
        if (k < K) {
            const int ak = __ldg(pa + elem * KW + k), s = __ffs(rest) - 1;
            rest &= rest - 1u;
            const int n = (rest ? __ffs(rest) - 1 : A) - s;
            if ((unsigned)ak < (unsigned)n) taken |= 1u << (s + ak);
            const unsigned hb = (unsigned)(((1ull << n) - 1ull) << s);  // an empty head is all-legal
            if (!(lg0 & hb)) lg |= hb;
        }
    }
    *lgo = lg;
    bool fresh = false, any = false;  // no legal entry of the open head seen yet; a head opened
    // current row: shift sh, maximum m, sum s; behaviour row: shb, mb, sb; ub = sum 2^(xb - mb) 2^d,
    // wb = sum 2^(xb - mb) (-d).  Closed heads: msc = sum of the maxima, prc / prb / pru = products of the sums
    float shc = 0.f, shb = 0.f, rs = 0.f, mc = 0.f, sc = 1.f, mb = 0.f, sb = 1.f, ub = 1.f, wb = 0.f;
    float msc = 0.f, prc = 1.f, prb = 1.f, pru = 1.f, klw = 0.f, za = 0.f, da = 0.f;
#pragma unroll
    for (int j0 = 0; j0 < AP; j0 += W) {
        float zc[W], zb[W];
        md_chunk<AP, VEC>(pc, elem, A, j0, zc);
        md_chunk<AP, VEC>(pb, elem, A, j0, zb);
#pragma unroll
        for (int u = 0; u < W; ++u) {
            const int j = j0 + u;
            fresh = fresh || ((hm >> j) & 1u);
            if (j < A && ((lg >> j) & 1u)) {
                const bool st = fresh;  // the head's first legal entry
                fresh = false;
                if (st) {
                    if (any) {  // close the previous head
                        msc += mc, prc *= sc, prb *= sb, pru *= ub;
                        if constexpr (DIAG) klw += __fdividef(wb, sb);
                    }
                    any = true;
                    shc = -zc[u] * kLog2e, shb = -zb[u] * kLog2e, rs = zc[u] - zb[u];
                }
                const float xc = fmaf(zc[u], kLog2e, shc), xb = fmaf(zb[u], kLog2e, shb);
                const float d = ((zc[u] - zb[u]) - rs) * kLog2e, ed = ex2f(d);
                if (st) {
                    mc = xc, sc = 1.f, mb = xb, sb = 1.f, ub = ed, wb = -d;
                } else {
                    float ec, eb;
                    md_online(xc, mc, sc, &ec);
                    const bool up = md_online(xb, mb, sb, &eb);
                    ub = up ? fmaf(ub, eb, ed) : fmaf(eb, ed, ub);
                    if constexpr (DIAG) wb = up ? fmaf(wb, eb, -d) : fmaf(eb, -d, wb);
                }
                if ((taken >> j) & 1u) za += xc, da += d;
            }
        }
    }
    msc += mc, prc *= sc, prb *= sb, pru *= ub;
    if constexpr (DIAG) klw += __fdividef(wb, sb);
    const float lrs = lg2f(pru / prb);  // sum_k log2 sum_j mu_j 2^d_j
    *lp2 = za - (msc + lg2f(prc));
    *lr2 = da - lrs;
    *kl2 = klw + lrs;
    return taken;
}
// md_grad for MASK (lg: md_terms_masked's *lgo): the forward sweep skips the illegal entries, each head's sums
// starting at its first legal entry; the head's last entry still parks c_k and H_k, legal or not (n_k >= 2 is the head
// size); the gradient is exactly zero at illegal entries.
template <int AP, bool VEC>
__device__ __forceinline__ float md_grad_masked(const float* __restrict__ pc, unsigned elem, int A, unsigned hm,
                                         unsigned taken, bool valid, float cp, float entropy_c, float inv_batch,
                                         float (&dz)[AP], unsigned lg) {
    constexpr int W = AP < 4 ? AP : 4;
    const unsigned em = (hm >> 1) | (1u << (A - 1));  // bit j: output j is the last of its head
    float sh = 0.f, m = 0.f, s = 1.f, t = 0.f, ent = 0.f;
    bool fresh = false;  // no legal entry of the open head seen yet
#pragma unroll
    for (int j0 = 0; j0 < AP; j0 += W) {
        float z[W];
        md_chunk<AP, VEC>(pc, elem, A, j0, z);
#pragma unroll
        for (int u = 0; u < W; ++u) {
            const int j = j0 + u;
            fresh = fresh || ((hm >> j) & 1u);
            if (j < A) {
                if ((lg >> j) & 1u) {
                    const bool st = fresh;  // the head's first legal entry
                    fresh = false;
                    if (st) sh = -z[u] * kLog2e;
                    const float x = fmaf(z[u], kLog2e, sh);
                    if (st) {
                        m = x, s = 1.f, t = x;
                    } else {
                        float e;
                        t = md_online(x, m, s, &e) ? fmaf(t, e, x) : fmaf(e, x, t);
                    }
                }
                if ((em >> j) & 1u) {
                    const float lse = m + lg2f(s), h = (lse - __fdividef(t, s)) * kLn2;
                    ent += h;
                    dz[j] = sh - lse;
                    if (j > 0) dz[j > 0 ? j - 1 : 0] = h;
                }
            }
        }
    }
    float c = 0.f, H = 0.f;
#pragma unroll
    for (int j0 = AP - W; j0 >= 0; j0 -= W) {
        float z[W];
        md_chunk<AP, VEC>(pc, elem, A, j0, z);
#pragma unroll
        for (int u = W - 1; u >= 0; --u) {
            const int j = j0 + u;
            if (j < A) {
                if ((em >> j) & 1u) {
                    c = dz[j];
                    if (j > 0) H = dz[j > 0 ? j - 1 : 0];
                }
                const float lp = fmaf(z[u], kLog2e, c), p = ex2f(lp);  // log2 p_j, p_j
                const float onehot = ((taken >> j) & 1u) ? 1.f : 0.f;
                const float d = inv_batch * (cp * (p - onehot) + entropy_c * p * (lp * kLn2 + H));
                dz[j] = (valid && ((lg >> j) & 1u)) ? d : 0.f;
            } else {
                dz[j] = 0.f;
            }
        }
    }
    return ent;
}

// POPART: {mu, sigma, 1 / sigma} as float32 in shared memory, read through a volatile pointer at every use so
// that the three values take no register across the unroll (the DIAG twins are at their register limit).
struct PopVals {
    const volatile float* s;
    __device__ __forceinline__ float mu() const { return s[0]; }
    __device__ __forceinline__ float sigma() const { return s[1]; }
    __device__ __forceinline__ float inv() const { return s[2]; }
};

// ------------------------------------------------------------------------------------------------
// Lane = trajectory, warp = time segment.
//
// A CTA owns 32 consecutive trajectories (one per lane: every global access of a time step is a
// fully coalesced row segment - 512 B of logits, 128 B of rewards / actions / values, 32 B of done
// flags per warp instruction - with no shared-memory transposition) and NSEG warps; warp w owns
// the S consecutive time steps [t0 + w S, t0 + (w + 1) S) of the current chunk of S * NSEG steps.
// The unroll is walked backwards chunk by chunk.  Per chunk a thread
//   1. loads its S rows (all loads independent of the recurrence, issued up front),
//   2. evaluates the per-step terms (log-softmax of both logit vectors, rho, c, the affine map
//      F_t(x) = fa_t + g_t x of the recurrence) and scans its segment with carry 0, keeping
//      acc0_t and the running product P_t = g_t ... g_(end of segment),
//   3. publishes the segment's composed map (acc0, P) in shared memory; after ONE barrier every
//      thread composes the maps of the later segments (<= NSEG - 1 FMAs) on top of the carry of the
//      previous chunk and gets the accumulator that enters its segment,
//   4. fixes up acc_t = acc0_t + P_t * carry in registers, forms vs / pg_adv (and, WITH_LOSS, the
//      loss terms and closed-form gradients) and stores them row-contiguously.
// Total threads = B * NSEG, so the small benchmark batch (T = 20, B = 4096) still spreads over
// 1280 warps and the long unroll (T = 100, B = 8192) keeps ~2 500 warps x S rows of loads in flight.
// Wide action sets (AP = 32, STREAM): the logit rows are not prefetched into registers (two row sets
// of both logit vectors would be ~130 registers on their own); step 2 reduces each row as it loads
// (row_lse2) and keeps the two taken-action logits, and step 4 re-reads the current row (an L1 / L2
// hit) for the entropy and the logit gradient.
//
// DIAG (with WITH_LOSS): also the eight off-policy sums of impala_vtrace_loss_diag.  Each thread keeps
// them as seven float32 registers for the whole unroll (at most ceil(T / (S nseg)) S steps per thread:
// 2 at T = 20, 16 at T = 100 for the default shapes) and converts to float64 only in the final
// reduction, next to the loss sums (the loss scalars keep the plain kernel's combination order, so they
// are bit-identical to it); the count of valid steps is sum_b lens[b], added by segment 0.
// Seven floats rather than float64 accumulators (14 registers) or float64 folds per chunk keeps the
// register budget of the plain kernel.  The log-ratio sum and the clip counts come from step 2, KL
// from step 2 as well: on the register path from the behaviour row's 2^zb terms already summed for its
// log-sum-exp (KL / ln 2 = sum_k 2^zb_k (zb_k - zc_k) / sum_k 2^zb_k + lse - lseb, both rows shifted by
// their maximum); on the streaming path VEC rows re-read both rows four logits at a time right after
// row_lse2 reduced them (row_kl2), non-VEC rows re-read the behaviour row in step 4 next to the current
// row's re-read (whichever keeps the twin's zero spills); vs and vs - v come from step 4.
//
// GAUSS (with WITH_LOSS): the diagonal-Gaussian policy terms in place of the softmax ones; everything else
// (the recurrence, the segment composition, the reward transform, PopArt and the reductions) is this same code.
// Like the streaming path no row is held across the chunk: step 2 reduces the current, behaviour and action
// rows of a step as they load into log2 pi(a), the log2 ratio and (DIAG) KL (gauss_terms); step 4 re-reads the
// current and action rows (L1 / L2 hits) for the entropy sum_k (s_k + (1 + log 2 pi) / 2) and the 2A gradients
//   d/dm_k = -policy_loss_c pg (a_k - m_k) / sigma_k^2 / B,   d/ds_k = (policy_loss_c pg (1 - u_k^2) - entropy_c) / B.
//
// POPART (with DIAG): v holds the normalized values n; every value row is turned into reward units
// v = sigma n + mu by one FMA as it is loaded (v[:1] included), so the recurrence, vs and the eight sums are
// those of the value function sigma n + mu.  The accumulator acc = vs - v enters dv, pg and the two loss
// sums scaled by 1 / sigma: the loss is that of the normalized targets, 0.5 sum ((v - vs) / sigma)^2, and
// the advantage pg / sigma.  mu = 0, sigma = 1 leaves every value as it is (FMA with 1 and 0, products by 1).
// ------------------------------------------------------------------------------------------------
// MD (with WITH_LOSS): the multi-discrete policy terms (md_terms, md_grad) in place of the softmax ones, AP = the
// padded output count N.  As on the GAUSS path no row is held across the chunk: step 2 reduces the current and
// behaviour rows and the K action indices of a step as they load, and keeps the step's taken mask in the action slot
// of the rows; step 4 re-reads the current row for the entropy and the N gradients.
// ------------------------------------------------------------------------------------------------
// MASK (categorical or MD): invalid-action masking.  The action row carries one more int32, the step's legal word
// (categorical: [a, legal], read with the index in one 64-bit load; MD: [a_0 .. a_{K-1}, legal], read by md_terms),
// kept as one register per step (legal_row: bits >= A dropped, an empty head all-legal).  Every sum over a row's
// entries (maxima, log-sum-exps, KL, entropy) takes the legal entries only, the maxima folding from -inf, and the
// gradient is selected to exactly zero at illegal entries, so no illegal logit reaches an output.  With every bit set
// the predicates are all true and the arithmetic and its order are those of the unmasked twin.
// ------------------------------------------------------------------------------------------------
// The body is one device function; vtrace_lane_kernel (softmax policies), vtrace_gauss_kernel (GAUSS),
// vtrace_md_kernel (MD), vtrace_mask_kernel (MASK) and vtrace_md_mask_kernel (MD and MASK) are its thin __global__
// entries, so the categorical instantiations keep their names and code.
template <int AP, int S, bool WITH_LOSS, bool VEC, bool DIAG, bool POPART, bool RCLIP, bool GAUSS, bool MD = false,
          bool MASK = false>
__device__ __forceinline__ void vtrace_lane_body(const VtArgsM<DIAG, POPART, RCLIP, MD>& a) {
    constexpr bool STREAM = !GAUSS && !MD && AP > 16;
    constexpr bool HELD = !STREAM && !GAUSS && !MD;  // the logit rows of a chunk are held in registers
    constexpr int SR = HELD ? S : 1, AR = HELD ? AP : 1;  // extent of the held logit rows
    static_assert(!STREAM || S == 1, "the streaming rows keep one step per thread");
    static_assert(!GAUSS || (WITH_LOSS && AP <= 16), "Gaussian policies: the loss kernel, up to 16 action dimensions");
    static_assert(!MD || (WITH_LOSS && !GAUSS), "multi-discrete policies: the loss kernel");
    static_assert(!MASK || (WITH_LOSS && !GAUSS), "action masks: categorical and multi-discrete loss kernels");
    // GAUSS: the (T, B, A) float32 action samples (the categorical kernels read int32 indices there)
    const float* const gact = reinterpret_cast<const float*>(a.actions);
    static_assert(!DIAG || WITH_LOSS, "the off-policy sums ride the loss reduction");
    static_assert(!POPART || DIAG, "the value statistics are formed from the DIAG sums");
    static_assert(!RCLIP || WITH_LOSS, "impala_vtrace has no reward transform");
    constexpr int NV = DIAG ? 12 : 4;  // per-CTA sums: 4 loss sums (+ 8 off-policy sums)
    __shared__ float2 s_map[2][kMaxSeg][32];
    __shared__ float2 s_cta[2][32];  // this CTA's segments composed into one map (read by the cluster)
    __shared__ double s_red[kMaxSeg][NV];
    pdl_wait();  // logits / values come from the forward kernel
    // POPART: v = sigma n + mu (reward units); acc / sigma = acc * (1 / sigma) (normalized)
    __shared__ float s_pop[POPART ? 3 : 1];
    const PopVals pop{s_pop};
    if constexpr (POPART) {
        if (threadIdx.x == 0) s_pop[0] = (float)a.popart[0], s_pop[1] = (float)a.popart[2], s_pop[2] = (float)(1.0 / a.popart[2]);
        __syncthreads();
    }
    // Long unrolls: the time segments of a trajectory group are spread over a thread-block CLUSTER
    // (csize CTAs x nw warps x S steps per chunk - T = 100 fits ONE chunk of 8 x 7 x 2 steps), so a
    // thread's critical path is one load -> math -> exchange -> fix-up -> store sequence instead of
    // T / (S nw) of them back to back; the CTA-level maps travel through distributed shared memory.
    cg::cluster_group cluster = cg::this_cluster();
    const int csize = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int nseg = nw * csize, seg = crank * nw + w;  // segments per chunk, this thread's segment
    const int T = a.T, B = a.B, A = VEC ? AP : a.A;
    const int b = (blockIdx.x / csize) * 32 + lane;
    const bool live = b < B;
    const int bl = live ? b : B - 1;  // column this lane loads
    const int L = live ? min(max(__ldg(a.lens + bl), 0), T) : 0;
    const float v0 = POPART ? fmaf(pop.sigma(), __ldg(a.v + bl), pop.mu()) : __ldg(a.v + bl);  // V(x_0): the reference's v[:1]
    const int rows = S * nseg;
    const int nch = (T + rows - 1) / rows;
    const bool ref_mode = a.mode == IMPALA_MODE_REFERENCE;

    double sum_vl = 0.0, sum_pl = 0.0, sum_ent = 0.0, sum_rw = 0.0;
    // DIAG: sum of log2 ratio, #ratio > rho_bar, #ratio > c_bar, sum KL / ln 2, sum vs, sum vs^2, sum (vs - v)
    float d_lr = 0.f, d_nrho = 0.f, d_nc = 0.f, d_kl = 0.f, d_vs = 0.f, d_vs2 = 0.f, d_err = 0.f;
    float chunk_carry = 0.f;  // accumulator at the first step after the current chunk
    // One chunk's raw rows of this thread (registers).  Unpredicated loads: steps past the unroll
    // (last chunk only) re-read step T - 1 and dead lanes read trajectory B - 1; both are masked
    // by `valid` below (rho = c = disc = 0).
    struct Rows {
        float zc[SR][AR], zb[SR][AR], r[S], vv[S + 1];
        int act[S];
        unsigned lg[MASK ? S : 1];  // MASK: the legal words (legal_row)
        unsigned char dn[S];  // raw: compared where it is used, so the load is not waited for at issue
    };
    auto load_rows = [&](Rows& R, const int c) {
        const int tb = c * rows + seg * S;
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const unsigned e = (unsigned)min(tb + i, T - 1) * (unsigned)B + (unsigned)bl;
            if constexpr (HELD) {
                load_logits<AP, VEC>(a.cur_logits, e, A, R.zc[i]);
                load_logits<AP, VEC>(a.beh_logits, e, A, R.zb[i]);
            }
            R.r[i] = __ldg(a.rewards + e);
            if constexpr (MASK && !MD) {
                const int2 q = __ldg(reinterpret_cast<const int2*>(a.actions) + e);  // [a, legal]
                R.act[i] = q.x, R.lg[i] = legal_row((unsigned)q.y, A);
            } else if constexpr (!GAUSS && !MD) {
                R.act[i] = __ldg(a.actions + e);
            }
            R.dn[i] = __ldg(a.done + e);
        }
#pragma unroll
        for (int i = 0; i <= S; ++i) {
            const float n = __ldg(a.v + (unsigned)min(tb + i, T) * (unsigned)B + (unsigned)bl);
            R.vv[i] = POPART ? fmaf(pop.sigma(), n, pop.mu()) : n;  // reward units
        }
    };
    auto process = [&](Rows& R, const int c) {
        const int tb = c * rows + seg * S;  // first step of this thread's segment
        // ---- 2. per-step terms and the zero-carry scan of this segment
        float rho[S], disc[S], fa[S], g[S], lp2a[S];
        float shc[SR], lsec[SR];  // STREAM: log2 pi(k) = fmaf(z_k, log2(e), shc) - lsec
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const bool valid = tb + i < L;
            float lr2;  // log2 pi(a) - log2 mu(a)
            if constexpr (GAUSS) {
                const unsigned e = (unsigned)min(tb + i, T - 1) * (unsigned)B + (unsigned)bl;
                float kl2;
                gauss_terms<AP, VEC, DIAG>(a.cur_logits, a.beh_logits, gact, e, A, &lp2a[i], &lr2, &kl2);
                if constexpr (DIAG) {
                    if (valid) d_kl += kl2;
                }
            } else if constexpr (MD) {
                const unsigned e = (unsigned)min(tb + i, T - 1) * (unsigned)B + (unsigned)bl;
                float kl2;
                if constexpr (MASK)
                    R.act[i] = (int)md_terms_masked<AP, VEC, DIAG>(a.cur_logits, a.beh_logits, a.actions, e, A,
                                                                   a.head_mask, &lp2a[i], &lr2, &kl2, &R.lg[MASK ? i : 0]);
                else
                    R.act[i] = (int)md_terms<AP, VEC, DIAG>(a.cur_logits, a.beh_logits, a.actions, e, A, a.head_mask,
                                                            &lp2a[i], &lr2, &kl2);
                if constexpr (DIAG) {
                    if (valid) d_kl += kl2;
                }
            } else {
                // log-softmax of both logit vectors in the base-2 domain (learner.py:298-303)
                float z_a, zb_a, lse, lseb;
                if constexpr (STREAM) {
                    const unsigned e = (unsigned)min(tb + i, T - 1) * (unsigned)B + (unsigned)bl;
                    float shb;
                    const unsigned lg = MASK ? R.lg[MASK ? i : 0] : 0u;
                    row_lse2<AP, VEC, MASK>(a.cur_logits, e, A, R.act[i], &shc[i], &lsec[i], &z_a, lg);
                    row_lse2<AP, VEC, MASK>(a.beh_logits, e, A, R.act[i], &shb, &lseb, &zb_a, lg);
                    lse = lsec[i];
                    if constexpr (DIAG && VEC) {
                        if (valid)
                            d_kl += row_kl2<AP, MASK>(a.cur_logits, a.beh_logits, e, shc[i], lsec[i], shb, lseb, lg);
                    } else if constexpr (DIAG) {
                        // non-VEC rows: KL in step 4 next to the current row's re-read (row_kl2 here spills); the
                        // behaviour row's shift and lse2 are parked in the row slots the streaming path leaves unused
                        R.zb[i][0] = shb, R.zc[i][0] = lseb;
                    }
                } else {
                    if constexpr (MASK) mask_row<AP>(R.lg[MASK ? i : 0], R.zc[i]), mask_row<AP>(R.lg[MASK ? i : 0], R.zb[i]);
                    float mx = R.zc[i][0], mxb = R.zb[i][0];
#pragma unroll
                    for (int k = 1; k < AP; ++k)
                        if (k < A) mx = fmaxf(mx, R.zc[i][k]), mxb = fmaxf(mxb, R.zb[i][k]);
                    float se = 0.f, seb = 0.f, klw = 0.f;  // DIAG: klw = sum_k 2^zb_k (zb_k - zc_k), shifted rows
                    const float mxl = -mx * kLog2e, mxbl = -mxb * kLog2e;
#pragma unroll
                    for (int k = 0; k < AP; ++k) {
                        R.zc[i][k] = fmaf(R.zc[i][k], kLog2e, mxl);   // (z - max) log2(e), one rounding
                        R.zb[i][k] = fmaf(R.zb[i][k], kLog2e, mxbl);
                        if (k < A) se += ex2f(R.zc[i][k]), seb += ex2f(R.zb[i][k]);
                        if constexpr (DIAG) {
                            if (k < A && (!MASK || is_legal(R.zb[i][k])))
                                klw = fmaf(ex2f(R.zb[i][k]), R.zb[i][k] - R.zc[i][k], klw);  // same ex2 as seb's
                        }
                    }
                    lse = lg2f(se), lseb = lg2f(seb);
                    if constexpr (DIAG) {
                        if (valid) d_kl += __fdividef(klw, seb) + (lse - lseb);  // KL(mu || pi) / ln 2
                    }
                    z_a = R.zc[i][0], zb_a = R.zb[i][0];
#pragma unroll
                    for (int k = 1; k < AP; ++k) {
                        const bool hit = k == R.act[i];
                        z_a = selp_f32(hit, R.zc[i][k], z_a), zb_a = selp_f32(hit, R.zb[i][k], zb_a);
                    }
#pragma unroll
                    for (int k = 0; k < AP; ++k) R.zc[i][k] -= lse;  // log2 pi(k)
                }
                lp2a[i] = z_a - lse;                                               // log2 pi(a)
                lr2 = lp2a[i] - (zb_a - lseb);
            }
            const float ratio = ex2f(lr2);                                     // :121-123
            rho[i] = valid ? fminf(ratio, a.rho_bar) : 0.f;                    // :124
            const float cc = valid ? fminf(ratio, a.c_bar) : 0.f;              // :125
            if constexpr (DIAG) {
                if (valid) {
                    d_lr += lr2;
                    d_nrho += ratio > a.rho_bar ? 1.f : 0.f;
                    d_nc += ratio > a.c_bar ? 1.f : 0.f;
                }
            }
            disc[i] = (valid && R.dn[i] == 0) ? a.gamma : 0.f;                       // :109
            if constexpr (RCLIP) {
                // the raw reward goes to batch_mean_reward here, the clipped one replaces it for delta and pg
                if (valid) sum_rw += (double)R.r[i];
                R.r[i] = clip_reward(R.r[i], a.reward_clip);
            }
            g[i] = disc[i] * cc;
            if (ref_mode) {
                const float delta = rho[i] * (R.r[i] + a.gamma * R.vv[i + 1] - v0);  // :126
                fa[i] = delta - g[i] * R.vv[i + 1];                                // :130
            } else {
                fa[i] = rho[i] * (R.r[i] + disc[i] * R.vv[i + 1] - R.vv[i]);
            }
        }
        float acc[S + 1], P[S];
        acc[S] = 0.f;
        float prod = 1.f;
#pragma unroll
        for (int i = S - 1; i >= 0; --i) {
            acc[i] = fmaf(g[i], acc[i + 1], fa[i]);
            prod *= g[i];
            P[i] = prod;
        }
        // ---- 3. exchange the composed maps of the segments, find the carry entering this segment.
        // Inside the CTA: the carry entering segment s is  A_s + Pm_s * x  with x the carry entering
        // the CTA's LAST segment; composing all nw maps gives the CTA's own map.  Across the cluster:
        // x comes from composing the maps of the later CTAs on top of the previous chunk's carry.
        const int par = c & 1;
        s_map[par][w][lane] = make_float2(acc[0], P[0]);
        __syncthreads();
        float cA = 0.f, cP = 1.f, mineA = 0.f, mineP = 1.f;
        for (int s2 = nw - 1; s2 >= 0; --s2) {
            if (s2 == w) mineA = cA, mineP = cP;
            const float2 q = s_map[par][s2][lane];
            cA = fmaf(q.y, cA, q.x);
            cP = q.y * cP;
        }
        float x = chunk_carry;
        if (csize > 1) {
            if (w == 0) s_cta[par][lane] = make_float2(cA, cP);
            cluster.sync();
            float xm = x;
            for (int r = csize - 1; r >= 0; --r) {
                if (r == crank) xm = x;
                const float2 q = *cluster.map_shared_rank(&s_cta[par][lane], r);
                x = fmaf(q.y, x, q.x);
            }
            chunk_carry = x;  // accumulator at the first step of this chunk
            x = xm;
        } else {
            chunk_carry = fmaf(cP, x, cA);
        }
        const float mine = fmaf(mineP, x, mineA);

        // ---- 4. fix-up, outputs, loss terms
        acc[S] = mine;
#pragma unroll
        for (int i = S - 1; i >= 0; --i) {
            const int t = tb + i;
            const bool valid = t < L;
            acc[i] = fmaf(P[i], mine, acc[i]);
            const float vs_n = acc[i + 1] + R.vv[i + 1];                         // :131
            const float pg_r = rho[i] * (R.r[i] + disc[i] * vs_n - R.vv[i]);        // :135
            const float pg = POPART ? pg_r * pop.inv() : pg_r;  // the normalized advantage: pg_adv, dlogits, the loss
            const unsigned e = (unsigned)t * (unsigned)B + (unsigned)b;
            if (live && t < T) {
                if (a.vs) a.vs[e] = (t <= L) ? acc[i] + R.vv[i] : 0.f;
                if (a.pg_adv) a.pg_adv[e] = pg;  // rho == 0 on padding
                if (t == T - 1 && a.vs) a.vs[e + B] = (L == T) ? R.vv[i + 1] : 0.f;  // bootstrap row
            }
            if constexpr (WITH_LOSS) {
                // d total / d v = v_loss_c (v - vs) / B = -v_loss_c acc / B  (:149, :306-307)
                float ent = 0.f, dz[GAUSS ? 2 * AP : AP];
                if constexpr (GAUSS) {
                    // re-read the current and action rows: the entropy and the 2A output gradients
                    float m[AP], s[AP], x[AP];
                    const unsigned er = (unsigned)min(t, T - 1) * (unsigned)B + (unsigned)bl;
                    load_gauss<AP, VEC>(a.cur_logits, er, A, m, s);
                    load_logits<AP, VEC>(gact, er, A, x);
                    const float cp = a.policy_loss_c * pg;
#pragma unroll
                    for (int k = 0; k < AP; ++k) {
                        const float iv = ex2f(-2.f * s[k] * kLog2e);  // 1 / sigma^2
                        const float d = x[k] - m[k], du = d * iv;   // (a - m) / sigma^2
                        ent += s[k];
                        dz[k] = valid ? a.inv_batch * (-cp * du) : 0.f;
                        dz[AP + k] = valid ? a.inv_batch * (cp * fmaf(-d, du, 1.f) - a.entropy_c) : 0.f;
                    }
                    ent = fmaf((float)A, kHalfLog2PiE, ent);
                } else if constexpr (MD) {
                    if constexpr (MASK)
                        ent = md_grad_masked<AP, VEC>(a.cur_logits, (unsigned)min(t, T - 1) * (unsigned)B + (unsigned)bl,
                                                      A, a.head_mask, (unsigned)R.act[i], valid, a.policy_loss_c * pg,
                                                      a.entropy_c, a.inv_batch, dz, R.lg[MASK ? i : 0]);
                    else
                        ent = md_grad<AP, VEC>(a.cur_logits, (unsigned)min(t, T - 1) * (unsigned)B + (unsigned)bl, A,
                                               a.head_mask, (unsigned)R.act[i], valid, a.policy_loss_c * pg, a.entropy_c,
                                               a.inv_batch, dz);
                } else if constexpr (STREAM) {
                    // re-read the row; dz holds log2 pi(k), then the gradient (one row of registers)
                    load_logits<AP, VEC>(a.cur_logits, (unsigned)min(t, T - 1) * (unsigned)B + (unsigned)bl, A, dz);
                    if constexpr (MASK) mask_row<AP>(R.lg[MASK ? i : 0], dz);
#pragma unroll
                    for (int k = 0; k < AP; ++k) {
                        dz[k] = fmaf(dz[k], kLog2e, shc[i]) - lsec[i];
                        // MASK: the twin's form - VEC, the unconditional FMA with a zero factor at an illegal entry
                        // (2^-inf = 0); otherwise the predicated one
                        if constexpr (MASK && VEC)
                            ent -= ex2f(dz[k]) * (is_legal(dz[k]) ? dz[k] * kLn2 : 0.f);
                        else if (k < A && (!MASK || is_legal(dz[k])))
                            ent -= ex2f(dz[k]) * (dz[k] * kLn2);
                    }
                    if constexpr (DIAG && !VEC) {
                        // KL(mu || pi) / ln 2 against the log2 pi(k) in dz: the behaviour row again
                        if (valid) {
                            const unsigned eb = (unsigned)t * (unsigned)B + (unsigned)bl;
                            float kl = 0.f;
#pragma unroll
                            for (int k = 0; k < AP; ++k) {
                                const float zb = k < A ? __ldg(a.beh_logits + eb * A + k) : 0.f;
                                const float lmu = fmaf(zb, kLog2e, R.zb[i][0]) - R.zc[i][0];  // log2 mu(k)
                                if (k < A && (!MASK || is_legal(dz[k]))) kl = fmaf(ex2f(lmu), lmu - dz[k], kl);
                            }
                            d_kl += kl;
                        }
                    }
#pragma unroll
                    for (int k = 0; k < AP; ++k) {
                        // MASK: pk = 2^-inf = 0 at an illegal entry already; its gradient (0 * -inf) is selected away
                        const bool ok = k < A && (!MASK || is_legal(dz[k]));
                        const float lz = dz[k] * kLn2, pk = (k < A) ? ex2f(dz[k]) : 0.f;
                        const float onehot = (k == R.act[i]) ? 1.f : 0.f;
                        const float d = a.inv_batch * (a.policy_loss_c * pg * (pk - onehot) +
                                                       a.entropy_c * pk * (lz + ent));
                        dz[k] = (valid && ok) ? d : 0.f;
                    }
                } else {
                    float pk[AP], lz[AP];
#pragma unroll
                    for (int k = 0; k < AP; ++k) {
                        const bool ok = k < A && (!MASK || is_legal(R.zc[i][k]));
                        lz[k] = R.zc[i][k] * kLn2;
                        pk[k] = ok ? ex2f(R.zc[i][k]) : 0.f;
                        if (ok) ent -= pk[k] * lz[k];                           // :310-314, :153
                    }
#pragma unroll
                    for (int k = 0; k < AP; ++k) {
                        const bool ok = k < A && (!MASK || is_legal(R.zc[i][k]));
                        const float onehot = (k == R.act[i]) ? 1.f : 0.f;
                        const float d = a.inv_batch * (a.policy_loss_c * pg * (pk[k] - onehot) +
                                                       a.entropy_c * pk[k] * (lz[k] + ent));
                        dz[k] = (valid && ok) ? d : 0.f;
                    }
                }
                if (live && t < T) {
                    // POPART: the normalized error (v - vs) / sigma in dv and the value loss
                    a.dv[e] = valid ? -a.v_loss_c * a.inv_batch * (POPART ? acc[i] * pop.inv() : acc[i]) : 0.f;
                    if (t == T - 1) a.dv[e + B] = 0.f;
                    if constexpr (GAUSS) store_gauss<AP, VEC>(a.dlogits, e, A, dz);
                    else store_logits<AP, VEC>(a.dlogits, e, A, dz);
                }
                if (valid) {
                    const float err_n = POPART ? acc[i] * pop.inv() : acc[i];
                    sum_vl += 0.5 * (double)err_n * (double)err_n;
                    sum_pl += (double)(-(lp2a[i] * kLn2) * pg);                // :317-321
                    sum_ent += (double)ent;
                    if constexpr (!RCLIP) sum_rw += (double)R.r[i];              // :108
                    if constexpr (DIAG) {
                        const float vs_t = acc[i] + R.vv[i];  // the value written to vs
                        d_vs += vs_t, d_vs2 = fmaf(vs_t, vs_t, d_vs2), d_err += acc[i];
                    }
                }
            }
        }
    };
    // Chunks are walked backwards with the NEXT chunk's loads already in flight while the current one
    // is processed (two register sets, loop unrolled by two): without it every CTA alternates between
    // a pure memory phase and a pure compute phase and, all CTAs having started together, so does
    // the whole GPU.
    {
        Rows R0, R1;
        int c = nch - 1;
        load_rows(R0, c);
        while (true) {
            if (c > 0) load_rows(R1, c - 1);
            process(R0, c);
            if (--c < 0) break;
            if (c > 0) load_rows(R0, c - 1);
            process(R1, c);
            if (--c < 0) break;
        }
    }

    if constexpr (WITH_LOSS) {
        // per-CTA sums -> workspace; the last CTA to arrive adds them up in a fixed order
        // (bitwise reproducible, no float64 atomics, no memset node) and re-arms the counter.
        __shared__ bool s_last;
        __shared__ double s_fin[32][NV];
        const int tid = threadIdx.x;
        sum_vl = warp_sum_f64(sum_vl);
        sum_pl = warp_sum_f64(sum_pl);
        sum_ent = warp_sum_f64(sum_ent);
        sum_rw = warp_sum_f64(sum_rw);
        if (lane == 0) s_red[w][0] = sum_vl, s_red[w][1] = sum_pl, s_red[w][2] = sum_ent, s_red[w][3] = sum_rw;
        if constexpr (DIAG) {
            constexpr double kLn2d = 0.6931471805599453;
            double dg[8] = {seg == 0 ? (double)L : 0.0, (double)d_lr * kLn2d, (double)d_nrho, (double)d_nc,
                            (double)d_kl * kLn2d, (double)d_vs, (double)d_vs2, (double)d_err};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                dg[j] = warp_sum_f64(dg[j]);
                if (lane == 0) s_red[w][4 + j] = dg[j];
            }
        }
        __syncthreads();
        if (tid < NV) {
            double s = 0.0;
            for (int i = 0; i < nw; ++i) s += s_red[i][tid];
            a.partials[(size_t)blockIdx.x * NV + tid] = s;
            __threadfence();
        }
        __syncthreads();
        if (tid == 0) s_last = atomicAdd(a.counter, 1u) == gridDim.x - 1;
        __syncthreads();
        if (s_last) {
            __threadfence();
            const int nthr = (int)blockDim.x, which = tid & 3, stripe = tid >> 2, nstripes = nthr >> 2;
            double s = 0.0;
            for (unsigned cta = stripe; cta < gridDim.x; cta += nstripes)
                s += __ldcg(a.partials + (size_t)cta * NV + which);
            // fixed-order tree over the stripes of each scalar: lanes {which, which + 4, ...} of a warp,
            // then the warps through shared memory
            s += __shfl_xor_sync(IMPALA_FULL_MASK, s, 4);
            s += __shfl_xor_sync(IMPALA_FULL_MASK, s, 8);
            s += __shfl_xor_sync(IMPALA_FULL_MASK, s, 16);
            if (lane < 4) s_fin[w][lane] = s;
            if constexpr (DIAG) {
                // the eight off-policy sums by the same scheme over stripes of 8 (the loss scalars above keep
                // exactly the plain kernel's order, so they stay bit-identical to it)
                const int wd = tid & 7, sd = tid >> 3, nsd = nthr >> 3;
                double q = 0.0;
                for (unsigned cta = sd; cta < gridDim.x; cta += nsd)
                    q += __ldcg(a.partials + (size_t)cta * NV + 4 + wd);
                q += __shfl_xor_sync(IMPALA_FULL_MASK, q, 8);
                q += __shfl_xor_sync(IMPALA_FULL_MASK, q, 16);
                if (lane < 8) s_fin[w][4 + lane] = q;
            }
            __syncthreads();
            if (tid < NV) {
                double tot = 0.0;
                for (int i = 0; i < nw; ++i) tot += s_fin[i][tid];
                if constexpr (DIAG) {
                    if (tid < 4) a.scalars[tid] = tot * (double)a.inv_batch;
                    else a.diag[tid - 4] = tot;  // not scaled: the off-policy sums add across ranks
                } else {
                    a.scalars[tid] = tot * (double)a.inv_batch;
                }
            }
            if (tid == 0) *a.counter = 0u;
        }
    }
    if (csize > 1) cluster.sync();  // no CTA leaves while a peer may still read its shared memory
}

template <int AP, int S, int MAXT, int MINB, bool WITH_LOSS, bool VEC, bool DIAG, bool POPART = false,
          bool RCLIP = false>
__global__ void __launch_bounds__(MAXT, MINB) vtrace_lane_kernel(const VtArgsT<DIAG, POPART, RCLIP> a) {
    vtrace_lane_body<AP, S, WITH_LOSS, VEC, DIAG, POPART, RCLIP, false>(a);
}
template <int AP, int S, int MAXT, int MINB, bool VEC, bool DIAG, bool POPART, bool RCLIP>
__global__ void __launch_bounds__(MAXT, MINB) vtrace_gauss_kernel(const VtArgsT<DIAG, POPART, RCLIP> a) {
    vtrace_lane_body<AP, S, true, VEC, DIAG, POPART, RCLIP, true>(a);
}
template <int AP, int S, int MAXT, int MINB, bool VEC, bool DIAG, bool POPART, bool RCLIP>
__global__ void __launch_bounds__(MAXT, MINB) vtrace_md_kernel(const VtArgsM<DIAG, POPART, RCLIP, true> a) {
    vtrace_lane_body<AP, S, true, VEC, DIAG, POPART, RCLIP, false, true>(a);
}
template <int AP, int S, int MAXT, int MINB, bool VEC, bool DIAG, bool POPART, bool RCLIP>
__global__ void __launch_bounds__(MAXT, MINB) vtrace_mask_kernel(const VtArgsT<DIAG, POPART, RCLIP> a) {
    vtrace_lane_body<AP, S, true, VEC, DIAG, POPART, RCLIP, false, false, true>(a);
}
template <int AP, int S, int MAXT, int MINB, bool VEC, bool DIAG, bool POPART, bool RCLIP>
__global__ void __launch_bounds__(MAXT, MINB) vtrace_md_mask_kernel(const VtArgsM<DIAG, POPART, RCLIP, true> a) {
    vtrace_lane_body<AP, S, true, VEC, DIAG, POPART, RCLIP, false, true, true>(a);
}

int pick_ap(int A) {
    if (A <= 2) return 2;
    if (A <= 4) return 4;
    if (A <= 8) return 8;
    if (A <= 16) return 16;
    if (A <= 32) return 32;
    return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int AP, int S, int MAXT, int MINB, bool WITH_LOSS, bool DIAG, bool POPART, bool RCLIP, bool GAUSS = false,
          bool MD = false, bool MASK = false>
int launch_s(const VtArgsM<DIAG, POPART, RCLIP, MD>& a, bool vec, unsigned groups, int nw, int cl, cudaStream_t st) {
    cudaError_t e;
    if constexpr (MD && MASK)
        e = vec ? impala_launch_cl(vtrace_md_mask_kernel<AP, S, MAXT, MINB, true, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a)
                : impala_launch_cl(vtrace_md_mask_kernel<AP, S, MAXT, MINB, false, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a);
    else if constexpr (MASK)
        e = vec ? impala_launch_cl(vtrace_mask_kernel<AP, S, MAXT, MINB, true, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a)
                : impala_launch_cl(vtrace_mask_kernel<AP, S, MAXT, MINB, false, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a);
    else if constexpr (MD)
        e = vec ? impala_launch_cl(vtrace_md_kernel<AP, S, MAXT, MINB, true, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a)
                : impala_launch_cl(vtrace_md_kernel<AP, S, MAXT, MINB, false, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a);
    else if constexpr (GAUSS)
        e = vec ? impala_launch_cl(vtrace_gauss_kernel<AP, S, MAXT, MINB, true, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a)
                : impala_launch_cl(vtrace_gauss_kernel<AP, S, MAXT, MINB, false, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a);
    else
        e = vec ? impala_launch_cl(vtrace_lane_kernel<AP, S, MAXT, MINB, WITH_LOSS, true, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a)
                : impala_launch_cl(vtrace_lane_kernel<AP, S, MAXT, MINB, WITH_LOSS, false, DIAG, POPART, RCLIP>, groups * cl, 32 * nw, 0, st, true, false, cl, a);
    if (e != cudaSuccess) return (int)e;
    return impala_launch_status();
}

constexpr int kMaxCluster = 8;  // portable cluster size

// Steps per thread (S), warps per CTA (nw) and CTAs per cluster (cl); wide action sets trade S for
// registers.  S = 2; up to 10 segments (T <= 20) one CTA holds the whole unroll in one chunk; longer
// unrolls walk chunks of 8 x S steps with 8 warps per CTA.  Spreading the segments of a long unroll
// over a thread-block cluster (DSMEM carry exchange, cl = 4 / 8) works, but its cluster barriers
// replace a cheap chunk loop, so cl = 1 unless overridden (scripts/tune_vtrace.py compares them).
// IMPALA_VTRACE_S / IMPALA_VTRACE_NSEG (warps per CTA) / IMPALA_VTRACE_CLUSTER override the choice.
// GAUSS: a.A action dimensions (rows of 2A policy outputs), AP = the padded dimension count, at most 16; S = 2 up
// to AP = 4 and S = 1 from AP = 8 on, where the five rows of two steps in flight would spill (IMPALA_VTRACE_S
// does not apply).
// MD: a.A = N policy outputs, AP = the padded N; S as the categorical twin at that AP (IMPALA_VTRACE_S does not apply),
// at most 8 warps per CTA at AP = 32 (the 256-thread bound of those instantiations).
// MASK: the launch shapes of the unmasked twin (categorical or MD), so a full mask gives its results bit for bit.
// IMPALA_VTRACE_S does not apply (the S = 1 and S = 5 overrides of AP <= 4 spill with the legal words), and the
// categorical AP = 32 kernels are bounded at 320 threads, the most the launcher picks there (IMPALA_VTRACE_NSEG is
// clamped to 10 warps): under 512 they spilled.
constexpr int kMaxGaussA = 16;
template <bool WITH_LOSS, bool DIAG = false, bool POPART = false, bool RCLIP = false, bool GAUSS = false, bool MD = false,
          bool MASK = false>
int launch(VtArgsM<DIAG, POPART, RCLIP, MD>& a, cudaStream_t st) {
    if (a.T < 1 || a.B < 1 || a.A < 1) return IMPALA_ERR_BAD_ARG;
    const int AP = (GAUSS && a.A > kMaxGaussA) ? 0 : pick_ap(a.A);
    if (!AP) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    // 32-bit element offsets inside the kernel
    if ((int64_t)(a.T + 1) * a.B * AP * (GAUSS ? 2 : 1) >= (int64_t)1 << 31) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    const unsigned groups = (unsigned)((a.B + 31) / 32);
    const bool vec = a.A == AP && aligned16(a.cur_logits) && aligned16(a.beh_logits) &&
                     (!WITH_LOSS || aligned16(a.dlogits)) && (!GAUSS || aligned16(a.actions));
    int S = AP >= (GAUSS ? 8 : 16) ? 1 : 2;
    const int s_env = (GAUSS || MD || MASK) ? 0 : impala_env_int("IMPALA_VTRACE_S", 0);
    if (AP <= 4 && (s_env == 1 || s_env == 2 || s_env == 5)) S = s_env;
    const int max_w = S == 5 ? 10 : (AP <= 4 && S == 1 ? kMaxSeg : 16);
    const int nseg = (a.T + S - 1) / S;
    const int cl_env = impala_env_int("IMPALA_VTRACE_CLUSTER", 0);
    const int cl = (cl_env >= 1 && cl_env <= kMaxCluster) ? cl_env : 1;
    int nw = (nseg + cl - 1) / cl;
    if (cl == 1 && nw > 10) nw = 8;  // chunk loop: 8 warps per CTA measured best for long unrolls
    if (nw > max_w) nw = max_w;
    const int n_env = impala_env_int("IMPALA_VTRACE_NSEG", 0);
    if (n_env >= 1 && n_env <= max_w) nw = n_env;
    if constexpr (MD) {
        if (AP == 2) return launch_s<2, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, true, MASK>(a, vec, groups, nw, cl, st);
        if (AP == 4) return launch_s<4, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, true, MASK>(a, vec, groups, nw, cl, st);
        if (AP == 8) return launch_s<8, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, true, MASK>(a, vec, groups, nw, cl, st);
        if (AP == 16) return launch_s<16, 1, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, true, MASK>(a, vec, groups, nw, cl, st);
        return launch_s<32, 1, 256, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, true, MASK>(a, vec, groups, 8 < nw ? 8 : nw, cl, st);
    } else if constexpr (GAUSS) {
        if (AP == 2) return launch_s<2, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, true>(a, vec, groups, nw, cl, st);
        if (AP == 4) return launch_s<4, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, true>(a, vec, groups, nw, cl, st);
        if (AP == 8) return launch_s<8, 1, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, true>(a, vec, groups, nw, cl, st);
        return launch_s<16, 1, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, true>(a, vec, groups, nw, cl, st);
    } else {
#define VT_AP(APV)                                                                                                    \
    if (AP == APV) {                                                                                                  \
        if constexpr (!MASK) {                                                                                        \
            if (S == 5) return launch_s<APV, 5, 320, 1, WITH_LOSS, DIAG, POPART, RCLIP>(a, vec, groups, nw, cl, st); \
            if (S == 1) return launch_s<APV, 1, 1024, 1, WITH_LOSS, DIAG, POPART, RCLIP>(a, vec, groups, nw, cl, st);\
        }                                                                                                             \
        return launch_s<APV, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, false, MASK>(a, vec, groups, nw, cl, st); \
    }
    VT_AP(2)
    VT_AP(4)
#undef VT_AP
    if (AP == 8) return launch_s<8, 2, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, false, MASK>(a, vec, groups, nw, cl, st);
    if (AP == 16) return launch_s<16, 1, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, false, MASK>(a, vec, groups, nw, cl, st);
    if constexpr (MASK) return launch_s<32, 1, 320, 1, WITH_LOSS, DIAG, POPART, RCLIP, false, false, true>(a, vec, groups, 10 < nw ? 10 : nw, cl, st);
    else return launch_s<32, 1, 512, 1, WITH_LOSS, DIAG, POPART, RCLIP>(a, vec, groups, nw, cl, st);
    }
}

// Per-CTA partial rows: 4 loss sums (plain) or [4 loss sums | 8 off-policy sums] (diag).
int64_t loss_workspace(int T, int B, int A, int row) {
    if (T < 1 || B < 1 || A < 1) return IMPALA_ERR_BAD_ARG;
    const int64_t grid = (((int64_t)B + 31) / 32) * kMaxCluster;  // one row per CTA, clusters of up to 8 per group
    return grid * row * (int64_t)sizeof(double) + 16;  // per-CTA sums + arrival counter
}

// Argument checks and packing shared by the loss entry points.
int loss_args(VtArgs& a, const float* cur_logits, const float* beh_logits, const int32_t* actions,
              const float* rewards, const uint8_t* done, const int32_t* lens, const float* v, float* vs,
              float* pg_adv, float* dlogits, float* dv, double* scalars, void* workspace,
              int64_t workspace_bytes, int64_t need, int T, int B, int A, float gamma, float rho_bar,
              float c_bar, float v_loss_c, float policy_loss_c, float entropy_c, float inv_batch, int mode) {
    if (!cur_logits || !beh_logits || !actions || !rewards || !done || !lens || !v || !dlogits ||
        !dv || !scalars || !workspace)
        return IMPALA_ERR_BAD_ARG;
    if (mode != IMPALA_MODE_REFERENCE && mode != IMPALA_MODE_PAPER) return IMPALA_ERR_BAD_ARG;
    if (need < 0) return (int)need;
    if (workspace_bytes < need) return IMPALA_ERR_WORKSPACE_TOO_SMALL;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return IMPALA_ERR_BAD_ARG;
    a.cur_logits = cur_logits, a.beh_logits = beh_logits, a.actions = actions, a.rewards = rewards;
    a.done = done, a.lens = lens, a.v = v, a.vs = vs, a.pg_adv = pg_adv, a.dlogits = dlogits;
    a.dv = dv, a.scalars = scalars;
    // workspace = [counter (16 bytes) | per-CTA sums]
    a.counter = reinterpret_cast<unsigned int*>(workspace);
    a.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + 16);
    a.T = T, a.B = B, a.A = A, a.mode = mode;
    a.gamma = gamma, a.rho_bar = rho_bar, a.c_bar = c_bar;
    a.v_loss_c = v_loss_c, a.policy_loss_c = policy_loss_c, a.entropy_c = entropy_c;
    a.inv_batch = inv_batch;
    return 0;
}

}  // namespace
