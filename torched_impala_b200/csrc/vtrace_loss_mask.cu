// Entry point of the masked V-trace + loss kernels (invalid-action masking, IMPALA_ACT_MASKED): the MASK
// instantiations of vtrace_loss.cuh's kernel for categorical policies (vtrace_mask_kernel) and multi-discrete ones
// (vtrace_md_mask_kernel), plain, diag and PopArt, each with and without the reward transform.
#include "vtrace_loss.cuh"

namespace {

template <bool MD, bool DIAG, bool POPART, bool RCLIP>
int launch_mask(VtArgsM<DIAG, POPART, RCLIP, MD>& a, cudaStream_t st) {
    return launch<true, DIAG, POPART, RCLIP, false, MD, true>(a, st);
}

// the flag combinations of one policy kind; `fill` sets the MD head mask (no-op for categorical)
template <bool MD, class Pack, class Fill>
int dispatch(Pack pack, Fill fill, double* diag, const double* popart, int reward_clip, cudaStream_t st) {
    if (reward_clip) {
        if (popart) {
            VtArgsM<true, true, true, MD> a{};
            if (const int rc = pack(a)) return rc;
            a.diag = diag, a.popart = popart, a.reward_clip = reward_clip, fill(a);
            return launch_mask<MD, true, true, true>(a, st);
        }
        if (diag) {
            VtArgsM<true, false, true, MD> a{};
            if (const int rc = pack(a)) return rc;
            a.diag = diag, a.reward_clip = reward_clip, fill(a);
            return launch_mask<MD, true, false, true>(a, st);
        }
        VtArgsM<false, false, true, MD> a{};
        if (const int rc = pack(a)) return rc;
        a.reward_clip = reward_clip, fill(a);
        return launch_mask<MD, false, false, true>(a, st);
    }
    if (popart) {
        VtArgsM<true, true, false, MD> a{};
        if (const int rc = pack(a)) return rc;
        a.diag = diag, a.popart = popart, fill(a);
        return launch_mask<MD, true, true, false>(a, st);
    }
    if (diag) {
        VtArgsM<true, false, false, MD> a{};
        if (const int rc = pack(a)) return rc;
        a.diag = diag, fill(a);
        return launch_mask<MD, true, false, false>(a, st);
    }
    VtArgsM<false, false, false, MD> a{};
    if (const int rc = pack(a)) return rc;
    fill(a);
    return launch_mask<MD, false, false, false>(a, st);
}

}  // namespace

extern "C" int impala_vtrace_loss_mask(const float* cur_logits, const float* beh_logits, const int32_t* actions,
                                       const float* rewards, const uint8_t* done, const int32_t* lens, const float* v,
                                       float* vs, float* pg_adv, float* dlogits, float* dv, double* scalars,
                                       void* workspace, int64_t workspace_bytes, int T, int B, int A, float gamma,
                                       float rho_bar, float c_bar, float v_loss_c, float policy_loss_c,
                                       float entropy_c, float inv_batch, int mode, double* diag, const double* popart,
                                       int reward_clip, const int32_t* host_heads, int K, void* stream) {
    if (A > 32) return IMPALA_ERR_UNSUPPORTED_SHAPE;  // one 32-bit legal word per step
    // multi-discrete: the heads, read here and packed by value into the argument block (captured graphs keep them)
    unsigned mask = 0u;
    if (host_heads) {
        if (K < 1) return IMPALA_ERR_BAD_ARG;
        if (K > kMaxHeads) return IMPALA_ERR_UNSUPPORTED_SHAPE;
        int start = 0;
        for (int k = 0; k < K; ++k) {
            if (host_heads[k] < 2 || start + host_heads[k] > A) return IMPALA_ERR_BAD_ARG;
            mask |= 1u << start;
            start += host_heads[k];
        }
        if (start != A) return IMPALA_ERR_BAD_ARG;
    } else if (reinterpret_cast<uintptr_t>(actions) & 7) {
        return IMPALA_ERR_BAD_ARG;  // [a, legal] is read as one 64-bit load
    }
    if (reward_clip != 0 && reward_clip != IMPALA_REWARD_CLIP_ABS_ONE &&
        reward_clip != IMPALA_REWARD_CLIP_SOFT_ASYMMETRIC)
        return IMPALA_ERR_BAD_ARG;
    if (popart && !diag) return IMPALA_ERR_BAD_ARG;
    const int64_t need = loss_workspace(T, B, A, diag ? 12 : 4);
    const cudaStream_t st = (cudaStream_t)stream;
    auto pack = [&](VtArgs& a) {
        return loss_args(a, cur_logits, beh_logits, actions, rewards, done, lens, v, vs, pg_adv, dlogits, dv, scalars,
                         workspace, workspace_bytes, need, T, B, A, gamma, rho_bar, c_bar, v_loss_c, policy_loss_c,
                         entropy_c, inv_batch, mode);
    };
    if (host_heads)
        return dispatch<true>(pack, [&](auto& a) { a.head_mask = mask; }, diag, popart, reward_clip, st);
    return dispatch<false>(pack, [](auto&) {}, diag, popart, reward_clip, st);
}
