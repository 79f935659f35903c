// Entry point of the reward-clipping V-trace + loss kernels: the RCLIP instantiations of vtrace_loss.cuh's
// kernel on top of the plain, diag and PopArt ones.
#include "vtrace_loss.cuh"

extern "C" int impala_vtrace_loss_rclip(const float* cur_logits, const float* beh_logits,
                                        const int32_t* actions, const float* rewards,
                                        const uint8_t* done, const int32_t* lens, const float* v,
                                        float* vs, float* pg_adv, float* dlogits, float* dv,
                                        double* scalars, void* workspace, int64_t workspace_bytes, int T,
                                        int B, int A, float gamma, float rho_bar, float c_bar,
                                        float v_loss_c, float policy_loss_c, float entropy_c,
                                        float inv_batch, int mode, double* diag, const double* popart,
                                        int reward_clip, void* stream) {
    if (reward_clip != IMPALA_REWARD_CLIP_ABS_ONE && reward_clip != IMPALA_REWARD_CLIP_SOFT_ASYMMETRIC)
        return IMPALA_ERR_BAD_ARG;
    if (popart && !diag) return IMPALA_ERR_BAD_ARG;
    const int64_t need = loss_workspace(T, B, A, diag ? 12 : 4);
    const cudaStream_t st = (cudaStream_t)stream;
    auto pack = [&](VtArgs& a) {
        return loss_args(a, cur_logits, beh_logits, actions, rewards, done, lens, v, vs, pg_adv, dlogits, dv,
                         scalars, workspace, workspace_bytes, need, T, B, A, gamma, rho_bar, c_bar, v_loss_c,
                         policy_loss_c, entropy_c, inv_batch, mode);
    };
    if (popart) {
        VtArgsT<true, true, true> a{};
        if (const int rc = pack(a)) return rc;
        a.diag = diag, a.popart = popart, a.reward_clip = reward_clip;
        return launch<true, true, true, true>(a, st);
    }
    if (diag) {
        VtArgsT<true, false, true> a{};
        if (const int rc = pack(a)) return rc;
        a.diag = diag, a.reward_clip = reward_clip;
        return launch<true, true, false, true>(a, st);
    }
    VtArgsT<false, false, true> a{};
    if (const int rc = pack(a)) return rc;
    a.reward_clip = reward_clip;
    return launch<true, false, false, true>(a, st);
}
