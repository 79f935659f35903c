// Entry point of the diagonal-Gaussian V-trace + loss kernels: the GAUSS instantiations of vtrace_loss.cuh's
// kernel, plain, diag and PopArt, each with and without the reward transform.
#include "vtrace_loss.cuh"

namespace {

template <bool DIAG, bool POPART, bool RCLIP>
int launch_gauss(VtArgsT<DIAG, POPART, RCLIP>& a, cudaStream_t st) {
    return launch<true, DIAG, POPART, RCLIP, true>(a, st);
}

}  // namespace

extern "C" int impala_vtrace_loss_gauss(const float* cur_params, const float* beh_params, const float* actions,
                                        const float* rewards, const uint8_t* done, const int32_t* lens,
                                        const float* v, float* vs, float* pg_adv, float* dparams, float* dv,
                                        double* scalars, void* workspace, int64_t workspace_bytes, int T, int B,
                                        int A, float gamma, float rho_bar, float c_bar, float v_loss_c,
                                        float policy_loss_c, float entropy_c, float inv_batch, int mode,
                                        double* diag, const double* popart, int reward_clip, void* stream) {
    if (reward_clip != 0 && reward_clip != IMPALA_REWARD_CLIP_ABS_ONE &&
        reward_clip != IMPALA_REWARD_CLIP_SOFT_ASYMMETRIC)
        return IMPALA_ERR_BAD_ARG;
    if (popart && !diag) return IMPALA_ERR_BAD_ARG;
    const int64_t need = loss_workspace(T, B, A, diag ? 12 : 4);
    const cudaStream_t st = (cudaStream_t)stream;
    // the kernel reads the float32 samples through the actions pointer of the argument block
    const int32_t* act = reinterpret_cast<const int32_t*>(actions);
    auto pack = [&](VtArgs& a) {
        return loss_args(a, cur_params, beh_params, act, rewards, done, lens, v, vs, pg_adv, dparams, dv, scalars,
                         workspace, workspace_bytes, need, T, B, A, gamma, rho_bar, c_bar, v_loss_c, policy_loss_c,
                         entropy_c, inv_batch, mode);
    };
    if (reward_clip) {
        if (popart) {
            VtArgsT<true, true, true> a{};
            if (const int rc = pack(a)) return rc;
            a.diag = diag, a.popart = popart, a.reward_clip = reward_clip;
            return launch_gauss<true, true, true>(a, st);
        }
        if (diag) {
            VtArgsT<true, false, true> a{};
            if (const int rc = pack(a)) return rc;
            a.diag = diag, a.reward_clip = reward_clip;
            return launch_gauss<true, false, true>(a, st);
        }
        VtArgsT<false, false, true> a{};
        if (const int rc = pack(a)) return rc;
        a.reward_clip = reward_clip;
        return launch_gauss<false, false, true>(a, st);
    }
    if (popart) {
        VtArgsT<true, true, false> a{};
        if (const int rc = pack(a)) return rc;
        a.diag = diag, a.popart = popart;
        return launch_gauss<true, true, false>(a, st);
    }
    if (diag) {
        VtArgsT<true, false, false> a{};
        if (const int rc = pack(a)) return rc;
        a.diag = diag;
        return launch_gauss<true, false, false>(a, st);
    }
    VtArgsT<false, false, false> a{};
    if (const int rc = pack(a)) return rc;
    return launch_gauss<false, false, false>(a, st);
}
