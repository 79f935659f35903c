// Entry points of the plain, diag and PopArt V-trace + loss kernels (the body: vtrace_loss.cuh).
#include "vtrace_loss.cuh"

extern "C" int impala_vtrace(const float* cur_logits, const float* beh_logits,
                             const int32_t* actions, const float* rewards, const uint8_t* done,
                             const int32_t* lens, const float* v, float* vs, float* pg_adv, int T,
                             int B, int A, float gamma, float rho_bar, float c_bar, int mode,
                             void* stream) {
    if (!cur_logits || !beh_logits || !actions || !rewards || !done || !lens || !v || !vs || !pg_adv)
        return IMPALA_ERR_BAD_ARG;
    if (mode != IMPALA_MODE_REFERENCE && mode != IMPALA_MODE_PAPER) return IMPALA_ERR_BAD_ARG;
    VtArgs a{};
    a.cur_logits = cur_logits, a.beh_logits = beh_logits, a.actions = actions, a.rewards = rewards;
    a.done = done, a.lens = lens, a.v = v, a.vs = vs, a.pg_adv = pg_adv;
    a.T = T, a.B = B, a.A = A, a.mode = mode;
    a.gamma = gamma, a.rho_bar = rho_bar, a.c_bar = c_bar;
    return launch<false>(a, (cudaStream_t)stream);
}

extern "C" int64_t impala_vtrace_loss_workspace(int T, int B, int A) { return loss_workspace(T, B, A, 4); }

extern "C" int impala_vtrace_loss(const float* cur_logits, const float* beh_logits,
                                  const int32_t* actions, const float* rewards,
                                  const uint8_t* done, const int32_t* lens, const float* v,
                                  float* vs, float* pg_adv, float* dlogits, float* dv,
                                  double* scalars, void* workspace, int64_t workspace_bytes, int T,
                                  int B, int A, float gamma, float rho_bar, float c_bar,
                                  float v_loss_c, float policy_loss_c, float entropy_c,
                                  float inv_batch, int mode, void* stream) {
    VtArgs a{};
    const int rc = loss_args(a, cur_logits, beh_logits, actions, rewards, done, lens, v, vs, pg_adv, dlogits, dv,
                             scalars, workspace, workspace_bytes, impala_vtrace_loss_workspace(T, B, A), T, B, A,
                             gamma, rho_bar, c_bar, v_loss_c, policy_loss_c, entropy_c, inv_batch, mode);
    if (rc) return rc;
    return launch<true>(a, (cudaStream_t)stream);
}

extern "C" int64_t impala_vtrace_loss_diag_workspace(int T, int B, int A) { return loss_workspace(T, B, A, 12); }

extern "C" int impala_vtrace_loss_diag(const float* cur_logits, const float* beh_logits,
                                       const int32_t* actions, const float* rewards,
                                       const uint8_t* done, const int32_t* lens, const float* v,
                                       float* vs, float* pg_adv, float* dlogits, float* dv,
                                       double* scalars, double* diag, void* workspace,
                                       int64_t workspace_bytes, int T, int B, int A, float gamma,
                                       float rho_bar, float c_bar, float v_loss_c,
                                       float policy_loss_c, float entropy_c, float inv_batch,
                                       int mode, void* stream) {
    if (!diag) return IMPALA_ERR_BAD_ARG;
    VtDiagArgs a{};
    const int rc = loss_args(a, cur_logits, beh_logits, actions, rewards, done, lens, v, vs, pg_adv, dlogits, dv,
                             scalars, workspace, workspace_bytes, impala_vtrace_loss_diag_workspace(T, B, A), T, B,
                             A, gamma, rho_bar, c_bar, v_loss_c, policy_loss_c, entropy_c, inv_batch, mode);
    if (rc) return rc;
    a.diag = diag;
    return launch<true, true>(a, (cudaStream_t)stream);
}

extern "C" int impala_vtrace_loss_popart(const float* cur_logits, const float* beh_logits,
                                         const int32_t* actions, const float* rewards,
                                         const uint8_t* done, const int32_t* lens, const float* v,
                                         float* vs, float* pg_adv, float* dlogits, float* dv,
                                         double* scalars, double* diag, void* workspace,
                                         int64_t workspace_bytes, int T, int B, int A, float gamma,
                                         float rho_bar, float c_bar, float v_loss_c,
                                         float policy_loss_c, float entropy_c, float inv_batch,
                                         int mode, const double* popart, void* stream) {
    if (!diag || !popart) return IMPALA_ERR_BAD_ARG;
    VtPopArgs a{};
    const int rc = loss_args(a, cur_logits, beh_logits, actions, rewards, done, lens, v, vs, pg_adv, dlogits, dv,
                             scalars, workspace, workspace_bytes, impala_vtrace_loss_diag_workspace(T, B, A), T, B,
                             A, gamma, rho_bar, c_bar, v_loss_c, policy_loss_c, entropy_c, inv_batch, mode);
    if (rc) return rc;
    a.diag = diag, a.popart = popart;
    return launch<true, true, true>(a, (cudaStream_t)stream);
}
