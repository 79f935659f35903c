// Two-layer MLP forward / backward on FP32 CUDA cores (reference models.py:12-25,40-52
// in eval mode; autograd of the same at learner.py:175).
//
// Mapping ("a thread owns hidden units"): thread `tid` owns hidden units
// j = tid + q*blockDim (q < JPT) and keeps their W1 rows, b1 and W2 columns in registers
// for the lifetime of its persistent CTA.  A tile is 32 consecutive rows of the flattened
// (M, O) observation matrix, staged in shared memory and consumed in register blocks of 8
// rows through warp-broadcast 128-bit loads (8*JPT FFMA per LDS.128).  Hidden activations
// never leave registers: the forward reduces layer 2 across the CTA with a transposing
// warp butterfly (the CTA spans the whole hidden layer); the backward recomputes them,
// and because every gradient entry of W1/b1/W2 belongs to exactly one hidden unit each
// thread accumulates its own slice in registers across all its tiles - no atomics,
// deterministic; wide hidden layers are split over blockIdx.y.  Per-CTA partials are then
// summed in float64 by a second small kernel.
//
// This file: the route that picks the kernels of every MLP call, the FP32 configuration, the occupancy
// cache, the partial reduction and the C-ABI entry points.  Kernel templates: mlp_kernels.cuh; instantiations: mlp_inst.cu.
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>

#include "mlp_kernels.cuh"

namespace {

// grad[i] = sum_c ws[c][i] in float64.  A CTA covers 32 consecutive entries (one 128-byte
// line per partial row); its 8 warps split the partial rows, so every load instruction is
// one fully coalesced line and 8 x 4 loads are in flight per entry.  Fixed summation
// order -> bitwise reproducible gradients.
constexpr int kRedWarps = 8;
constexpr int64_t kWsHeader = 256;  // control words of the tensor-core backward's grid barrier
__global__ void __launch_bounds__(kRedWarps * 32)
reduce_partials_kernel(const float* __restrict__ ws, double* __restrict__ grad, int nparts,
                       int64_t total) {
    __shared__ double s_sum[kRedWarps][33];
    const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * 32 + lane;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    if (i < total) {
        int c = g;
        for (; c + 3 * kRedWarps < nparts; c += 4 * kRedWarps) {
            const float a0 = __ldg(ws + (size_t)c * total + i);
            const float a1 = __ldg(ws + (size_t)(c + kRedWarps) * total + i);
            const float a2 = __ldg(ws + (size_t)(c + 2 * kRedWarps) * total + i);
            const float a3 = __ldg(ws + (size_t)(c + 3 * kRedWarps) * total + i);
            s0 += a0, s1 += a1, s2 += a2, s3 += a3;
        }
        for (; c < nparts; c += kRedWarps) s0 += __ldg(ws + (size_t)c * total + i);
    }
    s_sum[g][lane] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    if (g == 0 && i < total) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kRedWarps; ++w) s += s_sum[w][lane];
        grad[i] = s;
    }
}

bool pick_config(int O, int H, int N2, bool bwd, MlpConfig* c) {
    if (O < 1 || H < 1 || N2 < 1) return false;
    if (O <= 8) c->op = 8;
    else if (O <= 24) c->op = 24;
    else if (O <= 32) c->op = 32;
    else if (O <= 64) c->op = 64;
    else if (O <= 128) c->op = 128;
    else return false;
    if (N2 <= 1) c->np = 1;
    else if (N2 <= 4) c->np = 4;
    else if (N2 <= 16) c->np = 16;
    else if (N2 <= 32) c->np = 32;
    else return false;
    if (c->op == 128 || c->np == 32) {
        // wide observations or outputs: one hidden unit per thread (the forward then holds at most 256
        // units); the backward splits a unit's features over a lane quad from OP = 64 up (ks = 4: 2 x 32
        // at OP = 128) and over a lane pair below it, and at NP = 32 its W2 column as well
        c->jpt = 1, c->maxt = 256;
        c->ks = bwd ? (c->op >= 64 ? 4 : 2) : 1;
    } else {
        // register budget: forward holds JPT*OP weights, backward 2*JPT*OP (weights + gradient); at OP = 64
        // the backward splits the features of a hidden unit over a lane pair (ks = 2: 2 x 32 + 2 x 32)
        c->ks = (bwd && c->op == 64) ? 2 : 1;
        if (H < 128 || (bwd && c->op == 64)) c->jpt = 1, c->maxt = bwd && H >= 128 ? 256 : 128;
        else c->jpt = 2, c->maxt = 256;
    }
    const int want = (int)impala_round_up((int64_t)c->ks * ((H + c->jpt - 1) / c->jpt), 32);
    if (bwd) {
        c->threads = want < c->maxt ? want : c->maxt;
        const int units = c->threads / c->ks * c->jpt;  // hidden units per CTA
        c->slices = (H + units - 1) / units;
    } else {
        if (want > c->maxt) return false;  // forward needs the whole hidden layer in one CTA
        c->threads = want;
        c->slices = 1;
    }
    return true;
}

// Arguments and dynamic shared memory of the FP32 kernels in configuration c (pick_config).
size_t fill_args(MlpArgs* a, const MlpConfig& c, bool bwd, int M, int O, int H, int N2) {
    a->M = M, a->O = O, a->H = H, a->N2 = N2;
    a->num_tiles = (M + kRows - 1) / kRows;
    a->lay = impala_make_layout(O, H, N2);
    const size_t tail = bwd ? (size_t)kRows * c.np : (size_t)(c.threads / 32) * kRows * c.np;
    return ((size_t)kRows * c.op + tail) * sizeof(float);
}

int dispatch(bool bwd, const MlpSplitArgs& a, const MlpConfig& c, size_t smem, cudaStream_t st,
             int* grid) {
    switch (c.op) {
        case 8: return bwd ? impala_mlp_bwd_op8(a, c, smem, st, grid) : impala_mlp_fwd_op8(a, c, smem, st, grid);
        case 24: return bwd ? impala_mlp_bwd_op24(a, c, smem, st, grid) : impala_mlp_fwd_op24(a, c, smem, st, grid);
        case 32: return bwd ? impala_mlp_bwd_op32(a, c, smem, st, grid) : impala_mlp_fwd_op32(a, c, smem, st, grid);
        case 64: return bwd ? impala_mlp_bwd_op64(a, c, smem, st, grid) : impala_mlp_fwd_op64(a, c, smem, st, grid);
        default: return bwd ? impala_mlp_bwd_op128(a, c, smem, st, grid) : impala_mlp_fwd_op128(a, c, smem, st, grid);
    }
}

bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// The one place that decides which kernels run an MLP call: the first row below that takes the shape.
// Returns IMPALA_OK and the plan, or the error of the call: IMPALA_ERR_UNSUPPORTED_SHAPE when no kernel
// takes the shape, IMPALA_ERR_WORKSPACE_TOO_SMALL when a backward's ws_bytes is below p->ws.
//
//   O > 128 or byte rows  Obs: 128 < O <= 1024, O % 4 == 0, H = 128 k <= 1024, N2 <= 32.  There is no FP32
//                         kernel for these widths, and byte rows of O <= 128 are refused (their callers
//                         widen them once with impala_obs_u8_to_f32).  Shape, then workspace, then alignment.
//   backward              the FP32 configuration and the workspace first: the FP32 kernels size it for all
//   Narrow                O = 4 k <= 28, N2 <= 4; forward H = 32 k <= 256, backward H = 128 or 256 with dout
//                         and grad 16-byte aligned as well
//   Wide                  O = 4 k <= 128, H = 128 k <= 4096, N2 <= 32
//   Fp32                  otherwise (O <= 128, N2 <= 32; the forward holds the hidden layer in one CTA)
//
// x_al: x aligned as the tensor-core kernels load it (16 bytes for float rows, 4 for byte rows).  Every
// tensor-core row needs it; a misaligned float x at O <= 128 goes to the FP32 kernels.  IMPALA_MLP_TC=0
// turns off every tensor-core row and IMPALA_MLP_TCW=0 all but Narrow.  Both are read on every call, so a
// process may flip them between steps.
int route(bool bwd, int M, int O, int H, int N2, bool bytes, bool x_al, bool dout_al, bool grad_al, int64_t ws_bytes,
          MlpPlan* p) {
    const bool tc = impala_env_int("IMPALA_MLP_TC", 1) != 0;
    const bool tcw = tc && impala_env_int("IMPALA_MLP_TCW", 1) != 0;
    *p = MlpPlan{};
    if (O > 128 || bytes) {
        if (O <= 128 || !tcw || M < 1 || O > 1024 || O % 4 || H < 128 || H > 1024 || H % 128 || N2 < 1 || N2 > 32)
            return IMPALA_ERR_UNSUPPORTED_SHAPE;
        p->kernel = MlpKernel::Obs, p->np = N2 == 1 ? 1 : N2 <= 4 ? 4 : 32;
        if (bwd && ws_bytes < (p->ws = kWsHeader + impala_mlp_obs_bwd_layout(M, O, H, N2).bytes))
            return IMPALA_ERR_WORKSPACE_TOO_SMALL;
        return x_al ? IMPALA_OK : IMPALA_ERR_UNSUPPORTED_SHAPE;
    }
    if (bwd) {
        if (M < 1 || !pick_config(O, H, N2, true, &p->fp32)) return IMPALA_ERR_UNSUPPORTED_SHAPE;
        const int64_t tiles = std::min<int64_t>((M + kRows - 1) / kRows, kMaxParts);
        p->ws = kWsHeader + tiles * impala_make_layout(O, H, N2).total * (int64_t)sizeof(float);
        if (ws_bytes < p->ws) return IMPALA_ERR_WORKSPACE_TOO_SMALL;
    }
    const bool tc_shape = tc && x_al && M >= 1 && O >= 4 && O % 4 == 0 && N2 >= 1;
    if (tc_shape && O <= 28 && N2 <= 4 &&
        (bwd ? (H == 128 || H == 256) && dout_al && grad_al : H >= 32 && H <= 256 && H % 32 == 0)) {
        // one K atom, the whole hidden layer in one pass (forward) or one 64-unit block per CTA (backward)
        p->kernel = MlpKernel::Narrow, p->np = N2 == 1 ? 1 : 4, p->ka = 1, p->hb = H, p->rows = 64;
        p->reduce_in_kernel = bwd;
        return IMPALA_OK;
    }
    if (tcw && tc_shape && H >= 128 && H % 128 == 0 && H <= 4096 && N2 <= 32) {
        p->kernel = MlpKernel::Wide, p->rows = 64;
        // 256 hidden units per pass fit at 16 outputs too: 88 064 B at one K atom, 219 136 B at two
        p->hb = H <= 256 ? H : H % 256 ? 128 : 256;
        if (O <= 64 && N2 <= 16) {
            p->np = N2 == 1 ? 1 : N2 <= 4 ? 4 : 16, p->ka = O <= 32 ? 1 : 2;
        } else if (bwd) {
            // four K atoms, GEMM2 in 64-feature halves, 32-row tiles; 5..32 outputs padded to 32
            p->np = N2 == 1 ? 1 : N2 <= 4 ? 4 : 32, p->ka = 4, p->rows = 32;
        } else if (N2 > 16 && O <= 64) {
            p->np = 32, p->ka = O <= 32 ? 1 : 2;
            if (p->ka == 2) p->hb = 128;  // 256 units would need 235 520 B with the padded W2 rows
        } else {
            // four K atoms: 64 hidden units per pass keep W1 hi / lo + both warpgroups' x stages in 227 KB
            p->np = N2 > 16 ? 32 : N2 > 4 ? 16 : N2 == 1 ? 1 : 4, p->ka = 4, p->hb = 64;
        }
        return IMPALA_OK;
    }
    if (!bwd && (M < 1 || !pick_config(O, H, N2, false, &p->fp32))) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    p->kernel = MlpKernel::Fp32;
    return IMPALA_OK;
}

// out_b != nullptr: split heads (out = head a of M_a rows, out_b = head b; mlp_kernels.cuh split_out)
int forward(const MlpPlan& p, const float* x, const float* params, float* out, int M, int O, int H, int N2,
            cudaStream_t st, float* out_b = nullptr, int M_a = 0) {
    if (p.kernel == MlpKernel::Obs) return impala_mlp_fwd_obs(p, x, params, out, M, O, H, N2, st, out_b, M_a);
    if (p.kernel != MlpKernel::Fp32) return impala_mlp_fwd_tc(p, x, params, out, M, O, H, N2, st, out_b, M_a);
    MlpSplitArgs a{};
    const size_t smem = fill_args(&a, p.fp32, false, M, O, H, N2);
    a.x = x, a.params = params, a.out = out, a.out_b = out_b, a.M_a = M_a;
    int grid = 0;
    return dispatch(false, a, p.fp32, smem, st, &grid);
}

// Wide observations (O > 128, float or byte rows): DP^T and two sets of partial rows in the workspace,
// each summed in float64.
template <typename XT>
int backward_obs(const MlpPlan& p, const XT* x, const float* params, const float* dout, double* grad,
                 void* workspace, int M, int O, int H, int N2, cudaStream_t st, const float* dout_b = nullptr,
                 int M_a = 0) {
    const ObsBwdLayout L = impala_mlp_obs_bwd_layout(M, O, H, N2);
    char* ws = static_cast<char*>(workspace) + kWsHeader;
    const int rc = impala_mlp_bwd_obs(p, x, params, dout, ws, L, M, O, H, N2, st, dout_b, M_a);
    if (rc != IMPALA_OK) return rc;
    const MlpLayout lay = impala_make_layout(O, H, N2);
    const int64_t nr = lay.total - lay.ob1;
    reduce_partials_kernel<<<(unsigned)((nr + 31) / 32), kRedWarps * 32, 0, st>>>(
        reinterpret_cast<const float*>(ws + L.rest_off), grad + lay.ob1, L.r1, nr);
    if (const int e = impala_launch_status(); e != IMPALA_OK) return e;
    reduce_partials_kernel<<<(unsigned)((lay.ob1 + 31) / 32), kRedWarps * 32, 0, st>>>(
        reinterpret_cast<const float*>(ws + L.w1_off), grad, L.p2, lay.ob1);
    return impala_launch_status();
}

// dout_b != nullptr: split heads (dout = head a of M_a rows, dout_b = head b; mlp_kernels.cuh split_dz)
int backward(const MlpPlan& p, const float* x, const float* params, const float* dout, double* grad, void* workspace,
             int M, int O, int H, int N2, cudaStream_t st, const float* dout_b = nullptr, int M_a = 0) {
    if (p.kernel == MlpKernel::Obs)
        return backward_obs(p, x, params, dout, grad, workspace, M, O, H, N2, st, dout_b, M_a);
    // workspace = [control words (kWsHeader bytes, zero-filled once by the caller) | partial rows]
    float* ws = reinterpret_cast<float*>(static_cast<char*>(workspace) + kWsHeader);
    if (p.reduce_in_kernel)
        return impala_mlp_bwd_tc(x, params, dout, ws, grad, static_cast<unsigned int*>(workspace), M, O, H, N2, st,
                                 dout_b, M_a);
    int grid = 0, rc;
    if (p.kernel == MlpKernel::Wide) {
        rc = impala_mlp_bwd_tcw(p, x, params, dout, ws, M, O, H, N2, st, &grid, dout_b, M_a);
    } else {
        MlpSplitArgs a{};
        const size_t smem = fill_args(&a, p.fp32, true, M, O, H, N2);
        a.x = x, a.params = params, a.dout = dout, a.ws = ws, a.dout_b = dout_b, a.M_a = M_a;
        rc = dispatch(true, a, p.fp32, smem, st, &grid);
    }
    if (rc != IMPALA_OK) return rc;
    const int64_t total = impala_make_layout(O, H, N2).total;
    reduce_partials_kernel<<<(unsigned)((total + 31) / 32), kRedWarps * 32, 0, st>>>(ws, grad, grid, total);
    return impala_launch_status();
}

// The paired backward that pushes to the peers: both networks on Narrow plans, >= 2 tiles between them.
bool push_plans(int M_pi, int M_vf, int O, int H_pi, int H_vf, int A, bool x_al, bool dlogits_al, bool dv_al,
                MlpPlan* pi, MlpPlan* vf) {
    return A >= 2 && A <= 4 && route(true, M_pi, O, H_pi, A, false, x_al, dlogits_al, true, INT64_MAX, pi) == IMPALA_OK &&
           pi->kernel == MlpKernel::Narrow &&
           route(true, M_vf, O, H_vf, 1, false, x_al, dv_al, true, INT64_MAX, vf) == IMPALA_OK &&
           vf->kernel == MlpKernel::Narrow && (M_pi + 63) / 64 + (M_vf + 63) / 64 >= 2;
}

}  // namespace

cudaError_t impala_resident_ctas(const void* kernel, int threads, size_t smem, int* per_sm) {
    static std::mutex mu;
    // The dynamic shared-memory limit is a property of the KERNEL (per device), not of one launch
    // configuration: it is only ever raised.  (Setting it per (threads, smem) entry lowered it when the same
    // instantiation was used with a narrower hidden layer, and the next launch of the wider, already
    // cached configuration failed with cudaErrorInvalidValue.)
    static std::map<std::pair<const void*, int>, size_t> opted;
    static std::map<std::tuple<const void*, int, int, size_t>, int> cached;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    const auto key = std::make_tuple(kernel, dev, threads, smem);
    if (const auto it = cached.find(key); it != cached.end()) return *per_sm = it->second, cudaSuccess;
    size_t& o = opted[std::make_pair(kernel, dev)];
    if (smem > o) {
        if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return e;
        o = smem;
    }
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kernel, threads, smem)) != cudaSuccess) return e;
    cached[key] = *per_sm;
    return cudaSuccess;
}

// Persistent grid = resident CTAs per SM x SM count / slices.
template <typename Args>
int launch_persistent(void (*kernel)(Args), const Args& a, const MlpConfig& c, size_t smem, cudaStream_t st,
                      int* grid_out) {
    int per_sm = 0, sms = 0;
    cudaError_t e;
    if ((e = impala_resident_ctas((const void*)kernel, c.threads, smem, &per_sm)) != cudaSuccess) return (int)e;
    if ((e = impala_sm_count(&sms)) != cudaSuccess) return (int)e;
    if (per_sm < 1) return IMPALA_ERR_UNSUPPORTED_SHAPE;
    int grid = per_sm * sms / c.slices;
    if (grid < 1) grid = 1;
    if (grid > a.num_tiles) grid = a.num_tiles;
    if (grid > kMaxParts) grid = kMaxParts;
    kernel<<<dim3(grid, c.slices), c.threads, smem, st>>>(a);
    *grid_out = grid;
    return impala_launch_status();
}

int impala_mlp_launch(void (*kernel)(MlpArgs), const MlpArgs& a, const MlpConfig& c, size_t smem,
                      cudaStream_t st, int* grid_out) {
    return launch_persistent(kernel, a, c, smem, st, grid_out);
}
int impala_mlp_launch(void (*kernel)(MlpSplitArgs), const MlpSplitArgs& a, const MlpConfig& c, size_t smem,
                      cudaStream_t st, int* grid_out) {
    return launch_persistent(kernel, a, c, smem, st, grid_out);
}

extern "C" int impala_mlp_forward(const float* x, const float* params, float* out, int M, int O,
                                  int H, int N2, void* stream) {
    if (!x || !params || !out) return IMPALA_ERR_BAD_ARG;
    MlpPlan p;
    const int rc = route(false, M, O, H, N2, false, aligned(x, 16), true, true, 0, &p);
    return rc != IMPALA_OK ? rc : forward(p, x, params, out, M, O, H, N2, (cudaStream_t)stream);
}

extern "C" int impala_mlp_forward_pair(const float* x, const float* params_pi, const float* params_vf,
                                       float* logits, float* values, int M_pi, int M_vf, int O,
                                       int H_pi, int H_vf, int A, void* stream) {
    if (!x || !params_pi || !params_vf || !logits || !values) return IMPALA_ERR_BAD_ARG;
    const cudaStream_t st = (cudaStream_t)stream;
    MlpPlan pi, vf;
    int rc = route(false, M_pi, O, H_pi, A, false, aligned(x, 16), true, true, 0, &pi);
    if (rc == IMPALA_OK) rc = route(false, M_vf, O, H_vf, 1, false, aligned(x, 16), true, true, 0, &vf);
    if (rc != IMPALA_OK) return rc;
    if (A >= 2 && A <= 4 && pi.kernel == MlpKernel::Narrow && vf.kernel == MlpKernel::Narrow)
        return impala_mlp_fwd_tc_pair(x, params_pi, params_vf, logits, values, M_pi, M_vf, O, H_pi, H_vf, A, st);
    if ((rc = forward(pi, x, params_pi, logits, M_pi, O, H_pi, A, st)) != IMPALA_OK) return rc;
    return forward(vf, x, params_vf, values, M_vf, O, H_vf, 1, st);
}

extern "C" int64_t impala_mlp_backward_workspace(int M, int O, int H, int N2) {
    MlpPlan p;
    const int rc = route(true, M, O, H, N2, false, true, true, true, INT64_MAX, &p);
    return rc != IMPALA_OK ? rc : p.ws;
}

extern "C" int impala_mlp_backward(const float* x, const float* params, const float* dout,
                                   double* grad, void* workspace, int64_t workspace_bytes, int M,
                                   int O, int H, int N2, void* stream) {
    if (!x || !params || !dout || !grad || !workspace) return IMPALA_ERR_BAD_ARG;
    MlpPlan p;
    const int rc = route(true, M, O, H, N2, false, aligned(x, 16), aligned(dout, 16), aligned(grad, 16),
                         workspace_bytes, &p);
    return rc != IMPALA_OK ? rc : backward(p, x, params, dout, grad, workspace, M, O, H, N2, (cudaStream_t)stream);
}

// ---- byte observations: the K-streamed kernels read uint8 rows (O > 128); narrower shapes are refused,
// their callers widen the rows once with impala_obs_u8_to_f32
extern "C" int impala_mlp_forward_u8(const uint8_t* x, const float* params, float* out, int M, int O, int H, int N2,
                                     void* stream) {
    if (!x || !params || !out) return IMPALA_ERR_BAD_ARG;
    MlpPlan p;
    const int rc = route(false, M, O, H, N2, true, aligned(x, 4), true, true, 0, &p);
    return rc != IMPALA_OK ? rc : impala_mlp_fwd_obs(p, x, params, out, M, O, H, N2, (cudaStream_t)stream);
}

extern "C" int impala_mlp_backward_u8(const uint8_t* x, const float* params, const float* dout, double* grad,
                                      void* workspace, int64_t workspace_bytes, int M, int O, int H, int N2,
                                      void* stream) {
    if (!x || !params || !dout || !grad || !workspace) return IMPALA_ERR_BAD_ARG;
    MlpPlan p;
    const int rc = route(true, M, O, H, N2, true, aligned(x, 4), true, true, workspace_bytes, &p);
    return rc != IMPALA_OK ? rc
                           : backward_obs(p, x, params, dout, grad, workspace, M, O, H, N2, (cudaStream_t)stream);
}

extern "C" int impala_mlp_backward_pair(const float* x, const float* params_pi, const float* params_vf,
                                        const float* dlogits, const float* dv, double* grad_pi,
                                        double* grad_vf, void* workspace_pi, int64_t workspace_pi_bytes,
                                        void* workspace_vf, int64_t workspace_vf_bytes, int M_pi, int M_vf,
                                        int O, int H_pi, int H_vf, int A, void* stream) {
    if (!x || !params_pi || !params_vf || !dlogits || !dv || !grad_pi || !grad_vf || !workspace_pi ||
        !workspace_vf)
        return IMPALA_ERR_BAD_ARG;
    const cudaStream_t st = (cudaStream_t)stream;
    MlpPlan pi, vf;
    int rc = route(true, M_pi, O, H_pi, A, false, aligned(x, 16), aligned(dlogits, 16), aligned(grad_pi, 16),
                   workspace_pi_bytes, &pi);
    if (rc == IMPALA_OK)
        rc = route(true, M_vf, O, H_vf, 1, false, aligned(x, 16), aligned(dv, 16), aligned(grad_vf, 16),
                   workspace_vf_bytes, &vf);
    if (rc != IMPALA_OK) return rc;
    if (A >= 2 && A <= 4 && pi.kernel == MlpKernel::Narrow && vf.kernel == MlpKernel::Narrow)
        return impala_mlp_bwd_tc_pair(
            x, params_pi, params_vf, dlogits, dv,
            reinterpret_cast<float*>(static_cast<char*>(workspace_pi) + kWsHeader),
            reinterpret_cast<float*>(static_cast<char*>(workspace_vf) + kWsHeader), grad_pi, grad_vf,
            static_cast<unsigned int*>(workspace_pi), M_pi, M_vf, O, H_pi, H_vf, A, st);
    if ((rc = backward(pi, x, params_pi, dlogits, grad_pi, workspace_pi, M_pi, O, H_pi, A, st)) != IMPALA_OK) return rc;
    return backward(vf, x, params_vf, dv, grad_vf, workspace_vf, M_vf, O, H_vf, 1, st);
}

// ---- data-parallel learner: the paired backward that pushes its result to the peers (optim.cu)
extern "C" int impala_mlp_backward_pair_push_supported(int M_pi, int M_vf, int O, int H_pi, int H_vf, int A) {
    MlpPlan pi, vf;
    return push_plans(M_pi, M_vf, O, H_pi, H_vf, A, true, true, true, &pi, &vf);
}

// The two push entry points: n_extra logged extras (at most 32), then n_obs observation sums (0, or 2 O + 1).
static int pair_push(const float* x, const float* params_pi, const float* params_vf, const float* dlogits,
                     const float* dv, void* workspace_pi, int64_t workspace_pi_bytes, void* workspace_vf,
                     int64_t workspace_vf_bytes, int M_pi, int M_vf, int O, int H_pi, int H_vf, int A,
                     const double* extra, int n_extra, int n_obs, void* const* peer_gather, const long long* seq,
                     int64_t slot_stride, int64_t buf_stride, int rank, int world, void* stream) {
    if (!x || !params_pi || !params_vf || !dlogits || !dv || !workspace_pi || !workspace_vf || !peer_gather ||
        !seq || (n_extra + n_obs > 0 && !extra))
        return IMPALA_ERR_BAD_ARG;
    if (world < 1 || world > 8 || rank < 0 || rank >= world || n_extra < 0 || n_extra > 32) return IMPALA_ERR_BAD_ARG;
    n_extra += n_obs;
    MlpPlan pi, vf;
    if (!push_plans(M_pi, M_vf, O, H_pi, H_vf, A, aligned(x, 16), aligned(dlogits, 16), aligned(dv, 16), &pi, &vf))
        return IMPALA_ERR_UNSUPPORTED_SHAPE;
    const int64_t n_pi = impala_make_layout(O, H_pi, A).total, n_vf = impala_make_layout(O, H_vf, 1).total;
    if (slot_stride < n_pi + n_vf + n_extra || buf_stride < (int64_t)world * slot_stride) return IMPALA_ERR_BAD_ARG;
    if (workspace_pi_bytes < pi.ws || workspace_vf_bytes < vf.ws) return IMPALA_ERR_WORKSPACE_TOO_SMALL;
    const PushArgs push{reinterpret_cast<ulonglong2* const*>(peer_gather), seq, slot_stride, buf_stride, rank, world};
    return impala_mlp_bwd_tc_pair(
        x, params_pi, params_vf, dlogits, dv,
        reinterpret_cast<float*>(static_cast<char*>(workspace_pi) + kWsHeader),
        reinterpret_cast<float*>(static_cast<char*>(workspace_vf) + kWsHeader), nullptr, nullptr,
        static_cast<unsigned int*>(workspace_pi), M_pi, M_vf, O, H_pi, H_vf, A, (cudaStream_t)stream, &push, extra,
        n_extra);
}

extern "C" int impala_mlp_backward_pair_push(const float* x, const float* params_pi, const float* params_vf,
                                             const float* dlogits, const float* dv, void* workspace_pi,
                                             int64_t workspace_pi_bytes, void* workspace_vf,
                                             int64_t workspace_vf_bytes, int M_pi, int M_vf, int O, int H_pi,
                                             int H_vf, int A, const double* extra, int n_extra,
                                             void* const* peer_gather, const long long* seq,
                                             int64_t slot_stride, int64_t buf_stride, int rank, int world,
                                             void* stream) {
    return pair_push(x, params_pi, params_vf, dlogits, dv, workspace_pi, workspace_pi_bytes, workspace_vf,
                     workspace_vf_bytes, M_pi, M_vf, O, H_pi, H_vf, A, extra, n_extra, 0, peer_gather, seq, slot_stride,
                     buf_stride, rank, world, stream);
}

extern "C" int impala_mlp_backward_pair_push_obs_norm(const float* x, const float* params_pi, const float* params_vf,
                                                      const float* dlogits, const float* dv, void* workspace_pi,
                                                      int64_t workspace_pi_bytes, void* workspace_vf,
                                                      int64_t workspace_vf_bytes, int M_pi, int M_vf, int O, int H_pi,
                                                      int H_vf, int A, const double* extra, int n_extra,
                                                      void* const* peer_gather, const long long* seq,
                                                      int64_t slot_stride, int64_t buf_stride, int rank, int world,
                                                      void* stream) {
    if (O > IMPALA_OBS_NORM_MAX_FEATURES) return IMPALA_ERR_BAD_ARG;
    return pair_push(x, params_pi, params_vf, dlogits, dv, workspace_pi, workspace_pi_bytes, workspace_vf,
                     workspace_vf_bytes, M_pi, M_vf, O, H_pi, H_vf, A, extra, n_extra, 2 * O + 1, peer_gather, seq,
                     slot_stride, buf_stride, rank, world, stream);
}

// ---- shared-torso network: one MLP with N + 1 outputs [policy | value] over M = (T + 1) B rows, whose
// outputs (and output gradients) live in two buffers - the policy logits (M_a = T B rows of N) and the
// values (M rows) - so the V-trace kernel reads and writes them where it does for two networks.
// Bitwise equal to impala_mlp_forward / impala_mlp_backward with N2 = N + 1 on the interleaved layout.
namespace {

bool shared_args_ok(int x_dtype, int M_a, int M, int N) {
    return (x_dtype == IMPALA_OBS_F32 || x_dtype == IMPALA_OBS_U8) && N >= 1 && N + 1 <= 32 && M_a >= 0 && M_a <= M;
}

}  // namespace

extern "C" int impala_mlp_forward_shared(const void* x, int x_dtype, const float* params, float* logits,
                                         float* values, int M_a, int M, int O, int H, int N, void* stream) {
    if (!x || !params || !logits || !values || !shared_args_ok(x_dtype, M_a, M, N)) return IMPALA_ERR_BAD_ARG;
    const bool bytes = x_dtype == IMPALA_OBS_U8;
    const cudaStream_t st = (cudaStream_t)stream;
    MlpPlan p;
    const int rc = route(false, M, O, H, N + 1, bytes, aligned(x, bytes ? 4 : 16), true, true, 0, &p);
    if (rc != IMPALA_OK) return rc;
    if (bytes)
        return impala_mlp_fwd_obs(p, static_cast<const uint8_t*>(x), params, logits, M, O, H, N + 1, st, values, M_a);
    return forward(p, static_cast<const float*>(x), params, logits, M, O, H, N + 1, st, values, M_a);
}

extern "C" int impala_mlp_backward_shared(const void* x, int x_dtype, const float* params, const float* dlogits,
                                          const float* dv, double* grad, void* workspace, int64_t workspace_bytes,
                                          int M_a, int M, int O, int H, int N, void* stream) {
    if (!x || !params || !dlogits || !dv || !grad || !workspace || !shared_args_ok(x_dtype, M_a, M, N))
        return IMPALA_ERR_BAD_ARG;
    const bool bytes = x_dtype == IMPALA_OBS_U8;
    const cudaStream_t st = (cudaStream_t)stream;
    MlpPlan p;
    const int rc = route(true, M, O, H, N + 1, bytes, aligned(x, bytes ? 4 : 16), aligned(dlogits, 16) && aligned(dv, 16),
                         aligned(grad, 16), workspace_bytes, &p);
    if (rc != IMPALA_OK) return rc;
    if (bytes)
        return backward_obs(p, static_cast<const uint8_t*>(x), params, dlogits, grad, workspace, M, O, H, N + 1, st, dv,
                            M_a);
    return backward(p, static_cast<const float*>(x), params, dlogits, grad, workspace, M, O, H, N + 1, st, dv, M_a);
}

// out[i] = x[i] (exact): 4 bytes -> one float4 per thread and iteration when both pointers allow it
template <bool kVec>
__global__ void __launch_bounds__(256) obs_u8_to_f32_kernel(const uint8_t* __restrict__ x, float* __restrict__ out,
                                                            int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t done = 0;
    if constexpr (kVec) {
        const int64_t n4 = n >> 2;
        for (int64_t i = t; i < n4; i += stride) {
            const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(x) + i);
            reinterpret_cast<float4*>(out)[i] = make_float4((float)(w & 255u), (float)((w >> 8) & 255u),
                                                            (float)((w >> 16) & 255u), (float)(w >> 24));
        }
        done = n4 << 2;
    }
    for (int64_t i = done + t; i < n; i += stride) out[i] = (float)x[i];
}

extern "C" int impala_obs_u8_to_f32(const uint8_t* x, float* out, int64_t n, void* stream) {
    if (!x || !out || n < 0) return IMPALA_ERR_BAD_ARG;
    if (n == 0) return IMPALA_OK;
    int sms = 0;
    if (const cudaError_t e = impala_sm_count(&sms); e != cudaSuccess) return (int)e;
    const bool vec = ((reinterpret_cast<uintptr_t>(x) & 3) | (reinterpret_cast<uintptr_t>(out) & 15)) == 0;
    const int64_t work = vec ? (n + 3) / 4 : n;
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((work + 255) / 256, (int64_t)sms * 16));
    if (vec)
        obs_u8_to_f32_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(x, out, n);
    else
        obs_u8_to_f32_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(x, out, n);
    return impala_launch_status();
}
