// Layout helpers and ingest: the parts of the C ABI that launch no kernel of their own.
#include <string.h>

#include "common.cuh"

long long g_impala_launches = 0;

extern "C" int impala_abi_version(void) { return 1; }

extern "C" long long impala_launch_count(void) { return __atomic_load_n(&g_impala_launches, __ATOMIC_RELAXED); }

extern "C" int impala_compiled_sm(void) { return 90; }

extern "C" int impala_param_layout(int O, int H, int N2, int64_t offsets[4], int64_t* total) {
    if (O < 1 || H < 1 || N2 < 1 || !offsets || !total) return IMPALA_ERR_BAD_ARG;
    const MlpLayout l = impala_make_layout(O, H, N2);
    offsets[0] = l.oW1, offsets[1] = l.ob1, offsets[2] = l.oW2, offsets[3] = l.ob2;
    *total = l.total;
    return IMPALA_OK;
}

// bytes of one observation value, 0 for an unknown obs_dtype
static int64_t obs_bytes(int obs_dtype) {
    return obs_dtype == IMPALA_OBS_F32 ? 4 : obs_dtype == IMPALA_OBS_U8 ? 1 : 0;
}

// multi-discrete: 1 <= K <= 16 heads of at least two actions each among the A outputs; masked: categorical or
// multi-discrete, at most 32 outputs (one legal word)
static bool act_kind_ok(int act_kind, int A) {
    if (act_kind & IMPALA_ACT_MASKED) {
        const int base = act_kind & ~IMPALA_ACT_MASKED;
        return A <= 32 && (base == IMPALA_ACT_CATEGORICAL || (impala_md_heads(base) && act_kind_ok(base, A)));
    }
    if (act_kind == IMPALA_ACT_CATEGORICAL || act_kind == IMPALA_ACT_GAUSSIAN) return true;
    const int K = impala_md_heads(act_kind);
    return K >= 1 && K <= 16 && A >= 2 * K;
}

extern "C" int impala_batch_layout_act(int T, int B, int F, int frames, int A, int obs_dtype, int act_kind,
                                       int64_t offsets[6], int64_t* total_bytes) {
    const int64_t ob = obs_bytes(obs_dtype);
    if (T < 1 || B < 1 || F < 1 || frames < 1 || A < 1 || ob == 0 || !act_kind_ok(act_kind, A) || !offsets ||
        !total_bytes)
        return IMPALA_ERR_BAD_ARG;
    const int64_t al = 256;
    int64_t off = 0;
    const int64_t sizes[6] = {
        (int64_t)(T + frames) * B * F * ob,              // obs frames f32 | u8
        (int64_t)T * B * impala_beh_width(A, act_kind),  // beh_logits f32 (A | 2A per step)
        (int64_t)T * B * impala_act_width(A, act_kind),  // actions    i32 | f32 (A per step)
        (int64_t)T * B * 4,                              // rewards    f32
        (int64_t)T * B,                     // done       u8
        (int64_t)B * 4,                     // lens       i32
    };
    for (int i = 0; i < 6; ++i) {
        offsets[i] = off;
        off = impala_round_up(off + sizes[i], al);
    }
    *total_bytes = off;
    return IMPALA_OK;
}

extern "C" int impala_batch_layout_frames(int T, int B, int F, int frames, int A, int obs_dtype, int64_t offsets[6],
                                          int64_t* total_bytes) {
    return impala_batch_layout_act(T, B, F, frames, A, obs_dtype, IMPALA_ACT_CATEGORICAL, offsets, total_bytes);
}

extern "C" int impala_batch_layout_obs(int T, int B, int O, int A, int obs_dtype, int64_t offsets[6],
                                       int64_t* total_bytes) {
    return impala_batch_layout_frames(T, B, O, 1, A, obs_dtype, offsets, total_bytes);
}

extern "C" int impala_batch_layout(int T, int B, int O, int A, int64_t offsets[6],
                                   int64_t* total_bytes) {
    return impala_batch_layout_obs(T, B, O, A, IMPALA_OBS_F32, offsets, total_bytes);
}

extern "C" int impala_ingest(void* dev_slab, const void* host_slab, int64_t bytes, void* stream) {
    if (!dev_slab || !host_slab || bytes < 0) return IMPALA_ERR_BAD_ARG;
    cudaError_t e = cudaMemcpyAsync(dev_slab, host_slab, (size_t)bytes, cudaMemcpyHostToDevice,
                                    (cudaStream_t)stream);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

// Columns [b0, b0 + B_local) of a host batch slab laid out for B columns -> a device slab laid out
// for B_local columns: one strided 2-D copy per tensor (rows = time steps or frames), the lens vector 1-D.
extern "C" int impala_ingest_shard_act(void* dev_slab, const void* host_slab, int T, int B, int F, int frames, int A,
                                       int obs_dtype, int act_kind, int b0, int B_local, void* stream) {
    if (!dev_slab || !host_slab || b0 < 0 || B_local < 1 || b0 + B_local > B) return IMPALA_ERR_BAD_ARG;
    int64_t ho[6], doff[6], ht, dt;
    int rc = impala_batch_layout_act(T, B, F, frames, A, obs_dtype, act_kind, ho, &ht);
    if (rc != IMPALA_OK) return rc;
    if ((rc = impala_batch_layout_act(T, B_local, F, frames, A, obs_dtype, act_kind, doff, &dt)) != IMPALA_OK) return rc;
    const int64_t width[5] = {(int64_t)F * obs_bytes(obs_dtype), impala_beh_width(A, act_kind),
                              impala_act_width(A, act_kind), 4, 1};  // bytes per (row, column)
    const int rows[5] = {T + frames, T, T, T, T};
    const char* h = static_cast<const char*>(host_slab);
    char* d = static_cast<char*>(dev_slab);
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < 5; ++i) {
        cudaError_t e = cudaMemcpy2DAsync(d + doff[i], (size_t)B_local * width[i], h + ho[i] + (int64_t)b0 * width[i],
                                          (size_t)B * width[i], (size_t)B_local * width[i], (size_t)rows[i],
                                          cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return (int)e;
    }
    cudaError_t e = cudaMemcpyAsync(d + doff[5], h + ho[5] + (int64_t)b0 * 4, (size_t)B_local * 4, cudaMemcpyHostToDevice, st);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

extern "C" int impala_ingest_shard_frames(void* dev_slab, const void* host_slab, int T, int B, int F, int frames, int A,
                                          int obs_dtype, int b0, int B_local, void* stream) {
    return impala_ingest_shard_act(dev_slab, host_slab, T, B, F, frames, A, obs_dtype, IMPALA_ACT_CATEGORICAL, b0,
                                   B_local, stream);
}

extern "C" int impala_ingest_shard_obs(void* dev_slab, const void* host_slab, int T, int B, int O, int A,
                                       int obs_dtype, int b0, int B_local, void* stream) {
    return impala_ingest_shard_frames(dev_slab, host_slab, T, B, O, 1, A, obs_dtype, b0, B_local, stream);
}

extern "C" int impala_ingest_shard(void* dev_slab, const void* host_slab, int T, int B, int O, int A, int b0,
                                   int B_local, void* stream) {
    return impala_ingest_shard_obs(dev_slab, host_slab, T, B, O, A, IMPALA_OBS_F32, b0, B_local, stream);
}

// ---- node-local peer buffers (CUDA IPC) for impala_allreduce_clip_adam
extern "C" int impala_peer_alloc(int64_t bytes, void** dev_ptr, void* handle64) {
    if (bytes < 1 || !dev_ptr || !handle64) return IMPALA_ERR_BAD_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size is part of the ABI");
    cudaError_t e = cudaMalloc(dev_ptr, (size_t)bytes);
    if (e != cudaSuccess) return (int)e;
    if ((e = cudaMemset(*dev_ptr, 0, (size_t)bytes)) != cudaSuccess) return (int)e;
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return (int)e;
    e = cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64), *dev_ptr);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

extern "C" int impala_peer_open(const void* handle64, void** dev_ptr) {
    if (!handle64 || !dev_ptr) return IMPALA_ERR_BAD_ARG;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    cudaError_t e = cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

extern "C" int impala_peer_close(void* dev_ptr) {
    cudaError_t e = cudaIpcCloseMemHandle(dev_ptr);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

extern "C" int impala_peer_free(void* dev_ptr) {
    cudaError_t e = cudaFree(dev_ptr);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

// Debug only (not part of the public ABI): the pending error of this library's (statically linked)
// runtime instance, cleared by the call.
extern "C" int impala_debug_last_error(void) { return (int)cudaGetLastError(); }
