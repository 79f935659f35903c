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

extern "C" int impala_batch_layout(int T, int B, int O, int A, int64_t offsets[6],
                                   int64_t* total_bytes) {
    if (T < 1 || B < 1 || O < 1 || A < 1 || !offsets || !total_bytes) return IMPALA_ERR_BAD_ARG;
    const int64_t al = 256;
    int64_t off = 0;
    const int64_t sizes[6] = {
        (int64_t)(T + 1) * B * O * 4,  // obs        f32
        (int64_t)T * B * A * 4,        // beh_logits f32
        (int64_t)T * B * 4,            // actions    i32
        (int64_t)T * B * 4,            // rewards    f32
        (int64_t)T * B,                // done       u8
        (int64_t)B * 4,                // lens       i32
    };
    for (int i = 0; i < 6; ++i) {
        offsets[i] = off;
        off = impala_round_up(off + sizes[i], al);
    }
    *total_bytes = off;
    return IMPALA_OK;
}

extern "C" int impala_ingest(void* dev_slab, const void* host_slab, int64_t bytes, void* stream) {
    if (!dev_slab || !host_slab || bytes < 0) return IMPALA_ERR_BAD_ARG;
    cudaError_t e = cudaMemcpyAsync(dev_slab, host_slab, (size_t)bytes, cudaMemcpyHostToDevice,
                                    (cudaStream_t)stream);
    return e == cudaSuccess ? IMPALA_OK : (int)e;
}

// Columns [b0, b0 + B_local) of a host batch slab laid out for B columns -> a device slab laid out
// for B_local columns: one strided 2-D copy per tensor (rows = time steps), the lens vector 1-D.
extern "C" int impala_ingest_shard(void* dev_slab, const void* host_slab, int T, int B, int O, int A, int b0,
                                   int B_local, void* stream) {
    if (!dev_slab || !host_slab || b0 < 0 || B_local < 1 || b0 + B_local > B) return IMPALA_ERR_BAD_ARG;
    int64_t ho[6], doff[6], ht, dt;
    int rc = impala_batch_layout(T, B, O, A, ho, &ht);
    if (rc != IMPALA_OK) return rc;
    if ((rc = impala_batch_layout(T, B_local, O, A, doff, &dt)) != IMPALA_OK) return rc;
    const int64_t width[5] = {(int64_t)O * 4, (int64_t)A * 4, 4, 4, 1};  // bytes per (step, column)
    const int rows[5] = {T + 1, T, T, T, T};
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
