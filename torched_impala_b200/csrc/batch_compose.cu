// Experience replay: the fresh batches of the last updates stay in HBM (a store of Bf-column slabs); one
// launch per step gathers the B columns of the training slab out of it, column j from (slot, column) plan[j].
#include <algorithm>

#include "common.cuh"

namespace {

// One tensor of the batch layout as a [rows][columns][Wv vectors] array: source pitch Bf columns (in the
// store slab), destination pitch B columns (in the training slab).  The tensor's CTAs are
// [block0, block0 + nblocks) of the launch.
struct Seg {
    int64_t src_off, dst_off, rows;
    int Wv, vbytes;
    unsigned block0, nblocks;
};
struct ComposeArgs {
    Seg seg[6];
};

// dst vector i = (row B + j) Wv + v  <-  slab plan[j].x, vector (row Bf + plan[j].y) Wv + v; zero for a
// negative slot.  The destination is walked contiguously: the Wv lanes of one (row, column) read one
// contiguous source run, and for the 1- and 4-byte tensors (Wv = 1) consecutive lanes store consecutive
// columns.  (row, j, v) follow the grid stride as a mixed-radix counter, so no element pays a division.
template <typename Vec>
__device__ __forceinline__ void gather_columns(char* __restrict__ dst, const char* __restrict__ store,
                                               int64_t slab_bytes, const int2* __restrict__ plan, int B, int Bf,
                                               const Seg& sg) {
    const int Wv = sg.Wv;
    const int64_t row_vecs = (int64_t)B * Wv, stride = (int64_t)sg.nblocks * blockDim.x;
    const int64_t i0 = (int64_t)(blockIdx.x - sg.block0) * blockDim.x + threadIdx.x;
    int64_t row = i0 / row_vecs;
    const int c = (int)(i0 - row * row_vecs);
    int j = c / Wv, v = c - j * Wv;
    const int64_t dr = stride / row_vecs;
    const int dc = (int)(stride - dr * row_vecs), dj = dc / Wv, dv = dc - dj * Wv;
    Vec* __restrict__ out = reinterpret_cast<Vec*>(dst + sg.dst_off);
    for (int64_t i = i0; row < sg.rows; i += stride) {
        const int2 p = __ldg(plan + j);
        Vec val{};
        if (p.x >= 0)
            val = __ldg(reinterpret_cast<const Vec*>(store + p.x * slab_bytes + sg.src_off) + (row * Bf + p.y) * Wv + v);
        out[i] = val;
        v += dv, j += dj, row += dr;
        if (v >= Wv) v -= Wv, ++j;
        if (j >= B) j -= B, ++row;
    }
}

__global__ void __launch_bounds__(256) batch_compose_kernel(char* __restrict__ dst, const char* __restrict__ store,
                                                            int64_t slab_bytes, const int2* __restrict__ plan, int B,
                                                            int Bf, const ComposeArgs a) {
    Seg sg = a.seg[0];
#pragma unroll
    for (int s = 1; s < 6; ++s)
        if (blockIdx.x >= a.seg[s].block0) sg = a.seg[s];
    if (sg.vbytes == 16)
        gather_columns<uint4>(dst, store, slab_bytes, plan, B, Bf, sg);
    else if (sg.vbytes == 4)
        gather_columns<uint32_t>(dst, store, slab_bytes, plan, B, Bf, sg);
    else
        gather_columns<uint8_t>(dst, store, slab_bytes, plan, B, Bf, sg);
}

}  // namespace

extern "C" int impala_batch_compose_act(void* dst_slab, const void* store, int64_t store_slab_bytes,
                                        const int32_t* plan, int T, int B, int Bf, int F, int frames, int A,
                                        int obs_dtype, int act_kind, void* stream) {
    if (!dst_slab || !store || !plan || Bf <= 0 || Bf >= B) return IMPALA_ERR_BAD_ARG;
    int64_t so[6], dof[6], st_total, dt_total;
    int rc = impala_batch_layout_act(T, Bf, F, frames, A, obs_dtype, act_kind, so, &st_total);
    if (rc != IMPALA_OK) return rc;
    if ((rc = impala_batch_layout_act(T, B, F, frames, A, obs_dtype, act_kind, dof, &dt_total)) != IMPALA_OK) return rc;
    if (store_slab_bytes < st_total) return IMPALA_ERR_BAD_ARG;
    int sms = 0;
    if (const cudaError_t e = impala_sm_count(&sms); e != cudaSuccess) return (int)e;

    const int64_t width[6] = {(int64_t)F * (obs_dtype == IMPALA_OBS_U8 ? 1 : 4), impala_beh_width(A, act_kind),
                              impala_act_width(A, act_kind), 4, 1, 4};
    const int64_t rows[6] = {T + frames, T, T, T, T, 1};
    const uintptr_t ptrs = reinterpret_cast<uintptr_t>(dst_slab) | reinterpret_cast<uintptr_t>(store) |
                           (uintptr_t)store_slab_bytes;
    ComposeArgs a;
    unsigned grid = 0;
    for (int i = 0; i < 6; ++i) {
        // 16-byte vectors where the width and every address allow, 4-byte words next, bytes otherwise
        // (tensor offsets are multiples of 256)
        const int vb = (width[i] % 16 == 0 && (ptrs & 15) == 0) ? 16 : (width[i] % 4 == 0 && (ptrs & 3) == 0) ? 4 : 1;
        Seg& s = a.seg[i];
        s.src_off = so[i], s.dst_off = dof[i], s.rows = rows[i];
        s.Wv = (int)(width[i] / vb), s.vbytes = vb;
        const int64_t work = rows[i] * B * s.Wv;
        s.block0 = grid;
        s.nblocks = (unsigned)std::max<int64_t>(1, std::min<int64_t>((work + 255) / 256, (int64_t)sms * 16));
        grid += s.nblocks;
    }
    batch_compose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<char*>(dst_slab),
                                                                 static_cast<const char*>(store), store_slab_bytes,
                                                                 reinterpret_cast<const int2*>(plan), B, Bf, a);
    return impala_launch_status();
}

extern "C" int impala_batch_compose(void* dst_slab, const void* store, int64_t store_slab_bytes, const int32_t* plan,
                                    int T, int B, int Bf, int F, int frames, int A, int obs_dtype, void* stream) {
    return impala_batch_compose_act(dst_slab, store, store_slab_bytes, plan, T, B, Bf, F, frames, A, obs_dtype,
                                    IMPALA_ACT_CATEGORICAL, stream);
}
