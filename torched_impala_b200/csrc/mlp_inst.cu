// Instantiations of the MLP kernels for one padded observation width (IMPALA_OP) and one
// direction (IMPALA_BWD).  Built once per (width, direction) by torched_impala_b200/build.py.
#include "mlp_kernels.cuh"

#ifndef IMPALA_OP
#error "compile with -DIMPALA_OP=<8|24|32|64|128> -DIMPALA_BWD=<0|1>"
#endif

#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)

#if IMPALA_BWD
#define KERNEL impala_mlp::mlp_bwd_kernel
#define ENTRY CAT(impala_mlp_bwd_op, IMPALA_OP)
#define KS_WIDE , (IMPALA_OP >= 64 ? 4 : 2)  // lanes per hidden unit of the wide shapes (mlp.cu pick_config)
#define KS_ONE , 1
#define IS_SPLIT (a.dout_b != nullptr)
#else
#define KERNEL impala_mlp::mlp_fwd_kernel
#define ENTRY CAT(impala_mlp_fwd_op, IMPALA_OP)
#define KS_WIDE
#define KS_ONE
#define IS_SPLIT (a.out_b != nullptr)
#endif

// The dense kernel, or with s (split heads, mlp_kernels.cuh split_out) its split-head twin; one output (NP = 1) has
// no twin.  The template arguments are complete up to KS, so the twin's SPLIT = true lands in its place.
#define TWIN(...)                                                                          \
    (s ? impala_mlp_launch(KERNEL<__VA_ARGS__, true>, a, c, smem, st, grid)                \
       : impala_mlp_launch(KERNEL<__VA_ARGS__>, static_cast<const MlpArgs&>(a), c, smem, st, grid))

#define BY_NP(JPT, MAXT)                                                                        \
    switch (c.np) {                                                                             \
        case 1: return impala_mlp_launch(KERNEL<JPT, IMPALA_OP, 1, MAXT>, da, c, smem, st, grid); \
        case 4: return TWIN(JPT, IMPALA_OP, 4, MAXT KS_ONE);                                    \
        default: return TWIN(JPT, IMPALA_OP, 16, MAXT KS_ONE);                                  \
    }

#define BY_NP_KS2(MAXT)                                                                        \
    switch (c.np) {                                                                            \
        case 1: return impala_mlp_launch(KERNEL<1, IMPALA_OP, 1, MAXT, 2>, da, c, smem, st, grid); \
        case 4: return TWIN(1, IMPALA_OP, 4, MAXT, 2);                                         \
        default: return TWIN(1, IMPALA_OP, 16, MAXT, 2);                                       \
    }

int ENTRY(const MlpSplitArgs& a, const MlpConfig& c, size_t smem, cudaStream_t st, int* grid) {
    const bool s = IS_SPLIT;
    const MlpArgs& da = a;
#if IMPALA_OP == 128
    // only shapes beyond the O <= 64 limit get here: one hidden unit per thread (per lane quad backward)
    switch (c.np) {
        case 1: return impala_mlp_launch(KERNEL<1, 128, 1, 256 KS_WIDE>, da, c, smem, st, grid);
        case 4: return TWIN(1, 128, 4, 256 KS_WIDE);
        case 16: return TWIN(1, 128, 16, 256 KS_WIDE);
        default: return TWIN(1, 128, 32, 256 KS_WIDE);
    }
#else
    // 17..32 outputs: one hidden unit per thread (per lane group backward)
    if (c.np == 32) return TWIN(1, IMPALA_OP, 32, 256 KS_WIDE);
#if IMPALA_BWD && IMPALA_OP == 64
    // wide observations: a lane pair per hidden unit (KS = 2), see mlp_kernels.cuh
    if (c.maxt == 128) { BY_NP_KS2(128) }
    BY_NP_KS2(256)
#else
    if (c.jpt == 1) { BY_NP(1, 128) }
    BY_NP(2, 256)
#endif
#endif
}
