// api_col24.cu -- the narrow-column instantiations (24-bit) of the streaming CSR kernel
// (csr_kernels.cuh, FMT_COL24; format built by narrow.cuh at upload), compiled in a translation
// unit of their own.
#include "csr_launch.cuh"

namespace b200 {

template <int MODE, int L, bool HALO, class P>
int launch_ring_c24(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    return launch_ring_impl<MODE, L, HALO, P, FMT_COL24>(ctx, A, args);
}

// every (mode, precision) pair api_matrices.cu launches, for 1..8 lanes per row, with and
// without the multi-GPU halo
#define B200_C24_INST_L(MODE, L, P)                                                                  \
    template int launch_ring_c24<MODE, L, false, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);    \
    template int launch_ring_c24<MODE, L, true, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);
#define B200_C24_INST(MODE, P)                                                                       \
    B200_C24_INST_L(MODE, 1, P) B200_C24_INST_L(MODE, 2, P) B200_C24_INST_L(MODE, 4, P) B200_C24_INST_L(MODE, 8, P)

B200_C24_INST(MODE_SPMV, PrecDD)
B200_C24_INST(MODE_SPMV, PrecFF)
B200_C24_INST(MODE_SPMV, PrecFD)
B200_C24_INST(MODE_SPMV, PrecFFD)
B200_C24_INST(MODE_SPMV_ACC, PrecDD)
B200_C24_INST(MODE_SPMV_ACC, PrecFF)
B200_C24_INST(MODE_SPMV_ACC, PrecFD)
B200_C24_INST(MODE_SPMV_ACC, PrecFFD)
B200_C24_INST(MODE_RESID, PrecDD)
B200_C24_INST(MODE_RESID, PrecFF)
B200_C24_INST(MODE_RESID, PrecFD)
B200_C24_INST(MODE_RESID, PrecFDF)
B200_C24_INST(MODE_RESID_SCALED, PrecDD)
B200_C24_INST(MODE_RELAX, PrecDD)
B200_C24_INST(MODE_RELAX, PrecFF)
B200_C24_INST(MODE_RELAX, PrecFD)
B200_C24_INST(MODE_SPMV, PrecSD)
B200_C24_INST(MODE_SPMV_ACC, PrecSD)
B200_C24_INST(MODE_RESID, PrecSD)
B200_C24_INST(MODE_RESID_SCALED, PrecSD)
B200_C24_INST(MODE_RELAX, PrecSD)

// indexed values (PrecI8D / PrecI16D): single-GPU only, so without the halo
#define B200_C24_IDX_L(MODE, L, P)                                                                   \
    template int launch_ring_c24<MODE, L, false, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);
#define B200_C24_IDX(MODE, P) B200_C24_IDX_L(MODE, 1, P) B200_C24_IDX_L(MODE, 2, P) B200_C24_IDX_L(MODE, 4, P) B200_C24_IDX_L(MODE, 8, P)
#define B200_C24_IDX_P(P)                                                                             \
    B200_C24_IDX(MODE_SPMV, P) B200_C24_IDX(MODE_SPMV_ACC, P) B200_C24_IDX(MODE_RESID, P)                 \
    B200_C24_IDX(MODE_RESID_SCALED, P) B200_C24_IDX(MODE_RELAX, P)
B200_C24_IDX_P(PrecI8D)
B200_C24_IDX_P(PrecI16D)

} // namespace b200
