// api_patvals.cu -- the value-keyed pattern instantiations of the streaming CSR kernel
// (csr_kernels.cuh, csr_patval_kernel; tables built by patterns.cuh at upload), compiled in a
// translation unit of their own.
#include "csr_launch.cuh"

namespace b200 {

template <int MODE, int L, class P>
int launch_patval(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    // the tables (<= 12.3 KB) are all the dynamic shared memory: within the default opt-in limit
    const int smem = fmt_table_bytes(FMT_PATVAL, (int)sizeof(typename P::TV));
    // the grid of the ring kernel on the same operator: the same rows per thread, the same bits
    const int64_t cap = (int64_t)ctx->sm_count * ctx->opt_ctas_per_sm;
    const unsigned grid = (unsigned)std::min<int64_t>(A->nblocks, cap);
    B200_CUDA(launch_pdl(ctx, csr_patval_kernel<MODE, L, P>, dim3(grid), dim3(kThreads), (size_t)smem, args));
    return B200_OK;
}

// every (mode, precision) pair api_patterns.cu instantiates except the indexed ones, for 1..4
// lanes per row; single-GPU only, so without the multi-GPU halo
#define B200_PV_INST(MODE, P)                                                                        \
    template int launch_patval<MODE, 1, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);             \
    template int launch_patval<MODE, 2, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);             \
    template int launch_patval<MODE, 4, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);

B200_PV_INST(MODE_SPMV, PrecDD)
B200_PV_INST(MODE_SPMV, PrecFF)
B200_PV_INST(MODE_SPMV, PrecFD)
B200_PV_INST(MODE_SPMV, PrecFFD)
B200_PV_INST(MODE_SPMV_ACC, PrecDD)
B200_PV_INST(MODE_SPMV_ACC, PrecFF)
B200_PV_INST(MODE_SPMV_ACC, PrecFD)
B200_PV_INST(MODE_SPMV_ACC, PrecFFD)
B200_PV_INST(MODE_RESID, PrecDD)
B200_PV_INST(MODE_RESID, PrecFF)
B200_PV_INST(MODE_RESID, PrecFD)
B200_PV_INST(MODE_RESID, PrecFDF)
B200_PV_INST(MODE_RESID_SCALED, PrecDD)
B200_PV_INST(MODE_RELAX, PrecDD)
B200_PV_INST(MODE_RELAX, PrecFF)
B200_PV_INST(MODE_RELAX, PrecFD)
B200_PV_INST(MODE_SPMV, PrecSD)
B200_PV_INST(MODE_SPMV_ACC, PrecSD)
B200_PV_INST(MODE_RESID, PrecSD)
B200_PV_INST(MODE_RESID_SCALED, PrecSD)
B200_PV_INST(MODE_RELAX, PrecSD)

} // namespace b200
