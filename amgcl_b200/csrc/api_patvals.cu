// api_patvals.cu -- the value-keyed pattern launches of the streaming CSR kernel (csr_kernels.cuh,
// csr_patval_kernel, FMT_PATVAL; tables built by patterns.cuh at upload).  A translation unit of
// its own: the units compile concurrently.
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

// every pass of csr_launch.cuh's table on 1..4 lanes per row; single-GPU only, so without the
// multi-GPU halo, and never over a value index (the tables hold the values themselves)
static_assert(fmt_max_lanes(FMT_PATVAL) == 4 && !fmt_halo(FMT_PATVAL) && !fmt_indexed(FMT_PATVAL),
              "the lanes, halo and indexed launches FMT_PATVAL is instantiated for");
#define B200_PATVAL_INST(L, MODE, P) template int launch_patval<MODE, L, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);
#define B200_PATVAL_PASS(MODE, P, MAXL) B200_LANES_##MAXL(B200_PATVAL_INST, MODE, P)
B200_CSR_PASSES(B200_PATVAL_PASS, 4)

} // namespace b200
