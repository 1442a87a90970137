// csr_launch.cuh -- launching the persistent ring kernel (csr_kernels.cuh).  Shared by
// api_matrices.cu (plain operators), api_window.cu (windowed operators), api_offsets.cu
// (offset-indexed operators), api_patterns.cu (pattern-indexed operators) and api_col16.cu /
// api_col24.cu (narrow columns): the kernel instantiations of each storage format are compiled in
// a translation unit of their own so the build stays parallel.  Value-keyed pattern operators
// run csr_patval_kernel instead (no ring), launched from api_patvals.cu.
#pragma once
#include "internal.cuh"
#include "csr_kernels.cuh"

namespace b200 {

// dynamic shared memory a CTA may use when `ctas` of them share an SM: 228 KB per SM, 1 KB
// reserved per CTA, and the kernels' static scratch (reduction + exchange tickets, < 1.5 KB)
inline int ring_budget(int ctas) { return 228 * 1024 / ctas - 1024 - 1536; }

inline int value_table_bytes(int count) { return (count * (int)sizeof(double) + 15) & ~15; }

// Does the configured ring of an operator with `count` distinct values, indexed by `idx_bytes`-byte
// entries, keep all its stages beside the table of values?  (The index must never cost a stage.)
// fmt: the column format the launch streams (not FMT_WINDOW).
inline bool value_index_fits(b200_ctx_t ctx, int rows_cap, int nnz_cap, int fmt, int idx_bytes, int count) {
    const StageLayout lay = stage_layout(rows_cap, nnz_cap, idx_bytes, fmt);
    return fmt != FMT_WINDOW && ctx->opt_stages >= 1 &&
           kHeaderBytes + (int)ctx->opt_stages * lay.bytes + fmt_table_bytes(fmt, idx_bytes) + value_table_bytes(count) <=
               ring_budget((int)ctx->opt_ctas_per_sm);
}

// shared memory of one launch: header + ring of stages (+ the window / the offset table / the
// pattern tables, + an indexed operator's table of values); fewer stages if the configured ring
// does not fit beside opt_ctas_per_sm CTAs.  Returns 0 if a windowed launch does not fit even with
// one stage.
template <class P>
inline int ring_smem(b200_ctx_t ctx, b200_csr_t A, int fmt, int *stages_out) {
    const StageLayout lay = stage_layout(A->rows_cap, A->nnz_cap, (int)sizeof(typename P::TV), fmt, A->win_runs);
    const int extra = (fmt == FMT_WINDOW ? (int)(((size_t)A->win_slots * sizeof(typename P::TX) + 15) & ~(size_t)15)
                                         : fmt_table_bytes(fmt, (int)sizeof(typename P::TV))) +
                      (IndexedValues<typename P::TV>::value ? value_table_bytes(A->vtab_n) : 0);
    int stages = (int)ctx->opt_stages;
    const int per_cta_budget = ring_budget((int)ctx->opt_ctas_per_sm);
    while (stages > 1 && kHeaderBytes + stages * lay.bytes + extra > per_cta_budget) --stages;
    *stages_out = stages;
    const int smem = kHeaderBytes + stages * lay.bytes + extra;
    return (fmt == FMT_WINDOW && smem > per_cta_budget) ? 0 : smem;
}

template <int MODE, int L, bool HALO, class P, int FMT>
inline int launch_ring_impl(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    int stages = 1;
    const int smem = ring_smem<P>(ctx, A, FMT, &stages);
    static bool attr_set[64] = {};
    if (!attr_set[ctx->device & 63]) {
        // the opt-in limit covers static + dynamic shared memory (red_finish keeps a few
        // hundred bytes of static scratch)
        cudaFuncAttributes fa;
        B200_CUDA(cudaFuncGetAttributes(&fa, csr_ring_kernel<MODE, L, HALO, P, FMT>));
        B200_CUDA(cudaFuncSetAttribute(csr_ring_kernel<MODE, L, HALO, P, FMT>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       227 * 1024 - (int)fa.sharedSizeBytes));
        attr_set[ctx->device & 63] = true;
    }
    const int64_t cap = (int64_t)ctx->sm_count * ctx->opt_ctas_per_sm;
    const unsigned grid = (unsigned)std::min<int64_t>(A->nblocks, cap);
    B200_CUDA(launch_pdl(ctx, csr_ring_kernel<MODE, L, HALO, P, FMT>, dim3(grid), dim3(kThreads), (size_t)smem,
                         args, stages));
    return B200_OK;
}

// windowed operators (defined and instantiated in api_window.cu: 1..8 lanes per row)
template <int MODE, int L, bool HALO, class P>
int launch_ring_win(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);
// offset-indexed operators (defined and instantiated in api_offsets.cu: 1..4 lanes per row)
template <int MODE, int L, bool HALO, class P>
int launch_ring_off(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);
// pattern-indexed operators (defined and instantiated in api_patterns.cu: 1..4 lanes per row)
template <int MODE, int L, bool HALO, class P>
int launch_ring_pat(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);
// value-keyed patterns: csr_patval_kernel, no ring (api_patvals.cu: 1..4 lanes per row, single-GPU only)
template <int MODE, int L, class P>
int launch_patval(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);
// narrow columns (api_col16.cu / api_col24.cu: 1..8 lanes per row)
template <int MODE, int L, bool HALO, class P>
int launch_ring_c16(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);
template <int MODE, int L, bool HALO, class P>
int launch_ring_c24(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);

// the column format an operator is stored in (FMT_*)
inline int stored_format(b200_csr_t A) {
    if (A->pid) return A->pat_val ? FMT_PATVAL : FMT_PATTERN;
    if (A->idx8) return FMT_OFFSET;
    if (A->col16) return FMT_WINDOW;
    if (A->narrow) return A->narrow == 24 ? FMT_COL24 : FMT_COL16;
    return FMT_PLAIN;
}

// the table of values a value-keyed pattern operator keeps in the value type TV, or nullptr
template <class TV>
inline const TV *pattern_values(b200_csr_t A) {
    if constexpr (std::is_same<TV, double>::value) return A->pat_val;
    else if constexpr (std::is_same<TV, float>::value) return A->pat_val32;
    else return nullptr;
}

// which storage format does this launch stream?  (options may have changed since the upload)
template <class P>
inline int launch_format(b200_ctx_t ctx, b200_csr_t A) {
    if (ctx->opt_spmv_variant != 1) return FMT_PLAIN;
    if (A->pid && ctx->opt_patterns && A->lanes <= 4)
        return pattern_values<typename P::TV>(A) && ctx->opt_pattern_values ? FMT_PATVAL : FMT_PATTERN;
    if (A->idx8 && ctx->opt_offsets && A->lanes <= 4) return FMT_OFFSET;
    if (A->col16 && ctx->opt_window && A->lanes <= 8 && A->win_runs >= 1) {
        int stages;
        if (ring_smem<P>(ctx, A, FMT_WINDOW, &stages) != 0) return FMT_WINDOW;
    }
    if (A->narrow && ctx->opt_narrow && A->lanes <= 8) return A->narrow == 24 ? FMT_COL24 : FMT_COL16;
    return FMT_PLAIN;
}

} // namespace b200
