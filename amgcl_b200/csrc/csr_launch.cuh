// csr_launch.cuh -- launching the persistent ring kernel (csr_kernels.cuh), and the one table of
// the passes every column format is launched with.  api_matrices.cu launches the plain ring and
// dispatches the other formats (launch_csr_LH); each of those formats' kernels is instantiated in
// a translation unit of its own so the build stays parallel: api_window.cu, api_offsets.cu,
// api_patterns.cu, api_col16.cu, api_col24.cu (launch_ring), and api_patvals.cu for the
// value-keyed patterns' csr_patval_kernel (launch_patval, no ring).  The library is linked with
// --no-undefined, so a launch the dispatcher reaches but no unit instantiates fails the build.
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

// The (MODE, Prec) pairs of every pass over an operator, each format's launches instantiated for
// exactly these (X(MODE, P, ...) per pair) ...
#define B200_CSR_PASSES(X, ...)                                                                      \
    X(MODE_SPMV, PrecDD, __VA_ARGS__) X(MODE_SPMV, PrecFF, __VA_ARGS__) X(MODE_SPMV, PrecFD, __VA_ARGS__) \
    X(MODE_SPMV, PrecFFD, __VA_ARGS__) X(MODE_SPMV, PrecSD, __VA_ARGS__)                                \
    X(MODE_SPMV_ACC, PrecDD, __VA_ARGS__) X(MODE_SPMV_ACC, PrecFF, __VA_ARGS__)                         \
    X(MODE_SPMV_ACC, PrecFD, __VA_ARGS__) X(MODE_SPMV_ACC, PrecFFD, __VA_ARGS__)                        \
    X(MODE_SPMV_ACC, PrecSD, __VA_ARGS__)                                                              \
    X(MODE_RESID, PrecDD, __VA_ARGS__) X(MODE_RESID, PrecFF, __VA_ARGS__) X(MODE_RESID, PrecFD, __VA_ARGS__) \
    X(MODE_RESID, PrecFDF, __VA_ARGS__) X(MODE_RESID, PrecSD, __VA_ARGS__)                              \
    X(MODE_RESID_SCALED, PrecDD, __VA_ARGS__) X(MODE_RESID_SCALED, PrecSD, __VA_ARGS__)                 \
    X(MODE_RELAX, PrecDD, __VA_ARGS__) X(MODE_RELAX, PrecFF, __VA_ARGS__) X(MODE_RELAX, PrecFD, __VA_ARGS__) \
    X(MODE_RELAX, PrecSD, __VA_ARGS__)
// ... and the FP64 passes streaming an operator's value index (single-GPU only: never with the halo)
#define B200_CSR_INDEXED_PASSES(X, ...)                                                              \
    X(MODE_SPMV, PrecI8D, __VA_ARGS__) X(MODE_SPMV_ACC, PrecI8D, __VA_ARGS__) X(MODE_RESID, PrecI8D, __VA_ARGS__) \
    X(MODE_RESID_SCALED, PrecI8D, __VA_ARGS__) X(MODE_RELAX, PrecI8D, __VA_ARGS__)                      \
    X(MODE_SPMV, PrecI16D, __VA_ARGS__) X(MODE_SPMV_ACC, PrecI16D, __VA_ARGS__)                         \
    X(MODE_RESID, PrecI16D, __VA_ARGS__) X(MODE_RESID_SCALED, PrecI16D, __VA_ARGS__)                    \
    X(MODE_RELAX, PrecI16D, __VA_ARGS__)
// lanes per row: 1..4 or 1..8 (X(L, ...) per lane count)
#define B200_LANES_4(X, ...) X(1, __VA_ARGS__) X(2, __VA_ARGS__) X(4, __VA_ARGS__)
#define B200_LANES_8(X, ...) B200_LANES_4(X, __VA_ARGS__) X(8, __VA_ARGS__)
#define B200_IF_0(...)
#define B200_IF_1(...) __VA_ARGS__

// the most lanes per row an operator stored in a format is launched with (upload and dispatch)
constexpr int fmt_max_lanes(int fmt) {
    return fmt == FMT_PATTERN || fmt == FMT_OFFSET || fmt == FMT_PATVAL ? 4
         : fmt == FMT_WINDOW || fmt == FMT_COL16 || fmt == FMT_COL24   ? 8
                                                                       : 32;
}
// formats launched with the multi-GPU halo (value-keyed patterns are single-GPU only)
constexpr bool fmt_halo(int fmt) { return fmt != FMT_PATVAL; }
// formats launched over a value index (an indexed operator is never windowed; value-keyed patterns
// keep the values themselves)
constexpr bool fmt_indexed(int fmt) { return fmt != FMT_WINDOW && fmt != FMT_PATVAL; }
// is format FMT's launch on L lanes, with or without the halo, in precision P instantiated?
template <int FMT, int L, bool HALO, class P>
constexpr bool fmt_launches() {
    return L <= fmt_max_lanes(FMT) && (!HALO || fmt_halo(FMT)) &&
           (!IndexedValues<typename P::TV>::value || fmt_indexed(FMT));
}

// the ring launches of the formats other than FMT_PLAIN and FMT_PATVAL (B200_RING_UNIT)
template <int FMT, int MODE, int L, bool HALO, class P>
int launch_ring(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);
// value-keyed patterns: csr_patval_kernel, no ring (api_patvals.cu)
template <int MODE, int L, class P>
int launch_patval(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args);

// The body of one format's translation unit: defines launch_ring there only, out of
// api_matrices.cu's view so that it instantiates no format kernel itself, and instantiates it for
// every pass of the table on 1..MAXL lanes with and without the halo, plus, where IDX is 1, the
// indexed passes without it.
#define B200_RING_INST(L, FMT, MODE, P, HALO)                                                        \
    template int launch_ring<FMT, MODE, L, HALO, P>(b200_ctx_t, b200_csr_t, const CsrArgsT<P> &);
#define B200_RING_PASS(MODE, P, FMT, MAXL)                                                           \
    B200_LANES_##MAXL(B200_RING_INST, FMT, MODE, P, false) B200_LANES_##MAXL(B200_RING_INST, FMT, MODE, P, true)
#define B200_RING_INDEXED_PASS(MODE, P, FMT, MAXL) B200_LANES_##MAXL(B200_RING_INST, FMT, MODE, P, false)
#define B200_RING_UNIT(FMT, MAXL, IDX)                                                               \
    namespace b200 {                                                                                 \
    static_assert(fmt_max_lanes(FMT) == MAXL && fmt_halo(FMT) && fmt_indexed(FMT) == IDX,              \
                  "the lanes, halo and indexed launches " #FMT " is instantiated for");                \
    template <int F, int MODE, int L, bool HALO, class P>                                            \
    int launch_ring(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {                         \
        return launch_ring_impl<MODE, L, HALO, P, F>(ctx, A, args);                                  \
    }                                                                                                \
    B200_CSR_PASSES(B200_RING_PASS, FMT, MAXL)                                                       \
    B200_IF_##IDX(B200_CSR_INDEXED_PASSES(B200_RING_INDEXED_PASS, FMT, MAXL))                        \
    }

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
    if (A->pid && ctx->opt_patterns && A->lanes <= fmt_max_lanes(FMT_PATTERN))
        return pattern_values<typename P::TV>(A) && ctx->opt_pattern_values ? FMT_PATVAL : FMT_PATTERN;
    if (A->idx8 && ctx->opt_offsets && A->lanes <= fmt_max_lanes(FMT_OFFSET)) return FMT_OFFSET;
    if (A->col16 && ctx->opt_window && A->lanes <= fmt_max_lanes(FMT_WINDOW) && A->win_runs >= 1) {
        int stages;
        if (ring_smem<P>(ctx, A, FMT_WINDOW, &stages) != 0) return FMT_WINDOW;
    }
    if (A->narrow && ctx->opt_narrow && A->lanes <= fmt_max_lanes(A->narrow == 24 ? FMT_COL24 : FMT_COL16))
        return A->narrow == 24 ? FMT_COL24 : FMT_COL16;
    return FMT_PLAIN;
}

} // namespace b200
