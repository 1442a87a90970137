// api_matrices.cu -- CSR operators: row-block plan, upload, the streaming passes (spmv, residual, smoother sweep)
//
// Part of the implementation of the C ABI declared in include/amgcl_b200.h (host-side logic
// only: argument checking, bookkeeping, kernel launches; no CPU fallback anywhere).
#include "internal.cuh"
#include "csr_kernels.cuh"
#include "csr_launch.cuh"
#include "window.cuh"
#include "offsets.cuh"
#include "patterns.cuh"
#include "narrow.cuh"
#include "values.cuh"

namespace b200 {
int tail_enqueue_csr(b200_ctx_t ctx, int mode, b200_csr_t A, const CsrArgsT<PrecDD> &a);   // api_tail.cu
bool small_csr_accepts(b200_ctx_t ctx, b200_csr_t A);
int small_csr_launch(b200_ctx_t ctx, int mode, b200_csr_t A, const CsrArgsT<PrecDD> &a);
}

using namespace b200;

// ---------------------------------------------------------------------------
// matrices
// ---------------------------------------------------------------------------
namespace b200 {

static int choose_lanes(double avg) {
    // few lanes per row keep many rows -- and so many independent x-gathers -- in flight
    // per CTA; wide groups only pay off for long rows
    if (avg <= 12.0) return 1;
    if (avg <= 40.0) return 2;
    if (avg <= 64.0) return 4;
    if (avg <= 160.0) return 8;
    if (avg <= 320.0) return 16;
    return 32;
}

// Row-block plan (pure host logic, also exported as b200_plan_i64 for tests):
// consecutive rows, starting at a multiple of four, are packed greedily while
// they fit `rows_cap` rows and `nnz_cap` non-zeros.  A block that still exceeds
// nnz_cap (a single quad of very long rows) is counted as "long" and is handled
// by the strided path of the kernels.
struct RowBlockPlan {
    int lanes = 1, rows_cap = 256, nnz_cap = 2048;
    int64_t nlong = 0;
    std::vector<int2> blk;   // {first row, first non-zero}; last entry = {nrows, nnz}
};

template <class Ptr>
static void build_plan(int64_t nrows, const Ptr *ptr, int lanes_opt, int nnz_cap,
                       RowBlockPlan &plan) {
    const int64_t nnz = nrows ? (int64_t)ptr[nrows] : 0;
    const double avg = nrows ? (double)nnz / (double)nrows : 0.0;
    const int lanes = lanes_opt ? lanes_opt : choose_lanes(avg);
    const int groups = kThreads / lanes;
    // rows per block: a multiple of the number of row groups, sized so a typical
    // block fills the stage
    int k = 1;
    if (avg > 0.0) k = (int)std::floor((double)nnz_cap / (avg * groups));
    k = std::max(1, std::min(k, kRowsCapMax / groups));
    int rows_cap = std::min(kRowsCapMax, groups * k);
    rows_cap = std::max(4, rows_cap & ~3);
    plan.lanes = lanes; plan.rows_cap = rows_cap; plan.nnz_cap = nnz_cap; plan.nlong = 0;
    plan.blk.clear();
    plan.blk.reserve((size_t)(nnz / std::max(1, nnz_cap / 2) + nrows / rows_cap + 16));
    int64_t r = 0;
    while (r < nrows) {
        const int64_t r0 = r;
        const int64_t e0 = (int64_t)ptr[r0];
        // always take the first quad, then grow quad by quad while it fits
        int64_t r1 = std::min<int64_t>(nrows, r0 + 4);
        while (r1 < nrows) {
            const int64_t rn = std::min<int64_t>(nrows, r1 + 4);
            if (rn - r0 > rows_cap) break;
            if ((int64_t)ptr[rn] - e0 > nnz_cap) break;
            r1 = rn;
        }
        if ((int64_t)ptr[r1] - e0 > nnz_cap) ++plan.nlong;
        plan.blk.push_back(make_int2((int)r0, (int)e0));
        r = r1;
    }
    plan.blk.push_back(make_int2((int)nrows, (int)nnz));
}

// Shared validation of a host CSR matrix (both the single-GPU and the distributed path run it
// BEFORE anything reads through the arrays).
template <class Ptr, class Col>
static int csr_validate(int64_t nrows, int64_t ncols, const Ptr *ptr, const Col *col, bool have_val) {
    B200_REQUIRE(nrows >= 0 && ncols >= 0, "negative matrix dimension");
    B200_REQUIRE(ptr != nullptr, "null row pointer array");
    const int64_t imax = std::numeric_limits<int32_t>::max();
    if (nrows >= imax - 8 || ncols >= imax) return fail(B200_ERANGE, "matrix dimension exceeds int32");
    B200_REQUIRE(ptr[0] == 0, "ptr[0] must be 0");
    for (int64_t i = 1; i <= nrows; ++i)
        if ((int64_t)ptr[i] < (int64_t)ptr[i - 1]) return fail(B200_EINVAL, "row pointers not monotone");
    const int64_t nnz = (int64_t)ptr[nrows];
    if (nnz < 0) return fail(B200_EINVAL, "negative number of non-zeros");
    if (nnz >= imax - 8) return fail(B200_ERANGE, "number of non-zeros exceeds int32");
    B200_REQUIRE(nnz == 0 || (col != nullptr && have_val), "null col/val array");
    int bad = 0;
#pragma omp parallel for reduction(| : bad) schedule(static)
    for (int64_t e = 0; e < nnz; ++e) {
        const int64_t c = (int64_t)col[e];
        bad |= (c < 0 || c >= ncols) ? 1 : 0;
    }
    if (bad) return fail(B200_EINVAL, "column index out of range");
    return B200_OK;
}

// Host -> device copy of `count` elements through two pinned staging buffers of the context,
// converting Src -> Dst on the way (index narrowing).  The conversion runs on all host threads
// and overlaps the DMA of the previous chunk; a plain cudaMemcpy from pageable memory is staged
// by the driver on one thread at a fraction of the PCIe rate.
template <class Dst, class Src>
static cudaError_t staged_upload(b200_ctx_t ctx, Dst *dst, const Src *src, size_t count) {
    const size_t stage_bytes = (size_t)32 << 20;
    cudaError_t rc = cudaSuccess;
    for (int k = 0; k < 2 && rc == cudaSuccess; ++k) {
        if (!ctx->stage_host[k]) rc = cudaHostAlloc(&ctx->stage_host[k], stage_bytes, cudaHostAllocDefault);
        if (rc == cudaSuccess && !ctx->stage_event[k])
            rc = cudaEventCreateWithFlags(&ctx->stage_event[k], cudaEventDisableTiming);
    }
    if (rc != cudaSuccess) return rc;
    const size_t chunk = stage_bytes / sizeof(Dst);
    int k = 0;
    for (size_t off = 0; off < count && rc == cudaSuccess; off += chunk, k ^= 1) {
        const size_t m = std::min(chunk, count - off);
        rc = cudaEventSynchronize(ctx->stage_event[k]);        // the buffer's previous DMA is done
        if (rc != cudaSuccess) break;
        Dst *buf = static_cast<Dst *>(ctx->stage_host[k]);
        const Src *from = src + off;
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < (int64_t)m; ++i) buf[i] = (Dst)from[i];
        rc = cudaMemcpyAsync(dst + off, buf, m * sizeof(Dst), cudaMemcpyHostToDevice, ctx->stream);
        if (rc == cudaSuccess) rc = cudaEventRecord(ctx->stage_event[k], ctx->stream);
    }
    return rc;
}

// Do all n values keep their exact bits through double -> float -> double?  (Pure host logic, also
// exported as b200_values_fit_f32 for tests.)  Bits, not ==: -0.0 must stay -0.0, and a NaN
// qualifies only if its payload survives.  A float subnormal lost to rounding, a double subnormal
// or a value beyond FLT_MAX does not come back.
static bool values_fit_f32(const double *val, int64_t n) {
    int bad = 0;
#pragma omp parallel for reduction(| : bad) schedule(static)
    for (int64_t e = 0; e < n; ++e) {
        const double w = (double)(float)val[e];
        uint64_t a, b;
        memcpy(&a, val + e, 8);
        memcpy(&b, &w, 8);
        bad |= a != b ? 1 : 0;
    }
    return !bad;
}

// One device array of operator A: `bytes` allocated and recorded in A->arrays (csr_free frees it,
// A->bytes counts it), `count` elements of src uploaded into it as Dst, the rest (padding) zeroed.
template <class Dst, class T, class Src>
static cudaError_t csr_array(b200_csr_t A, T *&array, size_t bytes, const Src *src, size_t count) {
    void *p = nullptr;
    cudaError_t rc = cudaMalloc(&p, bytes);
    if (rc != cudaSuccess) return rc;
    A->arrays.emplace_back(p, bytes);
    array = static_cast<T *>(p);
    const size_t used = count * sizeof(Dst);
    if (bytes > used) rc = cudaMemsetAsync(static_cast<char *>(p) + used, 0, bytes - used, A->ctx->stream);
    if (rc == cudaSuccess && count) rc = staged_upload(A->ctx, static_cast<Dst *>(p), src, count);
    return rc;
}

static void csr_free(b200_csr_t A) {
    if (!A) return;
    for (const auto &a : A->arrays) cudaFree(a.first);
    if (A->send_idx) cudaFree(A->send_idx);
    if (A->halo_owned) cudaFree(A->halo_owned);
    if (A->ybuf) cudaFree(A->ybuf);
    if (A->scratch64) cudaFree(A->scratch64);
    if (A->pb_local) peer_release(A->ctx, A->pb_local, A->pb_peer);
    if (A->gb_local) peer_release(A->ctx, A->gb_local, A->gb_peer);
    delete A;
}

// Upload one CSR matrix exactly as the kernels will see it (indices narrowed to int32,
// row-block plan built).  Single-GPU matrices come straight through here; the
// distributed kinds hand in the local part produced by dist.cuh.
// halo_from >= 0: columns >= halo_from are owned by other ranks; the row blocks that gather
// them are marked and walked last, so the peers' pushes land while interior rows are computed.
template <class Ptr, class Col, class Val>
static int csr_upload(b200_ctx_t ctx, int64_t nrows, int64_t ncols, const Ptr *ptr,
                      const Col *col, const Val *val, b200_csr_t *out, int64_t halo_from = -1) {
    CHECK_CTX(ctx);
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    int vrc = csr_validate(nrows, ncols, ptr, col, val != nullptr);
    if (vrc) return vrc;
    const int64_t nnz = (int64_t)ptr[nrows];
    GUARD(ctx);

    // ---- narrow the row pointers (the plan needs them on the host) ---------------------
    std::vector<int32_t> hptr((size_t)nrows + 1);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i <= nrows; ++i) hptr[(size_t)i] = (int32_t)ptr[i];

    // ---- row-block plan -------------------------------------------------------
    RowBlockPlan plan;
    build_plan(nrows, hptr.data(), (int)ctx->opt_lanes, (int)ctx->opt_nnz_cap, plan);
    const int lanes = plan.lanes, rows_cap = plan.rows_cap, nnz_cap = plan.nnz_cap;
    const int64_t nlong = plan.nlong;
    std::vector<int2> &blk = plan.blk;
    int64_t nblocks = (int64_t)blk.size() - 1;

    // self-contained block descriptors in walk order
    std::vector<int4> blk4((size_t)nblocks + 1);
    if (halo_from >= 0 && nblocks > 0) {
        std::vector<char> outer((size_t)nblocks, 0);
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t b = 0; b < nblocks; ++b) {
            bool halo = false;
            for (int64_t e = blk[(size_t)b].y; e < blk[(size_t)b + 1].y && !halo; ++e)
                halo = (int64_t)col[e] >= halo_from;
            outer[(size_t)b] = halo;
        }
        size_t k = 0;
        for (int pass = 0; pass < 2; ++pass)
            for (int64_t b = 0; b < nblocks; ++b)
                if (outer[(size_t)b] == pass) {
                    const int2 lo = blk[(size_t)b], hi = blk[(size_t)b + 1];
                    blk4[k++] = make_int4(pass ? ~lo.x : lo.x, hi.x, lo.y, hi.y);
                }
    } else {
        for (int64_t b = 0; b < nblocks; ++b)
            blk4[(size_t)b] = make_int4(blk[(size_t)b].x, blk[(size_t)b + 1].x, blk[(size_t)b].y, blk[(size_t)b + 1].y);
    }
    blk4[(size_t)nblocks] = make_int4((int)nrows, (int)nrows, (int)nnz, (int)nnz);

    // ---- pattern-indexed rows, where the operator qualifies (patterns.cuh): keyed on the
    // entries' values as well where those patterns fit (single GPU), else on their offsets -----
    PatternPlan patp;
    const bool pattern_ok = ctx->opt_patterns && nnz >= ctx->opt_patterns_min_nnz && nlong == 0 &&
                            lanes <= fmt_max_lanes(FMT_PATTERN);
    const bool pattern_values = pattern_ok && ctx->opt_pattern_values && !ctx->dist &&
                                build_patterns(nrows, hptr.data(), col, patp, val);
    const bool pattern_indexed = pattern_values || (pattern_ok && build_patterns(nrows, hptr.data(), col, patp));
    // ... its table also in FP32: an FP32 operator's own values, an FP64 one's where all are exact
    const bool pattern_values32 = pattern_values &&
        (std::is_same<Val, float>::value ||
         (patp.val_f32 && ctx->opt_narrow_values && nnz >= ctx->opt_narrow_values_min_nnz));

    // ---- offset-indexed columns, where the operator qualifies (offsets.cuh) ------------------
    OffsetPlan offp;
    const bool offset_indexed = !pattern_indexed && ctx->opt_offsets && nnz >= ctx->opt_offsets_min_nnz && nlong == 0 &&
                                lanes <= fmt_max_lanes(FMT_OFFSET) &&
                                build_offsets(nrows, hptr.data(), col, offp);

    // ---- windowed format, where the operator qualifies (window.cuh) ------------------------
    WindowPlan win;
    bool windowed = false;
    if (!offset_indexed && ctx->opt_window && nnz >= ctx->opt_window_min_nnz && nlong == 0 && lanes <= fmt_max_lanes(FMT_WINDOW) &&
        ((ctx->opt_window_lanes >> (lanes == 1 ? 0 : lanes == 2 ? 1 : lanes == 4 ? 2 : 3)) & 1)) {
        // what the default launch configuration leaves for the window beside two stages
        const StageLayout wl = stage_layout(rows_cap, nnz_cap, (int)sizeof(Val), FMT_WINDOW, kWinRunCapMax);
        const int budget = ring_budget(4) - kHeaderBytes - 2 * wl.bytes;
        const int slot_cap = std::min(8192, (budget / 8) & ~3);
        windowed = build_windows(blk4.data(), nblocks, hptr.data(), col, ncols, nnz, slot_cap, kWinRunCapMax,
                                 (double)ctx->opt_window_ratio / 100.0, (int)ctx->opt_window_gap, win);
        if (windowed) {                   // (blocks whose window did not fit were cut)
            blk4.swap(win.blk4);
            nblocks = (int64_t)blk4.size() - 1;
        }
    }

    // ---- narrow columns for the operators no other format takes (narrow.cuh) -----------------
    NarrowPlan nar;
    const bool narrowed = !pattern_indexed && !offset_indexed && !windowed && ctx->opt_narrow && nlong == 0 &&
                          lanes <= fmt_max_lanes(FMT_COL16) && build_narrow(blk4.data(), nblocks, col, nnz, nar);

    // ---- FP32 copy of the values of an FP64 operator that loses nothing in FP32 ----------------
    // (not for value-keyed patterns: their passes stream no values)
    bool values32 = false;
    if constexpr (std::is_same<Val, double>::value)
        values32 = !pattern_values && ctx->opt_narrow_values && nnz >= ctx->opt_narrow_values_min_nnz &&
                   values_fit_f32(val, nnz);

    // ---- otherwise an index into the table of its distinct values (values.cuh), where the
    // table fits beside the configured ring of the format the operator is streamed in -----------
    ValueIndexPlan vip;
    bool indexed = false;
    if constexpr (std::is_same<Val, double>::value) {
        const int fmt = pattern_indexed ? FMT_PATTERN : offset_indexed ? FMT_OFFSET
                      : narrowed ? (nar.width == 24 ? FMT_COL24 : FMT_COL16) : FMT_PLAIN;
        indexed = !values32 && !pattern_values && ctx->opt_narrow_values && nnz > 0 &&
                  nnz >= ctx->opt_narrow_values_min_nnz &&
                  nlong == 0 && !windowed && !ctx->dist && build_value_index(val, nnz, vip) &&
                  value_index_fits(ctx, rows_cap, nnz_cap, fmt, vip.width / 8, vip.count);
    }

    // ---- block-relative row pointers of the final blocks --------------------------------
    std::vector<unsigned short> ptr16((size_t)nrows, 0);
    build_ptr16(blk4.data(), nblocks, hptr.data(), nnz_cap, ptr16);

    // ---- upload ---------------------------------------------------------------------
    b200_csr_s *A = new (std::nothrow) b200_csr_s();
    if (!A) return fail(B200_ENOMEM, "out of host memory");
    A->ctx = ctx; A->nrows = nrows; A->ncols = ncols; A->nnz = nnz;
    A->gl_rows = nrows; A->gl_cols = ncols; A->gl_nnz = nnz;
    A->dtype = std::is_same<Val, float>::value ? B200_F32 : B200_F64;
    A->lanes = lanes; A->rows_cap = rows_cap; A->nnz_cap = nnz_cap;
    A->nblocks = nblocks; A->nlong = nlong;
    {
        // blocks with fewer chunks of 32 / lanes rows than the CTA has warps (csr_ring_kernel)
        const int rw = 32 / lanes;
        int64_t few = 0;
        for (int64_t b = 0; b < nblocks; ++b) {
            const int4 q = blk4[(size_t)b];
            const int nr = q.y - (q.x < 0 ? ~q.x : q.x);
            if (q.w - q.z <= nnz_cap && (nr + rw - 1) / rw < kThreads / 32) ++few;
        }
        A->row_stream = 2 * few > nblocks;
    }
    // padding: bulk copies round sizes up to 16 bytes
    const size_t nn = (size_t)nnz, nr = (size_t)nrows, nb = (size_t)nblocks;
#define CSR_CUDA(call)                                                         \
    do {                                                                       \
        cudaError_t rc__ = (call);                                             \
        if (rc__ != cudaSuccess) {                                             \
            csr_free(A);                                                       \
            return cuda_fail(rc__, #call, __FILE__, __LINE__);                 \
        }                                                                      \
    } while (0)
    CSR_CUDA(csr_array<int>(A, A->ptr, (nr + 1 + 8) * sizeof(int), hptr.data(), nr + 1));
    CSR_CUDA(csr_array<int>(A, A->col, (nn + 8) * sizeof(int), col, nn));      // narrowed to int32 on the way
    CSR_CUDA(csr_array<Val>(A, A->val, (nn + 8) * sizeof(Val), val, nn));
    CSR_CUDA(csr_array<int4>(A, A->blk, (nb + 1) * sizeof(int4), blk4.data(), nb + 1));
    if (values32) CSR_CUDA(csr_array<float>(A, A->val32, (nn + 8) * sizeof(float), val, nn));   // exact: checked above
    if (indexed) {
        const size_t vix_bytes = ((nn + 32) * (size_t)(vip.width / 8) + 15) & ~(size_t)15;
        if (vip.width == 8) CSR_CUDA(csr_array<unsigned char>(A, A->vidx, vix_bytes, vip.idx8.data(), nn));
        else CSR_CUDA(csr_array<unsigned short>(A, A->vidx, vix_bytes, vip.idx16.data(), nn));
        CSR_CUDA(csr_array<uint64_t>(A, A->vtab, (size_t)vip.count * sizeof(double), vip.tab.data(), (size_t)vip.count));
        A->vidx_bytes = vip.width / 8;
        A->vtab_n = vip.count;
    }
    CSR_CUDA(csr_array<unsigned short>(A, A->ptr16, (nr + 16) * sizeof(unsigned short), ptr16.data(), nr));
    if (narrowed) {
        CSR_CUDA(csr_array<unsigned short>(A, A->clo16, (nn + 16) * sizeof(unsigned short), nar.lo16.data(), nn));
        CSR_CUDA(csr_array<int>(A, A->cbase, (nb + 1) * sizeof(int), nar.base.data(), nb));
        if (nar.width == 24)
            CSR_CUDA(csr_array<unsigned char>(A, A->chi8, (nn + 32 + 15) & ~(size_t)15, nar.hi8.data(), nn));
        A->narrow = nar.width;
    }
    if (windowed) {
        CSR_CUDA(csr_array<unsigned short>(A, A->col16, (nn + 16) * sizeof(unsigned short), win.col16.data(), nn));
        CSR_CUDA(csr_array<int2>(A, A->wrun, (win.runs.size() + 4) * sizeof(int2), win.runs.data(), win.runs.size()));
        CSR_CUDA(csr_array<int2>(A, A->wblk, (nb + 1) * sizeof(int2), win.wblk.data(), nb));
        A->win_slots = (win.max_slots + 3) & ~3;
        A->win_runs = win.max_runs;
        A->win_total = win.total_slots;
    }
    if (offset_indexed) {
        CSR_CUDA(csr_array<unsigned char>(A, A->idx8, (nn + 32 + 15) & ~(size_t)15, offp.idx8.data(), nn));
        CSR_CUDA(csr_array<int>(A, A->off_tab, kOffTabLen * sizeof(int), offp.tab, (size_t)kOffTabLen));
        A->off_count = offp.count;
    }
    if (pattern_indexed) {
        CSR_CUDA(csr_array<unsigned char>(A, A->pid, (nr + 32 + 15) & ~(size_t)15, patp.pid.data(), nr));
        CSR_CUDA(csr_array<unsigned short>(A, A->pat_start, (kPatCap + 1 + 7) * sizeof(unsigned short),
                                           patp.start.data(), (size_t)kPatCap + 1));
        CSR_CUDA(csr_array<int>(A, A->pat_off, kPatOffCap * sizeof(int), patp.off.data(), (size_t)kPatOffCap));
        A->pat_count = patp.count;
        A->pat_total = patp.total;
    }
    if (pattern_values)
        CSR_CUDA(csr_array<double>(A, A->pat_val, kPatOffCap * sizeof(double), patp.val.data(), (size_t)kPatOffCap));
    if (pattern_values32)
        CSR_CUDA(csr_array<float>(A, A->pat_val32, kPatOffCap * sizeof(float), patp.val32.data(), (size_t)kPatOffCap));
    CSR_CUDA(cudaStreamSynchronize(ctx->stream));   // host staging buffers die here
#undef CSR_CUDA
    for (const auto &a : A->arrays) A->bytes += a.second;
    if (nnz > ctx->big_nnz) {
        ctx->big_nnz = nnz;
        ctx->big_fmt = stored_format(A);
    }
    *out = A;
    return B200_OK;
}

// The public constructor.  On a distributed context (dist.cuh) the shape decides how the
// operator is shared out: a dimension >= the threshold belongs to a partitioned level, a smaller
// one to a replicated level; a rank always keeps whole rows.
template <class Ptr, class Col, class Val>
static int csr_create(b200_ctx_t ctx, int64_t nrows, int64_t ncols, const Ptr *ptr,
                      const Col *col, const Val *val, b200_csr_t *out) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "matrix creation");
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    if (!ctx->dist) return csr_upload(ctx, nrows, ncols, ptr, col, val, out);

    int rc = csr_validate(nrows, ncols, ptr, col, val != nullptr);
    if (rc) return rc;
    const int64_t nnz = (int64_t)ptr[nrows];
    const int64_t T = ctx->dist_min_rows;
    const bool rd = nrows >= T, cd = ncols >= T;
    if (!rd && !cd) return csr_upload(ctx, nrows, ncols, ptr, col, val, out);   // replicated level
    GUARD(ctx);

    // rows: the rank's block of a partitioned result, or its share of a replicated one
    const int P = ctx->nranks, rank = ctx->rank;
    const Partition rows(nrows, P), cols(ncols, P);
    SplitMatrix sp;
    split_rows(rows, cols, cd, rank, ptr, col, sp);

    b200_csr_t A = nullptr;
    rc = csr_upload(ctx, sp.nrows, sp.ncols, sp.ptr.data(), sp.col.data(), val + sp.val_offset, &A,
                    /* columns from here on live in the halo buffer */ cd ? sp.n_loc : (int64_t)-1);
    if (rc) return rc;
    A->kind = cd ? B200_CK_HALO : B200_CK_LOCAL;
    A->gl_rows = nrows; A->gl_cols = ncols; A->gl_nnz = nnz;
    A->rows_dist = rd; A->cols_dist = cd;
    A->gather_rows = !rd;
    A->row_off = rows.lo(rank); A->row_B = rows.B;
    A->n_loc = sp.n_loc;
#define DCSR_CUDA(call)                                                        \
    do {                                                                       \
        cudaError_t rc__ = (call);                                             \
        if (rc__ != cudaSuccess) {                                             \
            csr_free(A);                                                       \
            return cuda_fail(rc__, #call, __FILE__, __LINE__);                 \
        }                                                                      \
    } while (0)
    if (cd) {
        A->S = sp.S;
        A->n_send = (int64_t)sp.send_idx.size();
        std::vector<int32_t> idx(sp.send_idx.begin(), sp.send_idx.end());
        DCSR_CUDA(cudaMalloc(&A->send_idx, std::max<size_t>(1, idx.size()) * sizeof(int)));
        const size_t halo_n = std::max<size_t>(2, (size_t)(P * sp.S));
        DCSR_CUDA(cudaMalloc(&A->halo_owned, halo_n * sizeof(double)));
        A->halo = A->halo_owned;
        DCSR_CUDA(cudaMemsetAsync(A->halo, 0, halo_n * sizeof(double), ctx->stream));
        if (!idx.empty())
            DCSR_CUDA(cudaMemcpyAsync(A->send_idx, idx.data(), idx.size() * sizeof(int),
                                      cudaMemcpyHostToDevice, ctx->stream));
        A->bytes += idx.size() * sizeof(int) + (size_t)(P * sp.S) * sizeof(double);
        // who exchanges with whom: the symmetric closure of "rows of p reference columns of o"
        // (identical on every rank: derived from the global matrix).  A pair exchanges flags in
        // BOTH directions even if data flows one way only: that is what bounds how far one
        // rank can run ahead of another, i.e. what makes two parity buffers enough (peer.cuh).
        for (int q = 0; q < P; ++q)
            A->xchg[q] = q != rank && (sp.dep[(size_t)rank * P + q] || sp.dep[(size_t)q * P + rank]);
    }
    if (A->gather_rows && !ctx->p2p) {
        DCSR_CUDA(cudaMalloc((void **)&A->ybuf, ((size_t)P * (size_t)rows.B + 2) * sizeof(double)));
        DCSR_CUDA(cudaMemsetAsync(A->ybuf, 0, ((size_t)P * (size_t)rows.B + 2) * sizeof(double), ctx->stream));
        A->bytes += (size_t)P * (size_t)rows.B * sizeof(double);
    }
    DCSR_CUDA(cudaStreamSynchronize(ctx->stream));
#undef DCSR_CUDA
    if (ctx->p2p) {
        // collective allocations: every rank reaches them for every distributed operator
        if (cd) {
            size_t half = (size_t)P * (size_t)A->S * sizeof(double);
            half = (std::max<size_t>(half, 16) + 255) & ~size_t(255);
            A->pb_half = half;
            rc = peer_alloc(ctx, kFlagBytes + 2 * half, &A->pb_local, A->pb_peer);
            if (rc) {
                csr_free(A);
                return rc;
            }
            A->bytes += kFlagBytes + 2 * half;
        }
        if (A->gather_rows) {
            size_t half = (size_t)P * (size_t)rows.B * sizeof(double);
            half = (std::max<size_t>(half, 16) + 255) & ~size_t(255);
            A->gb_half = half;
            rc = peer_alloc(ctx, kFlagBytes + 2 * half, &A->gb_local, A->gb_peer);
            if (rc) {
                csr_free(A);
                return rc;
            }
            A->bytes += kFlagBytes + 2 * half;
        }
    }
    *out = A;
    return B200_OK;
}

// ---- launch one streaming pass over A ------------------------------------------------
// P = precision combination (csr_kernels.cuh).  Only FP64 carries the multi-GPU halo path
// and the one-block-per-CTA cross-check variant; the mixed-precision combinations use the
// persistent ring only.

// launch format FMT into rc if csr_launch.cuh's table instantiates that launch (else false)
template <int FMT, int MODE, int L, bool HALO, class P>
static bool launch_stored(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args, int &rc) {
    if constexpr (!fmt_launches<FMT, L, HALO, P>()) return false;
    else if constexpr (FMT == FMT_PATVAL) rc = launch_patval<MODE, L, P>(ctx, A, args);
    else rc = launch_ring<FMT, MODE, L, HALO, P>(ctx, A, args);
    return true;
}

template <int MODE, int L, bool HALO, class P>
static int launch_csr_LH(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    constexpr bool fp64 = std::is_same<P, PrecDD>::value;
    const StageLayout lay = stage_layout(A->rows_cap, A->nnz_cap, (int)sizeof(typename P::TV));
    if (fp64 && ctx->opt_spmv_variant == 0 && !HALO) {
        const int smem = kHeaderBytes + lay.bytes;
        static bool attr_set[64] = {};   // per instantiation and device
        if (!attr_set[ctx->device & 63]) {
            B200_CUDA(cudaFuncSetAttribute(csr_block_kernel<MODE, L, HALO, PrecDD>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            attr_set[ctx->device & 63] = true;
        }
        // (only reachable with P == PrecDD)
        csr_block_kernel<MODE, L, HALO, PrecDD><<<(unsigned)A->nblocks, kThreads, smem, ctx->stream>>>(
            *reinterpret_cast<const CsrArgsT<PrecDD> *>(&args));
    } else {
        int rc = B200_OK;
        bool done = false;
        switch (launch_format<P>(ctx, A)) {
        case FMT_PATVAL:  done = launch_stored<FMT_PATVAL, MODE, L, HALO, P>(ctx, A, args, rc); break;
        case FMT_PATTERN: done = launch_stored<FMT_PATTERN, MODE, L, HALO, P>(ctx, A, args, rc); break;
        case FMT_OFFSET:  done = launch_stored<FMT_OFFSET, MODE, L, HALO, P>(ctx, A, args, rc); break;
        case FMT_WINDOW:  done = launch_stored<FMT_WINDOW, MODE, L, HALO, P>(ctx, A, args, rc); break;
        case FMT_COL16:   done = launch_stored<FMT_COL16, MODE, L, HALO, P>(ctx, A, args, rc); break;
        case FMT_COL24:   done = launch_stored<FMT_COL24, MODE, L, HALO, P>(ctx, A, args, rc); break;
        }
        if (!done) rc = launch_ring_impl<MODE, L, HALO, P, FMT_PLAIN>(ctx, A, args);
        if (rc) return rc;
    }
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}

template <int MODE, int L, class P>
static int launch_csr_L(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    if constexpr (!IndexedValues<typename P::TV>::value) {   // (indexed: single-GPU contexts only)
        if (args.xh) return launch_csr_LH<MODE, L, true, P>(ctx, A, args);
    }
    return launch_csr_LH<MODE, L, false, P>(ctx, A, args);
}

template <int MODE, class P>
static int launch_csr_lanes(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    if (ctx->recording) A->in_graph = true;
    ProfScope prof(ctx, MODE, A->nrows, A->ncols, A->nnz, launch_format<P>(ctx, A), (int)sizeof(typename P::TV));
    switch (A->lanes) {
    case 1:  return launch_csr_L<MODE, 1>(ctx, A, args);
    case 2:  return launch_csr_L<MODE, 2>(ctx, A, args);
    case 4:  return launch_csr_L<MODE, 4>(ctx, A, args);
    case 8:  return launch_csr_L<MODE, 8>(ctx, A, args);
    case 16: return launch_csr_L<MODE, 16>(ctx, A, args);
    default: return launch_csr_L<MODE, 32>(ctx, A, args);
    }
}

// the arguments of an FP64 pass streaming `val` as the values of Q (the argument layouts differ
// only in the value type)
template <class Q>
static CsrArgsT<Q> retyped_args(const CsrArgsT<PrecDD> &args, const void *val) {
    CsrArgsT<Q> s;
    static_assert(sizeof(s) == sizeof(args), "arguments differ from PrecDD only in the value type");
    memcpy(&s, &args, sizeof(s));
    s.val = static_cast<const typename Q::TV *>(val);
    return s;
}

// ... streaming A's value index into its table of values
template <class PI>
static CsrArgsT<PI> indexed_args(b200_csr_t A, const CsrArgsT<PrecDD> &args) {
    CsrArgsT<PI> s = retyped_args<PI>(args, A->vidx);
    s.vtab = A->vtab;
    s.vtab_n = A->vtab_n;
    return s;
}

template <int MODE, class P>
static int launch_csr(b200_ctx_t ctx, b200_csr_t A, const CsrArgsT<P> &args) {
    if (A->nblocks == 0) return B200_OK;
    // small FP64 operator, nothing to reduce or exchange: defer into the coarse-tail list
    if (std::is_same<P, PrecDD>::value && !args.ndot && !args.xh && !args.gather_on &&
        tail_accepts_csr(ctx, A))
        return tail_enqueue_csr(ctx, MODE, A, *reinterpret_cast<const CsrArgsT<PrecDD> *>(&args));
    {
        const int trc = tail_flush(ctx);          // immediate launch: what was deferred goes first
        if (trc) return trc;
    }
    // a small FP64 operator: the direct-load kernel (same arithmetic) instead of the ring pipeline
    if (std::is_same<P, PrecDD>::value && MODE != MODE_RESID_SCALED && !args.ndot && !args.xh &&
        !args.gather_on && small_csr_accepts(ctx, A))
        return small_csr_launch(ctx, MODE, A, *reinterpret_cast<const CsrArgsT<PrecDD> *>(&args));
    if constexpr (std::is_same<P, PrecDD>::value) {
        // value-keyed patterns: the FP32 table where it is exact (same doubles once widened),
        // else the FP64 one; FMT_PATTERN streaming the FP64 values where the tables are not used
        if (A->pat_val32 && ctx->opt_narrow_values && launch_format<PrecSD>(ctx, A) == FMT_PATVAL) {
            CsrArgsT<PrecSD> s = retyped_args<PrecSD>(args, nullptr);   // (FMT_PATVAL streams no values)
            s.pat_val = A->pat_val32;
            return launch_csr_lanes<MODE>(ctx, A, s);
        }
        // the ring kernel streams the FP32 copy of an operator whose values are all exact FP32
        // (the cross-check variant, the tail and the small-operator kernel read the FP64 values)
        if (A->val32 && ctx->opt_narrow_values && ctx->opt_spmv_variant == 1)
            return launch_csr_lanes<MODE>(ctx, A, retyped_args<PrecSD>(args, A->val32));
        // ... or the 8- / 16-bit index of an operator with few distinct values, as long as the table
        // fits beside the configured ring (options may have changed since the upload)
        if (A->vidx && ctx->opt_narrow_values && ctx->opt_spmv_variant == 1 &&
            value_index_fits(ctx, A->rows_cap, A->nnz_cap, launch_format<PrecDD>(ctx, A), A->vidx_bytes, A->vtab_n)) {
            if (A->vidx_bytes == 1) return launch_csr_lanes<MODE>(ctx, A, indexed_args<PrecI8D>(A, args));
            return launch_csr_lanes<MODE>(ctx, A, indexed_args<PrecI16D>(A, args));
        }
    }
    return launch_csr_lanes<MODE>(ctx, A, args);
}

template <class P>
static CsrArgsT<P> base_args_t(b200_csr_t A) {
    CsrArgsT<P> a;
    memset(&a, 0, sizeof(a));
    a.ptr = A->ptr; a.ptr16 = A->ptr16; a.col = A->col; a.val = static_cast<const typename P::TV *>(A->val); a.blk = A->blk;
    a.nrows = (int)A->nrows; a.nblocks = (int)A->nblocks;
    a.rows_cap = A->rows_cap; a.nnz_cap = A->nnz_cap; a.row_stream = A->row_stream;
    a.col16 = A->col16; a.wrun = A->wrun; a.wblk = A->wblk; a.run_cap = A->win_runs;
    a.idx8 = A->idx8; a.off_tab = A->off_tab;
    a.pid = A->pid; a.pat_start = A->pat_start; a.pat_off = A->pat_off; a.pat_total = A->pat_total;
    a.pat_val = pattern_values<typename P::TV>(A);
    a.clo16 = A->clo16; a.chi8 = A->chi8; a.cbase = A->cbase;
    return a;
}
static CsrArgs base_args(b200_csr_t A) { return base_args_t<PrecDD>(A); }

// multi-GPU: make the boundary values of a.x visible and tell the kernel where they are
template <class P>
static int halo_into(b200_ctx_t ctx, b200_csr_t A, CsrArgsT<P> &a) {
    typedef typename P::TX TX;
    HaloArgs h;
    const int rc = halo_exchange(ctx, A, a.x, sizeof(TX), h);
    if (rc) return rc;
    a.xh = static_cast<const TX *>(h.xh); a.nloc = h.nloc;
    a.wait_flags = h.wait_flags; a.wait_mask = h.wait_mask; a.wait_seq = h.wait_seq;
    a.send_idx = h.send_idx; a.n_send = h.n_send; a.nranks = h.nranks;
    for (int q = 0; q < kMaxRanks; ++q) {
        a.push_data[q] = static_cast<TX *>(h.push_data[q]);
        a.push_flag[q] = h.push_flag[q];
    }
    a.push_ticket = h.push_ticket; a.push_seq = h.push_seq;
    return B200_OK;
}


} // namespace b200

extern "C" int b200_csr_create_i64(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                                   const int64_t *ptr, const int64_t *col, const double *val,
                                   b200_csr_t *A) {
    return csr_create(ctx, nrows, ncols, ptr, col, val, A);
}

extern "C" int b200_csr_create_i32(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                                   const int32_t *ptr, const int32_t *col, const double *val,
                                   b200_csr_t *A) {
    return csr_create(ctx, nrows, ncols, ptr, col, val, A);
}

extern "C" int b200_csr_create_i64_f32(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                                       const int64_t *ptr, const int64_t *col, const float *val,
                                       b200_csr_t *A) {
    return csr_create(ctx, nrows, ncols, ptr, col, val, A);
}

extern "C" int b200_csr_create_i32_f32(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                                       const int32_t *ptr, const int32_t *col, const float *val,
                                       b200_csr_t *A) {
    return csr_create(ctx, nrows, ncols, ptr, col, val, A);
}

extern "C" int b200_csr_dtype(b200_csr_t A, int *dtype) {
    B200_REQUIRE(A && dtype, "null argument");
    *dtype = A->dtype;
    return B200_OK;
}

extern "C" int b200_plan_i64(int64_t nrows, const int64_t *ptr, int lanes, int nnz_cap,
                             int32_t *blk_out, int64_t blk_capacity, int64_t *nblocks,
                             int *lanes_out, int *rows_cap_out, int64_t *nlong_out) {
    B200_REQUIRE(nrows >= 0 && ptr != nullptr && nblocks != nullptr, "bad argument");
    B200_REQUIRE(nnz_cap >= 256 && nnz_cap <= kNnzCapMax && nnz_cap % 8 == 0, "bad nnz_cap");
    B200_REQUIRE(lanes == 0 || (lanes >= 1 && lanes <= 32 && !(lanes & (lanes - 1))), "bad lanes");
    RowBlockPlan plan;
    build_plan(nrows, ptr, lanes, nnz_cap, plan);
    *nblocks = (int64_t)plan.blk.size() - 1;
    if (lanes_out) *lanes_out = plan.lanes;
    if (rows_cap_out) *rows_cap_out = plan.rows_cap;
    if (nlong_out) *nlong_out = plan.nlong;
    if (blk_out) {
        if ((int64_t)plan.blk.size() > blk_capacity)
            return fail(B200_EINVAL, "plan output buffer too small");
        for (size_t i = 0; i < plan.blk.size(); ++i) {
            blk_out[2 * i] = plan.blk[i].x;
            blk_out[2 * i + 1] = plan.blk[i].y;
        }
    }
    return B200_OK;
}

// The windowed format of a host matrix (window.cuh), for tests: the same plan + windows
// csr_upload builds, without a device.
extern "C" int b200_window_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                                    int lanes, int nnz_cap, int slot_cap, int max_ratio_percent, int gap,
                                    uint16_t *col16_out, int32_t *runs_out, int64_t runs_capacity,
                                    int32_t *blk_out, int64_t blk_capacity, int64_t *nblocks_out,
                                    int64_t *nruns_out, int *max_slots_out, int *max_runs_out, int *qualifies) {
    B200_REQUIRE(nrows >= 0 && ncols >= 0 && ptr && nblocks_out && nruns_out && qualifies, "bad argument");
    B200_REQUIRE(nnz_cap >= 256 && nnz_cap <= kNnzCapMax && nnz_cap % 8 == 0, "bad nnz_cap");
    B200_REQUIRE(lanes == 0 || (lanes >= 1 && lanes <= 32 && !(lanes & (lanes - 1))), "bad lanes");
    int rc = csr_validate(nrows, ncols, ptr, col, true);
    if (rc) return rc;
    RowBlockPlan plan;
    build_plan(nrows, ptr, lanes, nnz_cap, plan);
    int64_t nblocks = (int64_t)plan.blk.size() - 1;
    std::vector<int4> blk4((size_t)nblocks + 1);
    for (int64_t b = 0; b < nblocks; ++b)
        blk4[(size_t)b] = make_int4(plan.blk[(size_t)b].x, plan.blk[(size_t)b + 1].x, plan.blk[(size_t)b].y,
                                    plan.blk[(size_t)b + 1].y);
    const int64_t nnz = nrows ? ptr[nrows] : 0;
    blk4[(size_t)nblocks] = make_int4((int)nrows, (int)nrows, (int)nnz, (int)nnz);
    std::vector<int32_t> hptr((size_t)nrows + 1);
    for (int64_t i = 0; i <= nrows; ++i) hptr[(size_t)i] = (int32_t)ptr[i];
    WindowPlan w;
    const bool ok = plan.nlong == 0 && plan.lanes <= fmt_max_lanes(FMT_WINDOW) &&
                    build_windows(blk4.data(), nblocks, hptr.data(), col, ncols, nnz, slot_cap,
                                  kWinRunCapMax, max_ratio_percent / 100.0, gap, w);
    if (ok) {
        blk4.swap(w.blk4);
        nblocks = (int64_t)blk4.size() - 1;
    }
    *qualifies = ok ? 1 : 0;
    *nblocks_out = nblocks;
    *nruns_out = ok ? (int64_t)w.runs.size() : 0;
    if (max_slots_out) *max_slots_out = ok ? w.max_slots : 0;
    if (max_runs_out) *max_runs_out = ok ? w.max_runs : 0;
    if (!ok) return B200_OK;
    if (blk_out) {
        B200_REQUIRE(blk_capacity >= nblocks, "block output buffer too small");
        for (int64_t b = 0; b < nblocks; ++b) {
            blk_out[6 * b + 0] = blk4[(size_t)b].x; blk_out[6 * b + 1] = blk4[(size_t)b].y;
            blk_out[6 * b + 2] = blk4[(size_t)b].z; blk_out[6 * b + 3] = blk4[(size_t)b].w;
            blk_out[6 * b + 4] = w.wblk[(size_t)b].x; blk_out[6 * b + 5] = w.wblk[(size_t)b].y;
        }
    }
    if (runs_out) {
        B200_REQUIRE(runs_capacity >= (int64_t)w.runs.size(), "run output buffer too small");
        for (size_t i = 0; i < w.runs.size(); ++i) {
            runs_out[2 * i] = w.runs[i].x;
            runs_out[2 * i + 1] = w.runs[i].y;
        }
    }
    if (col16_out) std::copy(w.col16.begin(), w.col16.end(), col16_out);
    return B200_OK;
}

// The offset-indexed format of a host matrix (offsets.cuh), for tests.
extern "C" int b200_offset_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                                    uint8_t *idx8_out, int32_t *tab_out, int *count, int *qualifies) {
    B200_REQUIRE(nrows >= 0 && ncols >= 0 && ptr && qualifies, "bad argument");
    int rc = csr_validate(nrows, ncols, ptr, col, true);
    if (rc) return rc;
    std::vector<int32_t> hptr((size_t)nrows + 1);
    for (int64_t i = 0; i <= nrows; ++i) hptr[(size_t)i] = (int32_t)ptr[i];
    OffsetPlan o;
    const bool ok = build_offsets(nrows, hptr.data(), col, o);
    *qualifies = ok ? 1 : 0;
    if (count) *count = ok ? o.count : 0;
    if (!ok) return B200_OK;
    if (idx8_out) std::copy(o.idx8.begin(), o.idx8.end(), idx8_out);
    if (tab_out) std::copy(o.tab, o.tab + kOffTabLen, tab_out);
    return B200_OK;
}

// The pattern-indexed format of a host matrix (patterns.cuh), for tests.
extern "C" int b200_pattern_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                                     uint8_t *pid_out, uint16_t *start_out, int32_t *off_out, int *count,
                                     int *total, int *qualifies) {
    B200_REQUIRE(nrows >= 0 && ncols >= 0 && ptr && qualifies, "bad argument");
    int rc = csr_validate(nrows, ncols, ptr, col, true);
    if (rc) return rc;
    std::vector<int32_t> hptr((size_t)nrows + 1);
    for (int64_t i = 0; i <= nrows; ++i) hptr[(size_t)i] = (int32_t)ptr[i];
    PatternPlan o;
    const bool ok = build_patterns(nrows, hptr.data(), col, o);
    *qualifies = ok ? 1 : 0;
    if (count) *count = ok ? o.count : 0;
    if (total) *total = ok ? o.total : 0;
    if (!ok) return B200_OK;
    if (pid_out) std::copy(o.pid.begin(), o.pid.end(), pid_out);
    if (start_out) std::copy(o.start.begin(), o.start.end(), start_out);
    if (off_out) std::copy(o.off.begin(), o.off.end(), off_out);
    return B200_OK;
}

// The value-keyed pattern format of a host matrix (patterns.cuh), for tests.
extern "C" int b200_pattern_value_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                                           const double *val, uint8_t *pid_out, uint16_t *start_out,
                                           int32_t *off_out, double *val_out, int *count, int *total,
                                           int *exact_f32, int *qualifies) {
    B200_REQUIRE(nrows >= 0 && ncols >= 0 && ptr && qualifies, "bad argument");
    int rc = csr_validate(nrows, ncols, ptr, col, val != nullptr);
    if (rc) return rc;
    std::vector<int32_t> hptr((size_t)nrows + 1);
    for (int64_t i = 0; i <= nrows; ++i) hptr[(size_t)i] = (int32_t)ptr[i];
    PatternPlan o;
    const bool ok = build_patterns(nrows, hptr.data(), col, o, val);
    *qualifies = ok ? 1 : 0;
    if (count) *count = ok ? o.count : 0;
    if (total) *total = ok ? o.total : 0;
    if (exact_f32) *exact_f32 = ok && o.val_f32 ? 1 : 0;
    if (!ok) return B200_OK;
    if (pid_out) std::copy(o.pid.begin(), o.pid.end(), pid_out);
    if (start_out) std::copy(o.start.begin(), o.start.end(), start_out);
    if (off_out) std::copy(o.off.begin(), o.off.end(), off_out);
    if (val_out) memcpy(val_out, o.val.data(), (size_t)kPatOffCap * sizeof(double));
    return B200_OK;
}

// The narrow column format of a host matrix (narrow.cuh), for tests: the same plan csr_upload
// builds, without a device.  width_out: 16, 24, or 0 when the operator stays plain (a column span
// beyond 24 bits or a long block); ptr16_out: the block-relative row pointers of that plan.
extern "C" int b200_narrow_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                                    int lanes, int nnz_cap, int32_t *base_out, int64_t base_capacity,
                                    uint16_t *lo16_out, uint8_t *hi8_out, uint16_t *ptr16_out,
                                    int64_t *nblocks_out, int *width_out) {
    B200_REQUIRE(nrows >= 0 && ncols >= 0 && ptr && nblocks_out && width_out, "bad argument");
    B200_REQUIRE(nnz_cap >= 256 && nnz_cap <= kNnzCapMax && nnz_cap % 8 == 0, "bad nnz_cap");
    B200_REQUIRE(lanes == 0 || (lanes >= 1 && lanes <= 32 && !(lanes & (lanes - 1))), "bad lanes");
    int rc = csr_validate(nrows, ncols, ptr, col, true);
    if (rc) return rc;
    RowBlockPlan plan;
    build_plan(nrows, ptr, lanes, nnz_cap, plan);
    const int64_t nblocks = (int64_t)plan.blk.size() - 1;
    std::vector<int4> blk4((size_t)nblocks + 1);
    for (int64_t b = 0; b < nblocks; ++b)
        blk4[(size_t)b] = make_int4(plan.blk[(size_t)b].x, plan.blk[(size_t)b + 1].x, plan.blk[(size_t)b].y,
                                    plan.blk[(size_t)b + 1].y);
    const int64_t nnz = nrows ? ptr[nrows] : 0;
    std::vector<int32_t> hptr((size_t)nrows + 1);
    for (int64_t i = 0; i <= nrows; ++i) hptr[(size_t)i] = (int32_t)ptr[i];
    *nblocks_out = nblocks;
    if (ptr16_out) {
        std::vector<unsigned short> p16((size_t)nrows, 0);
        build_ptr16(blk4.data(), nblocks, hptr.data(), nnz_cap, p16);
        std::copy(p16.begin(), p16.end(), ptr16_out);
    }
    NarrowPlan o;
    const bool ok = plan.nlong == 0 && plan.lanes <= fmt_max_lanes(FMT_COL16) && build_narrow(blk4.data(), nblocks, col, nnz, o);
    *width_out = ok ? o.width : 0;
    if (!ok) return B200_OK;
    if (base_out) {
        B200_REQUIRE(base_capacity >= nblocks, "block output buffer too small");
        std::copy(o.base.begin(), o.base.end(), base_out);
    }
    if (lo16_out) std::copy(o.lo16.begin(), o.lo16.end(), lo16_out);
    if (hi8_out && o.width == 24) std::copy(o.hi8.begin(), o.hi8.end(), hi8_out);
    return B200_OK;
}

extern "C" int b200_ctx_largest_operator(b200_ctx_t ctx, int64_t *nnz, int *format) {
    CHECK_CTX(ctx);
    if (nnz) *nnz = ctx->big_nnz;
    if (format) *format = ctx->big_fmt;
    return B200_OK;
}

extern "C" int b200_csr_patterns(b200_csr_t A, int *pattern_indexed, int *count, int *total) {
    B200_REQUIRE(A, "null argument");
    if (pattern_indexed) *pattern_indexed = A->pid ? 1 : 0;
    if (count) *count = A->pat_count;
    if (total) *total = A->pat_total;
    return B200_OK;
}

extern "C" int b200_csr_offsets(b200_csr_t A, int *offset_indexed, int *count) {
    B200_REQUIRE(A, "null argument");
    if (offset_indexed) *offset_indexed = A->idx8 ? 1 : 0;
    if (count) *count = A->off_count;
    return B200_OK;
}

extern "C" int b200_csr_narrow(b200_csr_t A, int *width) {
    B200_REQUIRE(A && width, "null argument");
    *width = A->narrow;
    return B200_OK;
}

extern "C" int b200_csr_value_bytes(b200_csr_t A, int *bytes) {
    B200_REQUIRE(A && bytes, "null argument");
    *bytes = A->val32 || A->pat_val32 || A->dtype == B200_F32 ? 4 : A->vidx ? A->vidx_bytes : 8;
    return B200_OK;
}

extern "C" int b200_value_index_plan_i64(const double *val, int64_t n, double *table_out, int64_t table_capacity,
                                         void *idx_out, int *count_out, int *width_out) {
    B200_REQUIRE(n >= 0 && (val || n == 0) && count_out && width_out, "bad argument");
    ValueIndexPlan p;
    const bool ok = build_value_index(val, n, p);
    *count_out = p.count;
    *width_out = ok ? p.width : 0;
    if (!ok) return B200_OK;
    if (table_out) {
        B200_REQUIRE(table_capacity >= p.count, "table_out too small");
        memcpy(table_out, p.tab.data(), (size_t)p.count * sizeof(double));
    }
    if (idx_out && n) {
        if (p.width == 8) memcpy(idx_out, p.idx8.data(), (size_t)n);
        else memcpy(idx_out, p.idx16.data(), (size_t)n * 2);
    }
    return B200_OK;
}

extern "C" int b200_values_fit_f32(const double *val, int64_t n, int *qualifies) {
    B200_REQUIRE(n >= 0 && (val || n == 0) && qualifies, "bad argument");
    *qualifies = values_fit_f32(val, n) ? 1 : 0;
    return B200_OK;
}

extern "C" int b200_csr_window(b200_csr_t A, int *windowed, int *max_slots, int *max_runs, int64_t *total_slots) {
    B200_REQUIRE(A, "null argument");
    if (windowed) *windowed = A->col16 ? 1 : 0;
    if (max_slots) *max_slots = A->win_slots;
    if (max_runs) *max_runs = A->win_runs;
    if (total_slots) *total_slots = A->win_total;
    return B200_OK;
}

extern "C" int b200_csr_destroy(b200_csr_t A) {
    if (!A) return B200_OK;
    NOT_RECORDING(A->ctx, "matrix destruction");
    if (A->in_graph) A->ctx->destroy_epoch++;
    GUARD(A->ctx);
    csr_free(A);
    return B200_OK;
}

extern "C" int b200_csr_rows(b200_csr_t A, size_t *n) {
    B200_REQUIRE(A && n, "null argument");
    *n = (size_t)A->gl_rows;
    return B200_OK;
}
extern "C" int b200_csr_cols(b200_csr_t A, size_t *n) {
    B200_REQUIRE(A && n, "null argument");
    *n = (size_t)A->gl_cols;
    return B200_OK;
}
extern "C" int b200_csr_nonzeros(b200_csr_t A, size_t *n) {
    B200_REQUIRE(A && n, "null argument");
    *n = (size_t)A->gl_nnz;
    return B200_OK;
}
extern "C" int b200_csr_bytes(b200_csr_t A, size_t *bytes) {
    B200_REQUIRE(A && bytes, "null argument");
    *bytes = A->bytes;
    return B200_OK;
}
extern "C" int b200_csr_plan(b200_csr_t A, int *lanes_per_row, int64_t *n_blocks,
                             int64_t *n_long_blocks) {
    B200_REQUIRE(A, "null argument");
    if (lanes_per_row) *lanes_per_row = A->lanes;
    if (n_blocks) *n_blocks = A->nblocks;
    if (n_long_blocks) *n_long_blocks = A->nlong;
    return B200_OK;
}

// ---------------------------------------------------------------------------
// primitives
// ---------------------------------------------------------------------------
namespace b200 {

// what a caller wants reduced while the rows are in registers (reduce.cuh); slots == nullptr: nothing
struct DotReq {
    int           ndot  = 0;
    const double *w     = nullptr;     // second operand of the first product (nullptr: see CsrArgsT)
    const int    *slots = nullptr;
    unsigned      host_mask = 0;       // scalars the host will read right after a synchronize
    bool          done  = false;       // set when the launch produced the scalars
};
template <class P>
static void apply_req(b200_ctx_t ctx, b200_csr_t A, CsrArgsT<P> &a, DotReq *req) {
    if (!req || !req->ndot || ctx->opt_spmv_variant != 1 || a.nblocks == 0) return;
    if (!std::is_same<typename P::TY, double>::value) return;
    // partitioned result: every rank launches, the finishing CTAs all-reduce over the peers
    const bool across = A->rows_dist;
    if (across && !ctx->scal_x_table) return;       // NCCL transport: separate reduction instead
    a.ndot = req->ndot;
    a.w = req->w;
    red_out(ctx, req->ndot, req->slots, a.red, across, req->host_mask);
    req->done = true;
}

// y = alpha*A*x + beta*y for one precision combination, single- or multi-GPU
template <class P>
static int spmv_typed(b200_ctx_t ctx, double alpha, b200_csr_t A, b200_vec_t x, double beta,
                      b200_vec_t y, DotReq *req = nullptr) {
    typedef typename P::TX TX;
    typedef typename P::TY TY;
    CsrArgsT<P> a = base_args_t<P>(A);
    const double *px;
    int rc = rd(x, &px);
    if (rc) return rc;
    a.x = tp<TX>(px);
    a.alpha = alpha; a.beta = beta;
    // distributed context: x / y are blocks of partitioned vectors or whole replicated ones
    if (ctx->dist) {
        B200_REQUIRE((x->kind == B200_VK_DIST) == A->cols_dist && (y->kind == B200_VK_DIST) == A->rows_dist,
                     "spmv: vectors are not laid out like the operator (partitioned vs replicated)");
    }
    if (A->kind == B200_CK_HALO) {
        rc = halo_into(ctx, A, a);
        if (rc) return rc;
    }
    if (A->gather_rows) {
        // y is replicated, x partitioned: this rank computes its share of the rows, the shares
        // are all-gathered (R onto a small level)
        B200_REQUIRE(beta == 0.0 || y->zero_pending, "spmv onto a replicated level needs beta == 0");
        GatherArgs g;
        rc = gather_begin(ctx, A, sizeof(TY), g);
        if (rc) return rc;
        a.gather_on = g.on; a.nranks = ctx->nranks;
        for (int q = 0; q < kMaxRanks; ++q) {
            a.gather_data[q] = static_cast<TY *>(g.data[q]);
            a.gather_flag[q] = g.flag[q];
        }
        a.gather_ticket = g.ticket; a.gather_seq = g.seq;
        a.y = static_cast<TY *>(g.y_local);
        rc = launch_csr<MODE_SPMV>(ctx, A, a);
        if (rc) return rc;
        return gather_end(ctx, A, g, y);
    }
    apply_req(ctx, A, a, req);
    if (beta == 0.0 || y->zero_pending) {
        a.y = tp<TY>(wr(y));
        return launch_csr<MODE_SPMV>(ctx, A, a);
    }
    a.y = tp<TY>(mut(y));
    return launch_csr<MODE_SPMV_ACC>(ctx, A, a);
}

template <class P>
static int residual_typed(b200_ctx_t ctx, b200_vec_t f, b200_csr_t A, b200_vec_t x, b200_vec_t r,
                          DotReq *req = nullptr) {
    CsrArgsT<P> a = base_args_t<P>(A);
    const double *px, *pf;
    int rc = rd(x, &px);
    if (rc) return rc;
    rc = rd(f, &pf);
    if (rc) return rc;
    a.x = tp<typename P::TX>(px);
    a.f = tp<typename P::TF>(pf);
    if (A->kind == B200_CK_HALO) {
        B200_REQUIRE(x->kind == B200_VK_DIST && f->kind == B200_VK_DIST && r->kind == B200_VK_DIST,
                     "residual: vectors must be partitioned like the operator");
        rc = halo_into(ctx, A, a);
        if (rc) return rc;
    }
    a.y = tp<typename P::TY>((f == r) ? mut(r) : wr(r));   // r == f is fine: each row reads f[r] before writing
    apply_req(ctx, A, a, req);
    return launch_csr<MODE_RESID>(ctx, A, a);
}


} // namespace b200

namespace b200 {
static bool first_sweep_fusable(b200_ctx_t ctx, b200_csr_t A);      // (smoother section below)

static int spmv_impl(b200_ctx_t ctx, double alpha, b200_csr_t A, b200_vec_t x, double beta,
                     b200_vec_t y, DotReq *req) {
    CHECK_CTX(ctx);
    B200_REQUIRE(A && x && y, "null argument");
    touch(ctx, {x, y});
    B200_REQUIRE((int64_t)x->n == A->gl_cols, "spmv: x size != matrix columns");
    B200_REQUIRE((int64_t)y->n == A->gl_rows, "spmv: y size != matrix rows");
    B200_REQUIRE(x != y && (x->ptr != y->ptr || !x->ptr), "spmv: x and y must not alias");
    GUARD_DEFER(ctx);
    TailHold hold(ctx, {x, y});
    if (A->dtype == B200_F32) {
        // FP32 operator (mixed-precision hierarchy)
        if (all32({x, y})) return spmv_typed<PrecFF>(ctx, alpha, A, x, beta, y);
        if (all64({x, y})) return spmv_typed<PrecFD>(ctx, alpha, A, x, beta, y, req);
        if (x->dtype == B200_F32 && y->dtype == B200_F64)
            return spmv_typed<PrecFFD>(ctx, alpha, A, x, beta, y);
        return B200_BAD_MIX("spmv");
    }
    if (!all64({x, y})) return B200_BAD_MIX("spmv");
    return spmv_typed<PrecDD>(ctx, alpha, A, x, beta, y, req);
}

static int residual_impl(b200_ctx_t ctx, b200_vec_t f, b200_csr_t A, b200_vec_t x, b200_vec_t r,
                         DotReq *req) {
    CHECK_CTX(ctx);
    B200_REQUIRE(f && A && x && r, "null argument");
    touch(ctx, {f, x, r});
    B200_REQUIRE((int64_t)x->n == A->gl_cols, "residual: x size != matrix columns");
    B200_REQUIRE((int64_t)f->n == A->gl_rows && (int64_t)r->n == A->gl_rows,
                 "residual: rhs/r size != matrix rows");
    B200_REQUIRE(x != r && (x->ptr != r->ptr || !x->ptr), "residual: x and r must not alias");
    B200_REQUIRE(!A->gather_rows && (!ctx->dist || A->gl_rows == A->gl_cols || A->kind == B200_CK_LOCAL),
                 "residual: operator must be square");
    GUARD_RAW(ctx);
    TailHold hold(ctx, {f, x, r});
    if (ctx->lazy_vec) {
        // x = (omega*d).*f is still pending (b200_relax from x = 0 was the previous call): if
        // this is the residual of that very system, one pass forms x on the fly, writes it, and
        // writes r = f - A x (MODE_RESID_SCALED)
        if (ctx->lazy_vec == x && x->sc_fvec == f && f != r && x != r && r->ptr != x->ptr &&
            r->ptr != f->ptr && first_sweep_fusable(ctx, A) && all64({f, x, r}) && (!req || !req->ndot) &&
            r->owned && !r->escaped && f->ptr == x->sc_f && !f->zero_pending) {
            ctx->lazy_vec = nullptr;
            x->scale_pending = false;
            CsrArgs a = base_args(A);
            a.x = x->ptr;                         // (not gathered from: see gather_m)
            a.xw = x->ptr;
            a.f = x->sc_f; a.d = x->sc_d; a.alpha = x->sc_omega;
            x->sc_d = x->sc_f = nullptr; x->sc_fvec = nullptr;
            a.y = wr(r);
            ctx->fused_first_sweeps++;
            return launch_csr<MODE_RESID_SCALED>(ctx, A, a);
        }
        const int lrc = lazy_flush(ctx);
        if (lrc) return lrc;
    }
    if (A->dtype == B200_F32) {
        if (all32({f, x, r})) return residual_typed<PrecFF>(ctx, f, A, x, r);
        if (all64({f, x, r})) return residual_typed<PrecFD>(ctx, f, A, x, r, req);
        if (all64({f, x}) && r->dtype == B200_F32) return residual_typed<PrecFDF>(ctx, f, A, x, r);
        return B200_BAD_MIX("residual");
    }
    if (!all64({f, x, r})) return B200_BAD_MIX("residual");
    return residual_typed<PrecDD>(ctx, f, A, x, r, req);
}

// y = A x (alpha = 1, beta = 0) leaving <y, w> (and <y, y> when ndot == 2) in the table slots;
// falls back to a separate reduction launch where the streaming kernel cannot produce them.
int spmv_with_dots(b200_ctx_t ctx, b200_csr_t A, b200_vec_t x, b200_vec_t y, b200_vec_t w, int ndot,
                   const int *slots) {
    DotReq req;
    req.ndot = ndot; req.slots = slots;
    const double *pw = nullptr;
    if (w != y) {
        int rc = rd(w, &pw);
        if (rc) return rc;
    }
    req.w = pw;
    int rc = spmv_impl(ctx, 1.0, A, x, 0.0, y, &req);
    if (rc || req.done) return rc;
    return launch_dot_slots(ctx, y, w, ndot == 2 ? y : nullptr, slots);
}

// r = f - A x leaving <r, r> in the table slot
int residual_with_norm(b200_ctx_t ctx, b200_vec_t f, b200_csr_t A, b200_vec_t x, b200_vec_t r, int slot) {
    DotReq req;
    req.ndot = 1; req.slots = &slot; req.host_mask = 1u;
    int rc = residual_impl(ctx, f, A, x, r, &req);
    if (rc || req.done) return rc;
    return launch_dot_slots(ctx, r, r, nullptr, &slot, 1u);
}
} // namespace b200

extern "C" int b200_spmv(b200_ctx_t ctx, double alpha, b200_csr_t A, b200_vec_t x, double beta,
                         b200_vec_t y) {
    return spmv_impl(ctx, alpha, A, x, beta, y, nullptr);
}

extern "C" int b200_residual(b200_ctx_t ctx, b200_vec_t f, b200_csr_t A, b200_vec_t x,
                             b200_vec_t r) {
    return residual_impl(ctx, f, A, x, r, nullptr);
}

// ---------------------------------------------------------------------------
// smoother sweep
// ---------------------------------------------------------------------------
namespace b200 {

template <class TD, class TF, class TX>
static int relax_zero_t(b200_ctx_t ctx, double omega, const double *pd, const double *pf, b200_vec_t x) {
    if (x->len && std::is_same<TD, double>::value && std::is_same<TF, double>::value &&
        std::is_same<TX, double>::value && tail_enabled(ctx) && (int64_t)x->len <= ctx->opt_tail_max_vec &&
        x->kind == B200_VK_LOCAL) {
        const int rc = tail_enqueue_relax_zero(ctx, x->len, omega, pd, pf, wr(x));
        x->zero_pending = false;
        return rc;
    }
    if (x->len) {
        const int trc = tail_flush(ctx);
        if (trc) return trc;
        const int grid = grid_for(ctx, x->len, 2);
        ProfScope prof(ctx, B200_PROF_RELAX_ZERO, (int64_t)x->len, 1, 0);
        B200_CUDA(launch_pdl(ctx, relax_zero_kernel<TD, TF, TX>, dim3(grid), dim3(kThreads), 0, x->len, omega,
                             tp<TD>(pd), tp<TF>(pf), tp<TX>(wr(x))));
        B200_CHECK_LAUNCH();
        ctx->launches++;
    }
    x->zero_pending = false;
    return B200_OK;
}

} // namespace b200

namespace b200 {
// The pending first sweep x = (omega*d).*f is written out by its own element-wise kernel
// (what b200_relax would have launched): some call other than the matching b200_residual came.
int lazy_flush(b200_ctx_t ctx) {
    b200_vec_t v = ctx->lazy_vec;
    if (!v) return B200_OK;
    ctx->lazy_vec = nullptr;
    v->scale_pending = false;
    const double *pd = v->sc_d, *pf = v->sc_f;
    v->sc_d = v->sc_f = nullptr;
    v->sc_fvec = nullptr;
    DeviceGuard guard(ctx->device);
    if (!guard.ok) return fail(B200_ECUDA, "cudaSetDevice failed");
    return relax_zero_t<double, double, double>(ctx, v->sc_omega, pd, pf, v);
}

// first sweep + residual as one pass pays where the extra gathers are cheap (short rows: the
// finest level and the P-like operators) or where a launch costs more than the work (tiny levels)
static bool first_sweep_fusable(b200_ctx_t ctx, b200_csr_t A) {
    return ctx->opt_fuse_first_sweep && ctx->opt_zero_shortcut && ctx->opt_spmv_variant == 1 &&
           A->dtype == B200_F64 && A->kind == B200_CK_LOCAL && !A->gather_rows && A->nlong == 0 &&
           A->gl_rows == A->gl_cols && (A->lanes == 1 || A->nrows <= 32768) && !tail_enabled(ctx);
}
} // namespace b200

extern "C" int b200_relax(b200_ctx_t ctx, b200_csr_t A, b200_vec_t rhs, b200_vec_t x,
                          b200_vec_t tmp, b200_vec_t diag, double omega) {
    CHECK_CTX(ctx);
    B200_REQUIRE(A && rhs && x && tmp && diag, "null argument");
    touch(ctx, {rhs, x, tmp, diag});
    B200_REQUIRE(A->gl_rows == A->gl_cols, "relax: matrix must be square");
    B200_REQUIRE((int64_t)x->n == A->gl_rows && same_layout(x, rhs) && same_layout(x, diag) &&
                     same_layout(x, tmp),
                 "relax: vector size != matrix rows");
    B200_REQUIRE(x != tmp && x != rhs && tmp != rhs, "relax: x, tmp and rhs must be distinct vectors");
    B200_REQUIRE(!A->gather_rows, "relax: operator must be square");
    B200_REQUIRE(x->ptr != tmp->ptr, "relax: x and tmp must not alias");
    GUARD_DEFER(ctx);
    TailHold hold(ctx, {rhs, x, tmp, diag});

    // precision combination: 0 = FP64 throughout, 1 = FP32 throughout,
    // 2 = FP32 operator + diagonal sweeping an FP64 iterate (finest level of a mixed hierarchy;
    //     tmp is that level's FP32 scratch)
    int mix = -1;
    if (A->dtype == B200_F64 && all64({rhs, x, tmp, diag})) mix = 0;
    else if (A->dtype == B200_F32 && all32({rhs, x, tmp, diag})) mix = 1;
    else if (A->dtype == B200_F32 && all64({rhs, x}) && all32({tmp, diag})) mix = 2;
    if (mix < 0) return B200_BAD_MIX("relax");

    const double *pf, *pd;
    int rc = rd(rhs, &pf);
    if (rc) return rc;
    rc = rd(diag, &pd);
    if (rc) return rc;

    if (x->zero_pending && ctx->opt_zero_shortcut) {
        // residual(rhs, A, 0) == rhs exactly, so the sweep reduces to a scaling ...
        if (mix == 0 && first_sweep_fusable(ctx, A) && x->owned && !x->escaped && x->kind == B200_VK_LOCAL &&
            x->len == (size_t)A->nrows && !ctx->dist) {
            // ... which the b200_residual that normally follows can do on the fly: postpone it
            x->zero_pending = false;
            x->scale_pending = true;
            x->sc_d = pd; x->sc_f = pf; x->sc_fvec = rhs; x->sc_omega = omega;
            x->gen++;
            ctx->lazy_vec = x;
            return B200_OK;
        }
        if (mix == 0) return relax_zero_t<double, double, double>(ctx, omega, pd, pf, x);
        if (mix == 1) return relax_zero_t<float, float, float>(ctx, omega, pd, pf, x);
        return relax_zero_t<float, double, double>(ctx, omega, pd, pf, x);
    }

    if (!ctx->opt_fuse_relax) {
        // the literal reference sequence: tmp = rhs - A x ; x = omega*diag.*tmp + x
        rc = b200_residual(ctx, rhs, A, x, tmp);
        if (rc) return rc;
        return b200_vmul(ctx, omega, diag, tmp, 1.0, x);
    }

    if (mix == 1) {
        CsrArgsT<PrecFF> a = base_args_t<PrecFF>(A);
        const double *px;
        rc = rd(x, &px);
        if (rc) return rc;
        a.x = tp<float>(px); a.f = tp<float>(pf); a.d = tp<float>(pd); a.alpha = omega;
        if (A->kind == B200_CK_HALO) {
            B200_REQUIRE(x->kind == B200_VK_DIST, "relax: vectors must be partitioned like the operator");
            rc = halo_into(ctx, A, a);
            if (rc) return rc;
        }
        a.y = tp<float>(wr(tmp));
        rc = launch_csr<MODE_RELAX>(ctx, A, a);
        if (rc) return rc;
        x->gen++; tmp->gen++;
        if (x->owned && tmp->owned && x->cap == tmp->cap) std::swap(x->ptr, tmp->ptr);
        else {
            if ((rc = tail_flush(ctx))) return rc;
            B200_CUDA(cudaMemcpyAsync(x->ptr, tmp->ptr, x->len * x->esz, cudaMemcpyDeviceToDevice, ctx->stream));
        }
        return B200_OK;
    }
    if (mix == 2) {
        // the new FP64 iterate cannot live in the level's FP32 scratch: the operator owns an
        // FP64 buffer that trades places with x exactly like tmp does in the uniform case
        if (!A->scratch64)
            B200_CUDA(cudaMalloc(&A->scratch64, ((size_t)A->nrows + 4) * sizeof(double)));
        if (ctx->recording) touch_slot(ctx, &A->scratch64, nullptr);
        CsrArgsT<PrecFD> a = base_args_t<PrecFD>(A);
        const double *px;
        rc = rd(x, &px);
        if (rc) return rc;
        a.x = px; a.f = pf; a.d = tp<float>(pd); a.alpha = omega;
        if (A->kind == B200_CK_HALO) {
            B200_REQUIRE(x->kind == B200_VK_DIST, "relax: vectors must be partitioned like the operator");
            rc = halo_into(ctx, A, a);
            if (rc) return rc;
        }
        a.y = A->scratch64;
        // a Krylov solver of this size is alive: leave <rhs, x_new> behind (cg.hpp:184)
        DotReq req;
        int pslot = -1;
        if (product_wanted(ctx, (size_t)A->gl_rows)) {
            pslot = product_take_slot(ctx);
            req.ndot = 1; req.slots = &pslot;
            apply_req(ctx, A, a, &req);
        }
        rc = launch_csr<MODE_RELAX>(ctx, A, a);
        if (rc) return rc;
        x->gen++;
        if (x->owned && x->cap == (size_t)A->nrows) std::swap(x->ptr, A->scratch64);
        else {
            if ((rc = tail_flush(ctx))) return rc;
            B200_CUDA(cudaMemcpyAsync(x->ptr, A->scratch64, x->len * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
        }
        if (req.done) product_record(ctx, rhs, x, pslot);
        return B200_OK;
    }

    CsrArgs a = base_args(A);
    rc = rd(x, &a.x);
    if (rc) return rc;
    if (A->kind == B200_CK_HALO) {
        B200_REQUIRE(x->kind == B200_VK_DIST, "relax: vectors must be partitioned like the operator");
        rc = halo_into(ctx, A, a);
        if (rc) return rc;
    }
    a.f = pf; a.d = pd; a.alpha = omega;
    a.y = wr(tmp);
    // a Krylov solver of this size is alive: leave <rhs, x_new> behind (cg.hpp:184 asks for
    // exactly this product right after the V-cycle's last sweep)
    DotReq req;
    int pslot = -1;
    if (product_wanted(ctx, (size_t)A->gl_rows)) {
        pslot = product_take_slot(ctx);
        req.ndot = 1; req.slots = &pslot;
        apply_req(ctx, A, a, &req);
    }
    rc = launch_csr<MODE_RELAX>(ctx, A, a);
    if (rc) return rc;
    x->gen++;
    if (x->owned && tmp->owned && x->cap == tmp->cap) {
        std::swap(x->ptr, tmp->ptr);          // x now holds the new iterate
    } else {
        if ((rc = tail_flush(ctx))) return rc;
        B200_CUDA(cudaMemcpyAsync(x->ptr, tmp->ptr, x->len * sizeof(double),
                                  cudaMemcpyDeviceToDevice, ctx->stream));
    }
    if (req.done) product_record(ctx, rhs, x, pslot);
    return B200_OK;
}

