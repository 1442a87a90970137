// api_tail.cu -- deferred execution of the coarse tail of the V-cycle (tail_kernels.cuh)
//
// Part of the implementation of the C ABI declared in include/amgcl_b200.h (host-side logic
// only: argument checking, bookkeeping, kernel launches; no CPU fallback anywhere).
//
// b200_spmv / b200_residual / b200_relax / b200_coarse_solve on a SMALL operator do not launch:
// they append a command (the device pointers and scalars the stand-alone kernel would have
// received) to the context's pending list.  Everything else the library does on the device
// first flushes the list -- one cooperative launch of coarse_tail_kernel -- so the order of
// effects on the stream is exactly the order of the calls.  The host-side state a call updates
// (storage swaps of b200_relax, lazy-clear flags, generation counters) is updated when the call
// is made, as in the immediate path; only the device work is postponed.
#include "internal.cuh"
#include "tail_kernels.cuh"

using namespace b200;

namespace b200 {

static TailArgs *tail_list(b200_ctx_t ctx) {
    if (!ctx->tail) {
        ctx->tail = new (std::nothrow) TailArgs();
        if (ctx->tail) memset(ctx->tail, 0, sizeof(TailArgs));
    }
    return static_cast<TailArgs *>(ctx->tail);
}

void tail_destroy(b200_ctx_t ctx) {
    delete static_cast<TailArgs *>(ctx->tail);
    ctx->tail = nullptr;
    if (ctx->tail_bar) cudaFree(ctx->tail_bar);
    ctx->tail_bar = nullptr;
}

bool tail_enabled(b200_ctx_t ctx) {
    return ctx->opt_coarse_tail && !ctx->recording && !ctx->tail_hold;
}

bool tail_accepts_csr(b200_ctx_t ctx, b200_csr_t A) {
    return tail_enabled(ctx) && A->dtype == B200_F64 && A->kind == B200_CK_LOCAL && !A->gather_rows &&
           A->nlong == 0 && A->nrows > 0 && A->nnz <= ctx->opt_tail_max_nnz &&
           A->nrows < (int64_t)1 << 30;
}

int tail_flush(b200_ctx_t ctx) {
    TailArgs *t = static_cast<TailArgs *>(ctx->tail);
    if (!t || t->n == 0) return B200_OK;
    if (!ctx->tail_bar) {
        B200_CUDA(cudaMalloc(&ctx->tail_bar, sizeof(unsigned long long)));
        B200_CUDA(cudaMemsetAsync(ctx->tail_bar, 0, sizeof(unsigned long long), ctx->stream));
        ctx->tail_bar_count = 0;
    }
    t->bar = ctx->tail_bar;
    t->bar_base = ctx->tail_bar_count;
    ctx->tail_bar_count += (unsigned long long)(t->n - 1) * (unsigned long long)ctx->sm_count;
    int64_t work = 0;
    for (int k = 0; k < t->n; ++k) work += t->cmd[k].nrows;
    const int n = t->n;
    TailArgs args = *t;
    t->n = 0;                                   // (before anything below can re-enter)
    ProfScope prof(ctx, B200_PROF_TAIL, (int64_t)n, 1, work);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)ctx->sm_count);       // one CTA per SM, all co-resident
    cfg.blockDim = dim3(kTailThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B200_CUDA(cudaLaunchKernelEx(&cfg, coarse_tail_kernel, args));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    ctx->tail_flushes++;
    ctx->tail_commands += (uint64_t)n;
    return B200_OK;
}

static int tail_push(b200_ctx_t ctx, const TailCmd &c) {
    TailArgs *t = tail_list(ctx);
    if (!t) return fail(B200_ENOMEM, "out of host memory");
    if (t->n == kTailMaxCmds) {
        const int rc = tail_flush(ctx);
        if (rc) return rc;
    }
    t->cmd[t->n++] = c;
    return B200_OK;
}

// One small FP64 operator as one plain launch of the direct-load kernel (option
// "small_kernel_max_nnz"; modes 0-3).  Same arithmetic as the ring kernel.
bool small_csr_accepts(b200_ctx_t ctx, b200_csr_t A) {
    return ctx->opt_small_kernel_max_nnz > 0 && A->dtype == B200_F64 && A->kind == B200_CK_LOCAL &&
           !A->gather_rows && A->nlong == 0 && A->nrows > 0 && A->nnz <= ctx->opt_small_kernel_max_nnz;
}

int small_csr_launch(b200_ctx_t ctx, int mode, b200_csr_t A, const CsrArgsT<PrecDD> &a) {
    TailCmd c;
    memset(&c, 0, sizeof(c));
    c.op = TAIL_CSR; c.mode = mode; c.nrows = (int)A->nrows; c.lanes = A->lanes;
    c.ptr = A->ptr; c.col = A->col; c.val = static_cast<const double *>(A->val);
    c.x = a.x; c.f = a.f; c.d = a.d; c.y = a.y;
    c.alpha = a.alpha; c.beta = a.beta;
    const int64_t want = ((int64_t)A->nrows * A->lanes + kThreads - 1) / kThreads;
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)ctx->sm_count * 8));
    if (ctx->recording) A->in_graph = true;
    ProfScope prof(ctx, mode, A->nrows, A->ncols, A->nnz, 0, (int)sizeof(double));
    cudaError_t rc;
    switch (A->lanes) {
    case 1:  rc = launch_pdl(ctx, small_csr_kernel<1>, dim3(grid), dim3(kThreads), 0, c); break;
    case 2:  rc = launch_pdl(ctx, small_csr_kernel<2>, dim3(grid), dim3(kThreads), 0, c); break;
    case 4:  rc = launch_pdl(ctx, small_csr_kernel<4>, dim3(grid), dim3(kThreads), 0, c); break;
    case 8:  rc = launch_pdl(ctx, small_csr_kernel<8>, dim3(grid), dim3(kThreads), 0, c); break;
    case 16: rc = launch_pdl(ctx, small_csr_kernel<16>, dim3(grid), dim3(kThreads), 0, c); break;
    default: rc = launch_pdl(ctx, small_csr_kernel<32>, dim3(grid), dim3(kThreads), 0, c); break;
    }
    B200_CUDA(rc);
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}

int tail_enqueue_csr(b200_ctx_t ctx, int mode, b200_csr_t A, const CsrArgsT<PrecDD> &a) {
    TailCmd c;
    memset(&c, 0, sizeof(c));
    c.op = TAIL_CSR; c.mode = mode; c.nrows = (int)A->nrows; c.lanes = A->lanes;
    c.ptr = A->ptr; c.col = A->col; c.val = static_cast<const double *>(A->val);
    c.x = a.x; c.f = a.f; c.d = a.d; c.y = a.y;
    c.alpha = a.alpha; c.beta = a.beta;
    return tail_push(ctx, c);
}

int tail_enqueue_relax_zero(b200_ctx_t ctx, size_t n, double omega, const double *d, const double *f, double *x) {
    TailCmd c;
    memset(&c, 0, sizeof(c));
    c.op = TAIL_RELAX_ZERO; c.nrows = (int)n; c.d = d; c.f = f; c.y = x; c.alpha = omega;
    return tail_push(ctx, c);
}

int tail_enqueue_gemv(b200_ctx_t ctx, int n, const double *Ainv, const double *rhs, double *x) {
    TailCmd c;
    memset(&c, 0, sizeof(c));
    c.op = TAIL_GEMV; c.nrows = n; c.val = Ainv; c.x = rhs; c.y = x;
    return tail_push(ctx, c);
}

} // namespace b200

extern "C" int b200_tail_stats(b200_ctx_t ctx, uint64_t *flushes, uint64_t *commands) {
    CHECK_CTX(ctx);
    if (flushes) *flushes = ctx->tail_flushes;
    if (commands) *commands = ctx->tail_commands;
    return B200_OK;
}
