// api_coarse.cu -- coarsest-level direct solver (dense inverse on the device; levels above
// kCoarseDenseMax rows go to the banded LU of api_coarse_lu.cu)
//
// Part of the implementation of the C ABI declared in include/amgcl_b200.h (host-side logic
// only: argument checking, bookkeeping, kernel launches; no CPU fallback anywhere).
#include "internal.cuh"
#include "coarse_kernels.cuh"

using namespace b200;

// ---------------------------------------------------------------------------
// coarse solve
// ---------------------------------------------------------------------------
namespace b200 {

template <class Ptr, class Col, class Val>
static int coarse_create(b200_ctx_t ctx, int64_t n, const Ptr *ptr, const Col *col,
                         const Val *val, b200_coarse_t *out) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "coarse solver creation");
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    B200_REQUIRE(n > 0, "coarse solver: n must be positive");
    B200_REQUIRE(!ctx->dist || n <= kCoarseDenseMax,
                 "coarse solver: a multi-GPU context solves coarsest levels of at most 16384 rows "
                 "(lower coarse_enough)");
    B200_REQUIRE(n < ((int64_t)1 << 31), "coarse solver: n does not fit int32");
    B200_REQUIRE(ptr && ptr[0] == 0, "bad row pointer array");
    const int64_t nnz = (int64_t)ptr[n];
    B200_REQUIRE(nnz >= 0 && (nnz == 0 || (col && val)), "bad col/val array");
    GUARD(ctx);
    // multi-GPU: a coarsest level below the partition threshold is replicated -- every rank
    // forms the inverse and solves redundantly (no exchange); a partitioned one keeps the
    // inverse on every rank and applies its own rows to the all-gathered right-hand side
    const bool replicated = ctx->dist && n >= ctx->dist_min_rows;

    std::vector<int32_t> hptr((size_t)n + 1), hcol((size_t)nnz);
    for (int64_t i = 0; i <= n; ++i) hptr[(size_t)i] = (int32_t)ptr[i];
    for (int64_t e = 0; e < nnz; ++e) {
        const int64_t c = (int64_t)col[e];
        if (c < 0 || c >= n) return fail(B200_EINVAL, "coarse solver: column index out of range");
        hcol[(size_t)e] = (int32_t)c;
    }

    // the inverse is always formed and kept in FP64, whatever the hierarchy's precision
    std::vector<double> hval((size_t)nnz);
    for (int64_t e = 0; e < nnz; ++e) hval[(size_t)e] = (double)val[e];
    if (n > kCoarseDenseMax) {
        for (int64_t i = 0; i < n; ++i)
            if (hptr[(size_t)i + 1] < hptr[(size_t)i]) return fail(B200_EINVAL, "bad row pointer array");
        b200_coarse_s *S = new (std::nothrow) b200_coarse_s();
        if (!S) return fail(B200_ENOMEM, "out of host memory");
        S->ctx = ctx; S->n = n;
        S->dtype = std::is_same<Val, float>::value ? B200_F32 : B200_F64;
        const int rc = coarse_lu_create(ctx, n, hptr, hcol, hval, S);
        if (rc) { delete S; return rc; }
        *out = S;
        return B200_OK;
    }
    const int N = (int)n;
    int *dptr = nullptr, *dcol = nullptr, *dpiv = nullptr;
    double *dval = nullptr, *M = nullptr, *colk = nullptr, *pivval = nullptr, *Ainv = nullptr;
    auto cleanup = [&]() {
        cudaFree(dptr); cudaFree(dcol); cudaFree(dval); cudaFree(M);
        cudaFree(colk); cudaFree(dpiv); cudaFree(pivval);
    };
#define CO_CUDA(call)                                                          \
    do {                                                                       \
        cudaError_t rc__ = (call);                                             \
        if (rc__ != cudaSuccess) {                                             \
            cleanup();                                                         \
            cudaFree(Ainv);                                                    \
            return cuda_fail(rc__, #call, __FILE__, __LINE__);                 \
        }                                                                      \
    } while (0)
    const size_t Mbytes = (size_t)N * 2 * N * sizeof(double);
    CO_CUDA(cudaMalloc(&dptr, ((size_t)N + 1) * sizeof(int)));
    CO_CUDA(cudaMalloc(&dcol, std::max<size_t>(1, (size_t)nnz) * sizeof(int)));
    CO_CUDA(cudaMalloc(&dval, std::max<size_t>(1, (size_t)nnz) * sizeof(double)));
    CO_CUDA(cudaMalloc(&M, Mbytes));
    CO_CUDA(cudaMalloc(&colk, (size_t)N * sizeof(double)));
    CO_CUDA(cudaMalloc(&dpiv, sizeof(int)));
    CO_CUDA(cudaMalloc(&pivval, ((size_t)N + 1) * sizeof(double)));
    CO_CUDA(cudaMalloc(&Ainv, (size_t)N * N * sizeof(double)));
    cudaStream_t st = ctx->stream;
    CO_CUDA(cudaMemcpyAsync(dptr, hptr.data(), ((size_t)N + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
    if (nnz) {
        CO_CUDA(cudaMemcpyAsync(dcol, hcol.data(), (size_t)nnz * sizeof(int), cudaMemcpyHostToDevice, st));
        CO_CUDA(cudaMemcpyAsync(dval, hval.data(), (size_t)nnz * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    CO_CUDA(cudaMemsetAsync(M, 0, Mbytes, st));
    coarse_scatter_kernel<<<(N + 127) / 128, 128, 0, st>>>(N, dptr, dcol, dval, M);
    CO_CUDA(cudaGetLastError());
    ctx->launches++;

    const int gcol2 = (2 * N + kThreads - 1) / kThreads;
    const int gcol1 = (N + kThreads - 1) / kThreads;
    const int ysplit = std::max(1, std::min(N, (ctx->sm_count * 4) / std::max(1, gcol2)));
    for (int k = 0; k < N; ++k) {
        coarse_pivot_kernel<<<1, kThreads, 0, st>>>(N, k, M, dpiv, pivval + k);
        coarse_colk_kernel<<<gcol1, kThreads, 0, st>>>(N, k, M, dpiv, colk);
        coarse_swap_scale_kernel<<<gcol2, kThreads, 0, st>>>(N, k, M, dpiv, pivval + k);
        const int gx = (2 * N - k + kThreads - 1) / kThreads;
        coarse_eliminate_kernel<<<dim3(gx, ysplit), kThreads, 0, st>>>(N, k, M, colk);
        ctx->launches += 4;
    }
    CO_CUDA(cudaGetLastError());
    {
        const size_t tot = (size_t)N * N;
        coarse_extract_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(N, M, Ainv);
        CO_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    std::vector<double> hpiv((size_t)N);
    CO_CUDA(cudaMemcpyAsync(hpiv.data(), pivval, (size_t)N * sizeof(double), cudaMemcpyDeviceToHost, st));
    CO_CUDA(cudaStreamSynchronize(st));
#undef CO_CUDA
    cleanup();
    double pmax = 0.0, pmin = std::numeric_limits<double>::infinity();
    for (double p : hpiv) {
        const double a = std::fabs(p);
        if (!(a == a)) { pmin = 0.0; break; }   // NaN
        pmax = std::max(pmax, a);
        pmin = std::min(pmin, a);
    }
    if (!(pmin > 0.0) || pmin < pmax * 1e-14 || !std::isfinite(pmax)) {
        cudaFree(Ainv);
        return fail(B200_ESINGULAR, "coarse matrix is numerically singular");
    }

    b200_coarse_s *S = new (std::nothrow) b200_coarse_s();
    if (!S) {
        cudaFree(Ainv);
        return fail(B200_ENOMEM, "out of host memory");
    }
    S->ctx = ctx; S->n = n; S->Ainv = Ainv; S->bytes = (size_t)N * N * sizeof(double);
    S->dtype = std::is_same<Val, float>::value ? B200_F32 : B200_F64;
    if (replicated) {
        // the coarsest level is itself partitioned: every rank keeps the inverse and
        // applies its own rows to the all-gathered right-hand side
        S->replicated = true;
        S->block = Partition(n, ctx->nranks).B;
        cudaError_t rc = cudaMalloc(&S->gbuf, ((size_t)S->block * ctx->nranks + 2) * sizeof(double));
        if (rc != cudaSuccess) {
            cudaFree(Ainv);
            delete S;
            return cuda_fail(rc, "cudaMalloc(coarse gather buffer)", __FILE__, __LINE__);
        }
        S->bytes += (size_t)S->block * ctx->nranks * sizeof(double);
    }
    *out = S;
    return B200_OK;
}

} // namespace b200

extern "C" int b200_coarse_create_i64(b200_ctx_t ctx, int64_t n, const int64_t *ptr,
                                      const int64_t *col, const double *val, b200_coarse_t *S) {
    return coarse_create(ctx, n, ptr, col, val, S);
}
extern "C" int b200_coarse_create_i32(b200_ctx_t ctx, int64_t n, const int32_t *ptr,
                                      const int32_t *col, const double *val, b200_coarse_t *S) {
    return coarse_create(ctx, n, ptr, col, val, S);
}

extern "C" int b200_coarse_create_i64_f32(b200_ctx_t ctx, int64_t n, const int64_t *ptr,
                                          const int64_t *col, const float *val, b200_coarse_t *S) {
    CHECK_CTX(ctx);
    return coarse_create(ctx, n, ptr, col, val, S);
}
extern "C" int b200_coarse_create_i32_f32(b200_ctx_t ctx, int64_t n, const int32_t *ptr,
                                          const int32_t *col, const float *val, b200_coarse_t *S) {
    CHECK_CTX(ctx);
    return coarse_create(ctx, n, ptr, col, val, S);
}

extern "C" int b200_coarse_destroy(b200_coarse_t S) {
    if (!S) return B200_OK;
    NOT_RECORDING(S->ctx, "coarse solver destruction");
    if (S->in_graph) S->ctx->destroy_epoch++;
    GUARD(S->ctx);
    if (S->Ainv) cudaFree(S->Ainv);
    coarse_lu_destroy(S->lu);
    if (S->gbuf) cudaFree(S->gbuf);
    delete S;
    return B200_OK;
}

extern "C" int b200_coarse_bytes(b200_coarse_t S, size_t *bytes) {
    B200_REQUIRE(S && bytes, "null argument");
    *bytes = S->bytes;
    return B200_OK;
}

extern "C" int b200_coarse_solve(b200_ctx_t ctx, b200_coarse_t S, b200_vec_t rhs, b200_vec_t x) {
    CHECK_CTX(ctx);
    B200_REQUIRE(S && rhs && x, "null argument");
    touch(ctx, {rhs, x});
    if (ctx->recording) S->in_graph = true;
    B200_REQUIRE((int64_t)rhs->n == S->n && (int64_t)x->n == S->n, "coarse solve: size mismatch");
    GUARD_DEFER(ctx);
    TailHold hold(ctx, {rhs, x});
    const int N = (int)S->n;
    const int warps_per_cta = kThreads / 32;
    if (S->replicated) {
        B200_REQUIRE(rhs->kind == B200_VK_DIST && x->kind == B200_VK_DIST &&
                         (int64_t)rhs->cap == S->block && rhs != x,
                     "coarse solve: vectors must be partitioned like the coarsest level");
        int rc = materialize(rhs);
        if (rc) return rc;
        if ((rc = tail_flush(ctx))) return rc;
        if (rhs->dtype != x->dtype) return B200_BAD_MIX("coarse solve");
        const bool f32 = rhs->dtype == B200_F32;
        B200_NCCL(nccl().AllGather(rhs->ptr, S->gbuf, (size_t)S->block, f32 ? ncclFloat : ncclDouble,
                                   comm_of(ctx), ctx->stream));
        const int nloc = (int)x->len;
        if (nloc) {
            ProfScope prof(ctx, B200_PROF_COARSE, nloc, S->n, (int64_t)nloc * S->n);
            const unsigned grid = (unsigned)((nloc + warps_per_cta - 1) / warps_per_cta);
            if (f32)
                coarse_gemv_kernel<float><<<grid, kThreads, 0, ctx->stream>>>(
                    N, (int)x->off, nloc, S->Ainv, tp<float>(S->gbuf), tp<float>(wr(x)));
            else
                coarse_gemv_kernel<double><<<grid, kThreads, 0, ctx->stream>>>(
                    N, (int)x->off, nloc, S->Ainv, S->gbuf, wr(x));
            B200_CHECK_LAUNCH();
            ctx->launches++;
        }
        x->zero_pending = false;
        return B200_OK;
    }
    B200_REQUIRE(rhs->kind == B200_VK_LOCAL && x->kind == B200_VK_LOCAL,
                 "coarse solve: vectors must live on this rank");
    B200_REQUIRE(rhs != x && rhs->ptr != x->ptr, "coarse solve: rhs and x must not alias");
    if (rhs->dtype != x->dtype) return B200_BAD_MIX("coarse solve");
    if (S->lu) return coarse_lu_solve(ctx, S, rhs, x);        // flushes the coarse tail
    const double *pr;
    int rc = rd(rhs, &pr);
    if (rc) return rc;
    if (rhs->dtype == B200_F64 && tail_enabled(ctx) && (int64_t)N * N <= 4 * ctx->opt_tail_max_nnz)
        return tail_enqueue_gemv(ctx, N, S->Ainv, pr, wr(x));      // part of the coarse tail
    if ((rc = tail_flush(ctx))) return rc;
    ProfScope prof(ctx, B200_PROF_COARSE, S->n, S->n, S->n * S->n);
    if (rhs->dtype == B200_F32)
        B200_CUDA(launch_pdl(ctx, coarse_gemv_kernel<float>, dim3((N + warps_per_cta - 1) / warps_per_cta),
                             dim3(kThreads), 0, N, 0, N, (const double *)S->Ainv, tp<float>(pr),
                             tp<float>(wr(x))));
    else
        B200_CUDA(launch_pdl(ctx, coarse_gemv_kernel<double>, dim3((N + warps_per_cta - 1) / warps_per_cta),
                             dim3(kThreads), 0, N, 0, N, (const double *)S->Ainv, pr, wr(x)));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}

