// api_vectors.cu -- vectors, element-wise kernels, inner product
//
// Part of the implementation of the C ABI declared in include/amgcl_b200.h (host-side logic
// only: argument checking, bookkeeping, kernel launches; no CPU fallback anywhere).
#include "internal.cuh"
#include "vec_kernels.cuh"

using namespace b200;

// ---------------------------------------------------------------------------
// vectors
// ---------------------------------------------------------------------------
static int vec_create_typed(b200_ctx_t ctx, size_t n, int dtype, b200_vec_t *out) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "vector creation");
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    GUARD(ctx);
    b200_vec_s *v = new (std::nothrow) b200_vec_s();
    if (!v) return fail(B200_ENOMEM, "out of host memory");
    v->ctx = ctx;
    v->n = n;
    v->owned = true;
    v->dtype = dtype;
    v->esz = dtype == B200_F32 ? sizeof(float) : sizeof(double);
    if (ctx->dist && (int64_t)n >= ctx->dist_min_rows) {
        const Partition part((int64_t)n, ctx->nranks);
        v->kind = B200_VK_DIST;
        v->off = (size_t)part.lo(ctx->rank);
        v->len = (size_t)part.count(ctx->rank);
        v->cap = (size_t)part.B;
    } else {
        // single GPU, or a level below the partition threshold: replicated on every rank
        v->kind = B200_VK_LOCAL;
        v->len = n;
        v->cap = n;
    }
    // +2 doubles of padding so 16-byte vector accesses of the tail stay in bounds
    cudaError_t rc = cudaMalloc(&v->ptr, (v->cap + 4) * v->esz);
    if (rc != cudaSuccess) {
        delete v;
        return cuda_fail(rc, "cudaMalloc(vector)", __FILE__, __LINE__);
    }
    if (v->cap > v->len) {
        // padding of a partial block takes part in collectives: keep it zero
        rc = cudaMemsetAsync(reinterpret_cast<char *>(v->ptr) + v->len * v->esz, 0, (v->cap - v->len) * v->esz,
                             ctx->stream);
        if (rc != cudaSuccess) {
            cudaFree(v->ptr);
            delete v;
            return cuda_fail(rc, "cudaMemsetAsync(vector padding)", __FILE__, __LINE__);
        }
    }
    v->zero_pending = true;   // logically zero; memset only if somebody looks
    *out = v;
    return B200_OK;
}

extern "C" int b200_vec_create(b200_ctx_t ctx, size_t n, b200_vec_t *out) {
    return vec_create_typed(ctx, n, B200_F64, out);
}

extern "C" int b200_vec_create_f32(b200_ctx_t ctx, size_t n, b200_vec_t *out) {
    return vec_create_typed(ctx, n, B200_F32, out);
}

extern "C" int b200_vec_dtype(b200_vec_t v, int *dtype) {
    B200_REQUIRE(v && dtype, "null argument");
    *dtype = v->dtype;
    return B200_OK;
}

extern "C" int b200_vec_wrap(b200_ctx_t ctx, double *device_ptr, size_t n, b200_vec_t *out) {
    CHECK_CTX(ctx);
    B200_REQUIRE(out != nullptr, "null output pointer");
    B200_REQUIRE(device_ptr != nullptr || n == 0, "null device pointer");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(device_ptr) & 7) == 0, "device pointer not 8-byte aligned");
    B200_REQUIRE(!ctx->dist, "b200_vec_wrap is not available on a distributed context");
    b200_vec_s *v = new (std::nothrow) b200_vec_s();
    if (!v) return fail(B200_ENOMEM, "out of host memory");
    v->ctx = ctx;
    v->n = n;
    v->len = n;
    v->cap = n;
    v->ptr = device_ptr;
    v->owned = false;
    v->escaped = true;
    v->zero_pending = false;
    *out = v;
    return B200_OK;
}

extern "C" int b200_vec_destroy(b200_vec_t v) {
    if (!v) return B200_OK;
    if (v->ctx->lazy_vec == v) {            // a pending first sweep nobody will ever read
        v->ctx->lazy_vec = nullptr;
        v->scale_pending = false;
    }
    for (b200_ctx_s::Product &p : v->ctx->products)      // products that name this vector are gone
        if (p.a == v || p.b == v) p = b200_ctx_s::Product();
    if (b200_graph_s *g = v->ctx->recording) {
        // Typically a garbage-collected handle of the host language that has nothing to do with
        // the recording: its storage is released once the recording is over (cudaFree would
        // synchronise the device in the middle of a capture).  A vector the recording itself
        // uses cannot go away underneath it.
        for (const GraphSlot &s : g->slots)
            if (s.slot == &v->ptr)
                return fail(B200_EINVAL, "vector is used by the graph being recorded");
        if (v->in_graph) v->ctx->destroy_epoch++;
        if (v->owned && v->ptr) v->ctx->graph_deferred.push_back(v->ptr);
        delete v;
        return B200_OK;
    }
    if (v->in_graph) v->ctx->destroy_epoch++;      // recorded graphs that refer to it are dead
    GUARD(v->ctx);
    if (v->owned && v->ptr) {
        // cudaFree synchronises the device, so no kernel can still be using it
        cudaFree(v->ptr);
    }
    delete v;
    return B200_OK;
}

extern "C" int b200_vec_size(b200_vec_t v, size_t *n) {
    B200_REQUIRE(v && n, "null argument");
    *n = v->n;
    return B200_OK;
}

extern "C" int b200_vec_bytes(b200_vec_t v, size_t *bytes) {
    B200_REQUIRE(v && bytes, "null argument");
    *bytes = v->len * v->esz;
    return B200_OK;
}

extern "C" int b200_vec_data(b200_vec_t v, double **device_ptr) {
    B200_REQUIRE(v && device_ptr, "null argument");
    B200_REQUIRE(v->dtype == B200_F64, "b200_vec_data: FP64 vectors only");
    GUARD(v->ctx);
    int rc = materialize(v);
    *device_ptr = v->ptr;
    v->escaped = true;          // the caller may write through the raw pointer
    v->gen++;
    return rc;
}

extern "C" int b200_vec_upload_f32(b200_vec_t v, const float *host, size_t n) {
    B200_REQUIRE(v && (host || n == 0), "null argument");
    NOT_RECORDING(v->ctx, "host transfer");
    B200_REQUIRE(n == v->n, "size mismatch in vector upload");
    B200_REQUIRE(v->dtype == B200_F32, "upload_f32: FP32 vector expected");
    GUARD(v->ctx);
    if (v->len) {
        // distributed: every rank is handed the full host vector and keeps its block
        B200_CUDA(cudaMemcpyAsync(wr(v), host + v->off, v->len * sizeof(float), cudaMemcpyHostToDevice,
                                  v->ctx->stream));
        B200_CUDA(cudaStreamSynchronize(v->ctx->stream));
    }
    v->zero_pending = false;
    return B200_OK;
}

extern "C" int b200_vec_download_f32(b200_vec_t v, float *host, size_t n) {
    B200_REQUIRE(v && (host || n == 0), "null argument");
    NOT_RECORDING(v->ctx, "host transfer");
    B200_REQUIRE(n == v->n, "size mismatch in vector download");
    B200_REQUIRE(v->dtype == B200_F32 && v->kind == B200_VK_LOCAL,
                 "download_f32: FP32 vector of a replicated level (or a single GPU) expected");
    GUARD(v->ctx);
    if (!n) return B200_OK;
    int rc = materialize(v);
    if (rc) return rc;
    B200_CUDA(cudaMemcpyAsync(host, v->ptr, n * sizeof(float), cudaMemcpyDeviceToHost, v->ctx->stream));
    B200_CUDA(cudaStreamSynchronize(v->ctx->stream));
    return B200_OK;
}

extern "C" int b200_vec_upload(b200_vec_t v, const double *host, size_t n) {
    B200_REQUIRE(v && (host || n == 0), "null argument");
    NOT_RECORDING(v->ctx, "host transfer");
    B200_REQUIRE(n == v->n, "size mismatch in vector upload");
    B200_REQUIRE(v->dtype == B200_F64, "b200_vec_upload: FP64 vector expected (use _f32)");
    GUARD(v->ctx);
    if (v->len) {
        // distributed: every rank is handed the full host vector and keeps its block
        B200_CUDA(cudaMemcpyAsync(wr(v), host + v->off, v->len * sizeof(double),
                                  cudaMemcpyHostToDevice, v->ctx->stream));
        B200_CUDA(cudaStreamSynchronize(v->ctx->stream));
    }
    v->zero_pending = false;
    return B200_OK;
}

extern "C" int b200_vec_download(b200_vec_t v, double *host, size_t n) {
    B200_REQUIRE(v && (host || n == 0), "null argument");
    NOT_RECORDING(v->ctx, "host transfer");
    B200_REQUIRE(n == v->n, "size mismatch in vector download");
    B200_REQUIRE(v->dtype == B200_F64, "b200_vec_download: FP64 vector expected (use _f32)");
    b200_ctx_t ctx = v->ctx;
    GUARD(ctx);
    if (!n) return B200_OK;
    if (v->kind == B200_VK_DIST) {
        // every rank receives the complete vector: all-gather the blocks, then one D2H copy
        int rc = materialize(v);
        if (rc) return rc;
        double *full = nullptr;
        B200_CUDA(cudaMalloc(&full, (size_t)ctx->nranks * v->cap * sizeof(double)));
        ncclResult_t nrc = nccl().AllGather(v->ptr, full, v->cap, ncclDouble, comm_of(ctx), ctx->stream);
        if (nrc != ncclSuccess) {
            cudaFree(full);
            return fail(B200_ENCCL, std::string("ncclAllGather: ") + nccl().GetErrorString(nrc));
        }
        cudaError_t crc = cudaMemcpyAsync(host, full, n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
        if (crc == cudaSuccess) crc = cudaStreamSynchronize(ctx->stream);
        cudaFree(full);
        if (crc != cudaSuccess) return cuda_fail(crc, "download(distributed)", __FILE__, __LINE__);
        return B200_OK;
    }
    if (v->zero_pending) {          // nothing to fetch: the vector is zero
        B200_CUDA(cudaStreamSynchronize(ctx->stream));
        memset(host, 0, n * sizeof(double));
        return B200_OK;
    }
    B200_CUDA(cudaMemcpyAsync(host, v->ptr, n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    return B200_OK;
}

// Partitioned vectors (multi-GPU): the block this rank owns, and a download of just that block
// into its place in a full-size host array -- what a row-distributed caller needs (each rank
// keeps the rows it owns, cf. amgcl::mpi's distributed vectors), without the all-gather of
// b200_vec_download.
extern "C" int b200_vec_local_range(b200_vec_t v, size_t *offset, size_t *len) {
    B200_REQUIRE(v && offset && len, "null argument");
    *offset = v->off;
    *len = v->len;
    return B200_OK;
}

extern "C" int b200_vec_download_local(b200_vec_t v, double *host, size_t n) {
    B200_REQUIRE(v && (host || n == 0), "null argument");
    NOT_RECORDING(v->ctx, "host transfer");
    B200_REQUIRE(n == v->n, "size mismatch in vector download");
    B200_REQUIRE(v->dtype == B200_F64, "b200_vec_download_local: FP64 vector expected");
    if (v->kind != B200_VK_DIST) return b200_vec_download(v, host, n);
    b200_ctx_t ctx = v->ctx;
    GUARD(ctx);
    if (!v->len) return B200_OK;
    if (v->zero_pending) {
        B200_CUDA(cudaStreamSynchronize(ctx->stream));
        memset(host + v->off, 0, v->len * sizeof(double));
        return B200_OK;
    }
    B200_CUDA(cudaMemcpyAsync(host + v->off, v->ptr, v->len * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    return B200_OK;
}

namespace b200 {

// ---- element-wise launch helpers ----------------------------------------------------------
// all streams of one element type T: 16-byte vector path when aligned
template <class F, bool RY, bool RZ, class T>
static int launch_ew(b200_ctx_t ctx, size_t n, F f, const T *x, const T *y, const T *z, T *out) {
    if (n == 0) return B200_OK;
    const bool vec_ok = aligned16(x) && aligned16(out) && (!RY || aligned16(y)) &&
                        (!RZ || aligned16(z));
    const int grid = grid_for(ctx, n, 16 / (int)sizeof(T) * 2);
    ProfScope prof(ctx, B200_PROF_VECTOR + (RY ? 1 : 0) + (RZ ? 1 : 0), (int64_t)n, 1, 0);
    B200_CUDA(launch_pdl(ctx, ew_kernel_same<F, RY, RZ, T>, dim3(grid), dim3(kThreads), 0, n, f, x, y, z, out,
                         vec_ok));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}
// mixed element types (FP32 inputs accumulated into an FP64 vector, precision-changing copy)
template <class F, bool RY, bool RZ, class TX, class TY, class TZ, class TO>
static int launch_ew_mixed(b200_ctx_t ctx, size_t n, F f, const TX *x, const TY *y, const TZ *z,
                           TO *out) {
    if (n == 0) return B200_OK;
    const int grid = grid_for(ctx, n, 2);
    ProfScope prof(ctx, B200_PROF_VECTOR + (RY ? 1 : 0) + (RZ ? 1 : 0), (int64_t)n, 1, 0);
    B200_CUDA(launch_pdl(ctx, ew_kernel<F, RY, RZ, TX, TY, TZ, TO>, dim3(grid), dim3(kThreads), 0, n, f, x, y,
                         z, out, false));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}

} // namespace b200

extern "C" int b200_clear(b200_ctx_t ctx, b200_vec_t x) {
    CHECK_CTX(ctx);
    B200_REQUIRE(x, "null argument");
    touch(ctx, {x});
    if (x->scale_pending) {                 // a first sweep nobody looked at: dropped
        x->scale_pending = false;
        x->sc_d = x->sc_f = nullptr;
        x->sc_fvec = nullptr;
        if (ctx->lazy_vec == x) ctx->lazy_vec = nullptr;
    }
    x->gen++;
    // memory the caller can see (wrapped, or its raw pointer handed out) is cleared at once:
    // the caller reads it behind the library's back
    if (ctx->opt_zero_shortcut && x->owned && !x->escaped) {
        x->zero_pending = true;
        return B200_OK;
    }
    GUARD(ctx);
    x->zero_pending = true;
    return materialize(x);
}

extern "C" int b200_copy(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y) {
    CHECK_CTX(ctx);
    B200_REQUIRE(x && y, "null argument");
    touch(ctx, {x, y});
    B200_REQUIRE(same_layout(x, y), "copy: size mismatch");
    if (x == y || x->ptr == y->ptr) return B200_OK;
    if (x->zero_pending) return b200_clear(ctx, y);     // drops a pending sweep of y, bumps its gen
    GUARD(ctx);
    if (all64({x, y}))
        return launch_ew<CopyF<double>, false, false, double>(ctx, x->len, CopyF<double>(), x->ptr, nullptr, nullptr, wr(y));
    if (all32({x, y}))
        return launch_ew<CopyF<float>, false, false, float>(ctx, x->len, CopyF<float>(), tp<float>(x->ptr), nullptr, nullptr, tp<float>(wr(y)));
    if (x->dtype == B200_F64)      // precision-changing copies
        return launch_ew_mixed<CopyF<float>, false, false>(ctx, x->len, CopyF<float>(), x->ptr, (const float *)nullptr, (const float *)nullptr, tp<float>(wr(y)));
    return launch_ew_mixed<CopyF<double>, false, false>(ctx, x->len, CopyF<double>(), tp<float>(x->ptr), (const double *)nullptr, (const double *)nullptr, wr(y));
}

namespace b200 {
template <class T>
static int launch_dot_kernel(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y, double *result_dev) {
    const bool vec_ok = aligned16(x->ptr) && aligned16(y->ptr);
    const int grid = std::min(grid_for(ctx, x->len, 32 / (int)sizeof(T) * 2), kDotMaxBlocks);
    ProfScope prof(ctx, B200_PROF_DOT, (int64_t)x->len, 1, 0);
    B200_CUDA(launch_pdl(ctx, dot_kernel<T>, dim3(grid), dim3(kThreads), 0, x->len,
                         (const T *)tp<T>(x->ptr), (const T *)tp<T>(y->ptr), ctx->dot_partial,
                         ctx->dot_ticket, result_dev, vec_ok));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}

// The stand-alone reduction kernel with the result in mapped host memory: FP32 vectors, and
// partitioned vectors when the exchange transport is NCCL (the peer-memory transport reduces
// inside the kernel, api_krylov.cu).  Arguments were checked by b200_dot.
int dot_legacy(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y, double *result) {
    const bool dist = x->kind == B200_VK_DIST;
    const bool trivial = x->len == 0 || x->zero_pending || y->zero_pending;
    int rc;
    if (!dist) {
        if (trivial) {
            B200_CUDA(cudaStreamSynchronize(ctx->stream));
            *result = 0.0;
            return B200_OK;
        }
        rc = x->dtype == B200_F64 ? launch_dot_kernel<double>(ctx, x, y, ctx->dot_result_d)
                                  : launch_dot_kernel<float>(ctx, x, y, ctx->dot_result_d);
        if (rc) return rc;
        B200_CUDA(cudaStreamSynchronize(ctx->stream));
        *result = *reinterpret_cast<volatile double *>(ctx->dot_result_h);
        return B200_OK;
    }
    // partitioned vectors: local partial -> device scalar -> all-reduce -> host
    // (mpi/inner_product.hpp:53-62 does the same with MPI_Allreduce on the host)
    if (trivial) {
        B200_CUDA(cudaMemsetAsync(ctx->dot_dev, 0, sizeof(double), ctx->stream));
    } else {
        rc = launch_dot_kernel<double>(ctx, x, y, ctx->dot_dev);
        if (rc) return rc;
    }
    return dist_dot_finish(ctx, result);
}
} // namespace b200

namespace b200 {
template <class T>
static int axpby_t(b200_ctx_t ctx, double a, b200_vec_t x, double b, b200_vec_t y) {
    const double *px;
    int rc = rd(x, &px);
    if (rc) return rc;
    if (b == 0.0 || y->zero_pending) {
        AxF<T> f{(T)a};
        return launch_ew<AxF<T>, false, false, T>(ctx, x->len, f, tp<T>(px), nullptr, nullptr, tp<T>(wr(y)));
    }
    AxpbyF<T> f{(T)a, (T)b};
    return launch_ew<AxpbyF<T>, true, false, T>(ctx, x->len, f, tp<T>(px), tp<T>(y->ptr), nullptr, tp<T>(mut(y)));
}
template <class T>
static int axpbypcz_t(b200_ctx_t ctx, double a, b200_vec_t x, double b, b200_vec_t y, double c, b200_vec_t z) {
    const double *px, *py;
    int rc = rd(x, &px);
    if (rc) return rc;
    rc = rd(y, &py);
    if (rc) return rc;
    if (c == 0.0 || z->zero_pending) {
        AxpbyF<T> f{(T)a, (T)b};
        return launch_ew<AxpbyF<T>, true, false, T>(ctx, x->len, f, tp<T>(px), tp<T>(py), nullptr, tp<T>(wr(z)));
    }
    AxpbypczF<T> f{(T)a, (T)b, (T)c};
    return launch_ew<AxpbypczF<T>, true, true, T>(ctx, x->len, f, tp<T>(px), tp<T>(py), tp<T>(z->ptr), tp<T>(mut(z)));
}
template <class T>
static int vmul_t(b200_ctx_t ctx, double alpha, b200_vec_t x, b200_vec_t y, double beta, b200_vec_t z) {
    const double *px, *py;
    int rc = rd(x, &px);
    if (rc) return rc;
    rc = rd(y, &py);
    if (rc) return rc;
    if (beta == 0.0 || z->zero_pending) {
        VmulF<T> f{(T)alpha};
        return launch_ew<VmulF<T>, true, false, T>(ctx, x->len, f, tp<T>(px), tp<T>(py), nullptr, tp<T>(wr(z)));
    }
    VmulAccF<T> f{(T)alpha, (T)beta};
    return launch_ew<VmulAccF<T>, true, true, T>(ctx, x->len, f, tp<T>(px), tp<T>(py), tp<T>(z->ptr), tp<T>(mut(z)));
}
} // namespace b200

extern "C" int b200_axpby(b200_ctx_t ctx, double a, b200_vec_t x, double b, b200_vec_t y) {
    CHECK_CTX(ctx);
    B200_REQUIRE(x && y, "null argument");
    touch(ctx, {x, y});
    B200_REQUIRE(same_layout(x, y), "axpby: size mismatch");
    GUARD(ctx);
    if (all64({x, y})) return axpby_t<double>(ctx, a, x, b, y);
    if (all32({x, y})) return axpby_t<float>(ctx, a, x, b, y);
    return B200_BAD_MIX("axpby");
}

extern "C" int b200_axpbypcz(b200_ctx_t ctx, double a, b200_vec_t x, double b, b200_vec_t y,
                             double c, b200_vec_t z) {
    CHECK_CTX(ctx);
    B200_REQUIRE(x && y && z, "null argument");
    touch(ctx, {x, y, z});
    B200_REQUIRE(same_layout(x, y) && same_layout(x, z), "axpbypcz: size mismatch");
    GUARD(ctx);
    if (all64({x, y, z})) return axpbypcz_t<double>(ctx, a, x, b, y, c, z);
    if (all32({x, y, z})) return axpbypcz_t<float>(ctx, a, x, b, y, c, z);
    return B200_BAD_MIX("axpbypcz");
}

extern "C" int b200_vmul(b200_ctx_t ctx, double alpha, b200_vec_t x, b200_vec_t y, double beta,
                         b200_vec_t z) {
    CHECK_CTX(ctx);
    B200_REQUIRE(x && y && z, "null argument");
    touch(ctx, {x, y, z});
    B200_REQUIRE(same_layout(x, y) && same_layout(x, z), "vmul: size mismatch");
    GUARD(ctx);
    if (all64({x, y, z})) return vmul_t<double>(ctx, alpha, x, y, beta, z);
    if (all32({x, y, z})) return vmul_t<float>(ctx, alpha, x, y, beta, z);
    if (all32({x, y}) && z->dtype == B200_F64) {
        // FP32 smoother diagonal and residual accumulated into an FP64 iterate
        const double *px, *py;
        int rc = rd(x, &px);
        if (rc) return rc;
        rc = rd(y, &py);
        if (rc) return rc;
        if (beta == 0.0 || z->zero_pending) {
            VmulF<double> f{alpha};
            return launch_ew_mixed<VmulF<double>, true, false>(ctx, x->len, f, tp<float>(px), tp<float>(py),
                                                               (const double *)nullptr, wr(z));
        }
        VmulAccF<double> f{alpha, beta};
        return launch_ew_mixed<VmulAccF<double>, true, true>(ctx, x->len, f, tp<float>(px), tp<float>(py),
                                                            (const double *)z->ptr, mut(z));
    }
    return B200_BAD_MIX("vmul");
}


// ---------------------------------------------------------------------------
// index lists: gather / scatter
// ---------------------------------------------------------------------------
extern "C" int b200_index_create_i64(b200_ctx_t ctx, const int64_t *idx, size_t n, size_t range,
                                     b200_index_t *out) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "index list creation");
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    B200_REQUIRE(idx != nullptr || n == 0, "null index array");
    B200_REQUIRE(!ctx->dist, "index lists are not supported on a distributed context");
    B200_REQUIRE(range < ((size_t)1 << 31), "index range must be below 2^31");
    std::vector<int> narrow(n);
    for (size_t k = 0; k < n; ++k) {
        if (idx[k] < 0 || (size_t)idx[k] >= range) return fail(B200_ERANGE, "index out of range");
        narrow[k] = (int)idx[k];
    }
    GUARD(ctx);
    b200_index_s *I = new (std::nothrow) b200_index_s();
    if (!I) return fail(B200_ENOMEM, "out of host memory");
    I->ctx = ctx; I->n = n; I->range = range;
    cudaError_t rc = cudaMalloc(&I->idx, (n + 4) * sizeof(int));
    if (rc == cudaSuccess) rc = cudaMalloc(&I->stage_d, (n + 4) * sizeof(double));
    if (rc == cudaSuccess && n)
        rc = cudaMemcpyAsync(I->idx, narrow.data(), n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream);
    if (rc == cudaSuccess) rc = cudaStreamSynchronize(ctx->stream);     // `narrow` dies here
    if (rc != cudaSuccess) {
        if (I->idx) cudaFree(I->idx);
        if (I->stage_d) cudaFree(I->stage_d);
        delete I;
        return cuda_fail(rc, "index list upload", __FILE__, __LINE__);
    }
    *out = I;
    return B200_OK;
}

extern "C" int b200_index_destroy(b200_index_t I) {
    if (!I) return B200_OK;
    NOT_RECORDING(I->ctx, "index list destruction");
    if (I->in_graph) I->ctx->destroy_epoch++;
    GUARD(I->ctx);
    if (I->idx) cudaFree(I->idx);
    if (I->stage_d) cudaFree(I->stage_d);
    delete I;
    return B200_OK;
}

extern "C" int b200_index_size(b200_index_t I, size_t *n) {
    B200_REQUIRE(I && n, "null argument");
    *n = I->n;
    return B200_OK;
}

namespace b200 {
template <class T>
static int gather_launch(b200_ctx_t ctx, b200_index_t I, const double *src, double *dst) {
    if (!I->n) return B200_OK;
    const int grid = grid_for(ctx, I->n, 2);
    ProfScope prof(ctx, B200_PROF_VECTOR + 1, (int64_t)I->n, 1, 0);
    B200_CUDA(launch_pdl(ctx, gather_kernel<T>, dim3(grid), dim3(kThreads), 0, I->n, (const int *)I->idx,
                         (const T *)tp<T>(src), tp<T>(dst)));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}
} // namespace b200

extern "C" int b200_gather(b200_ctx_t ctx, b200_index_t I, b200_vec_t src, b200_vec_t dst) {
    CHECK_CTX(ctx);
    B200_REQUIRE(I && src && dst, "null argument");
    touch(ctx, {src, dst});
    if (ctx->recording) I->in_graph = true;
    B200_REQUIRE(src->n == I->range && dst->n == I->n, "gather: vector sizes do not match the index list");
    B200_REQUIRE(src != dst && src->ptr != dst->ptr, "gather: src and dst must not alias");
    if (src->dtype != dst->dtype) return B200_BAD_MIX("gather");
    GUARD(ctx);
    const double *ps;
    int rc = rd(src, &ps);
    if (rc) return rc;
    return src->dtype == B200_F64 ? gather_launch<double>(ctx, I, ps, wr(dst))
                                  : gather_launch<float>(ctx, I, ps, wr(dst));
}

// gather into a host array (the reference's second overload, cuda.hpp:560-563): host-synchronous
extern "C" int b200_gather_host(b200_ctx_t ctx, b200_index_t I, b200_vec_t src, void *host) {
    CHECK_CTX(ctx);
    B200_REQUIRE(I && src && (host || I->n == 0), "null argument");
    NOT_RECORDING(ctx, "gather to the host");
    B200_REQUIRE(src->n == I->range, "gather: vector size does not match the index list");
    GUARD(ctx);
    if (!I->n) return B200_OK;
    const double *ps;
    int rc = rd(src, &ps);
    if (rc) return rc;
    rc = src->dtype == B200_F64 ? gather_launch<double>(ctx, I, ps, static_cast<double *>(I->stage_d))
                                : gather_launch<float>(ctx, I, ps, static_cast<double *>(I->stage_d));
    if (rc) return rc;
    B200_CUDA(cudaMemcpyAsync(host, I->stage_d, I->n * src->esz, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    return B200_OK;
}

extern "C" int b200_scatter(b200_ctx_t ctx, b200_index_t I, b200_vec_t src, b200_vec_t dst) {
    CHECK_CTX(ctx);
    B200_REQUIRE(I && src && dst, "null argument");
    touch(ctx, {src, dst});
    if (ctx->recording) I->in_graph = true;
    B200_REQUIRE(dst->n == I->range && src->n == I->n, "scatter: vector sizes do not match the index list");
    B200_REQUIRE(src != dst && src->ptr != dst->ptr, "scatter: src and dst must not alias");
    if (src->dtype != dst->dtype) return B200_BAD_MIX("scatter");
    GUARD(ctx);
    if (!I->n) return B200_OK;
    const double *ps, *pd;
    int rc = rd(src, &ps);
    if (rc) return rc;
    rc = rd(dst, &pd);                  // partial overwrite: a pending clear must land first
    if (rc) return rc;
    const int grid = grid_for(ctx, I->n, 2);
    ProfScope prof(ctx, B200_PROF_VECTOR + 1, (int64_t)I->n, 1, 0);
    if (src->dtype == B200_F64)
        B200_CUDA(launch_pdl(ctx, scatter_kernel<double>, dim3(grid), dim3(kThreads), 0, I->n,
                             (const int *)I->idx, ps, mut(dst)));
    else
        B200_CUDA(launch_pdl(ctx, scatter_kernel<float>, dim3(grid), dim3(kThreads), 0, I->n,
                             (const int *)I->idx, (const float *)tp<float>(ps), tp<float>(mut(dst))));
    B200_CHECK_LAUNCH();
    ctx->launches++;
    return B200_OK;
}
