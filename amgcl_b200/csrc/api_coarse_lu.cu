// api_coarse_lu.cu -- coarsest levels above the dense inverse's size: banded LU on the device
//
// Part of the implementation of the C ABI declared in include/amgcl_b200.h.  The symbolic
// phase (ordering, profile, tiles) runs on the host; the factorisation and both sweeps run on
// the device (coarse_lu.cuh).
#include "internal.cuh"
#include "coarse_lu.cuh"

using namespace b200;

namespace b200 {

// the symbolic phase: everything that depends on the pattern alone
struct LuPlan {
    int64_t n = 0, ntiles = 0;
    int bl = 0, bu = 0;                     // lower / upper bandwidth of the ordered matrix
    std::vector<int32_t> perm, iperm;       // perm[new] = old, iperm[old] = new
    std::vector<int32_t> lower, upper;      // per-row lower, per-column upper bandwidth
    std::vector<int64_t> lfirst, ulast;     // per tile: first / last tile its panels reach
    std::vector<int64_t> offL, offU;        // per tile: first chunk of its L / U panel
    size_t factor_bytes = 0, setup_bytes = 0;
};

struct CoarseLu {
    int64_t ntiles = 0;
    int bl = 0, bu = 0;
    int grid = 0;
    int64_t chunks = 0;                     // chunks one solve streams (panels + inverses)
    int *perm = nullptr;
    int64_t *offL = nullptr, *offU = nullptr;
    double *panL = nullptr, *panU = nullptr, *Linv = nullptr, *Uinv = nullptr, *z = nullptr;
    unsigned long long *sync = nullptr;     // [2 tickets | ntiles forward flags | ntiles backward]
};

// Reverse Cuthill-McKee of the symmetrised pattern: per connected component, breadth-first
// from a pseudo-peripheral vertex (repeated searches from a vertex of least degree in the
// last level), neighbours visited by increasing degree; then the whole order is reversed.
static void rcm_order(int64_t n, const std::vector<int64_t> &sptr, const std::vector<int32_t> &sadj,
                      std::vector<int32_t> &perm) {
    std::vector<int32_t> deg((size_t)n), level((size_t)n, -1), order, bfs, lv, nb;
    for (int64_t i = 0; i < n; ++i) deg[(size_t)i] = (int32_t)(sptr[(size_t)i + 1] - sptr[(size_t)i]);
    order.reserve((size_t)n);
    std::vector<char> done((size_t)n, 0);
    auto before = [&](int32_t a, int32_t b) {        // least degree first, then lower index
        return deg[(size_t)a] != deg[(size_t)b] ? deg[(size_t)a] < deg[(size_t)b] : a < b;
    };
    // breadth-first search of s's component: vertices in visit order (bfs) and their levels (lv)
    auto search = [&](int32_t s) {
        bfs.assign(1, s);
        lv.assign(1, 0);
        level[(size_t)s] = 0;
        for (size_t h = 0; h < bfs.size(); ++h) {
            const int32_t v = bfs[h];
            for (int64_t e = sptr[(size_t)v]; e < sptr[(size_t)v + 1]; ++e) {
                const int32_t w = sadj[(size_t)e];
                if (level[(size_t)w] < 0) {
                    level[(size_t)w] = lv[h] + 1;
                    bfs.push_back(w);
                    lv.push_back(lv[h] + 1);
                }
            }
        }
        for (int32_t v : bfs) level[(size_t)v] = -1;
    };
    for (int64_t s0 = 0; s0 < n; ++s0) {
        if (done[(size_t)s0]) continue;
        int32_t root = (int32_t)s0;
        search(root);
        for (int32_t v : bfs) if (before(v, root)) root = v;
        // pseudo-peripheral vertex: restart from a least-degree vertex of the last level while
        // the eccentricity grows
        int ecc = -1;
        for (int it = 0; it < 16; ++it) {
            search(root);
            if (lv.back() <= ecc) break;
            ecc = lv.back();
            int32_t best = -1;
            for (size_t h = 0; h < bfs.size(); ++h)
                if (lv[h] == ecc && (best < 0 || before(bfs[h], best))) best = bfs[h];
            if (best == root) break;
            root = best;
        }
        // Cuthill-McKee from root
        const size_t first = order.size();
        order.push_back(root);
        done[(size_t)root] = 1;
        for (size_t h = first; h < order.size(); ++h) {
            const int32_t v = order[h];
            nb.clear();
            for (int64_t e = sptr[(size_t)v]; e < sptr[(size_t)v + 1]; ++e) {
                const int32_t w = sadj[(size_t)e];
                if (!done[(size_t)w]) { done[(size_t)w] = 1; nb.push_back(w); }
            }
            std::sort(nb.begin(), nb.end(), before);
            order.insert(order.end(), nb.begin(), nb.end());
        }
    }
    perm.assign(order.rbegin(), order.rend());
}

// Symbolic phase for an n x n matrix with validated int32 indices.
template <class Ptr, class Col>
static int lu_plan(int64_t n, const Ptr *ptr, const Col *col, LuPlan &p) {
    if (n >= (int64_t)1 << 31) return fail(B200_ERANGE, "coarse solver: n does not fit int32");
    const int64_t nnz = (int64_t)ptr[n];
    p.n = n;
    // symmetrised pattern without the diagonal, duplicates removed
    std::vector<int64_t> cnt((size_t)n + 1, 0);
    for (int64_t i = 0; i < n; ++i)
        for (int64_t e = (int64_t)ptr[i]; e < (int64_t)ptr[i + 1]; ++e) {
            const int64_t j = (int64_t)col[e];
            if (j != i) { cnt[(size_t)i + 1]++; cnt[(size_t)j + 1]++; }
        }
    for (int64_t i = 0; i < n; ++i) cnt[(size_t)i + 1] += cnt[(size_t)i];
    std::vector<int32_t> adj((size_t)cnt[(size_t)n]);
    {
        std::vector<int64_t> pos(cnt.begin(), cnt.end() - 1);
        for (int64_t i = 0; i < n; ++i)
            for (int64_t e = (int64_t)ptr[i]; e < (int64_t)ptr[i + 1]; ++e) {
                const int64_t j = (int64_t)col[e];
                if (j != i) { adj[(size_t)pos[(size_t)i]++] = (int32_t)j; adj[(size_t)pos[(size_t)j]++] = (int32_t)i; }
            }
    }
    std::vector<int64_t> sptr((size_t)n + 1, 0);
    {
        int64_t w = 0;
        for (int64_t i = 0; i < n; ++i) {
            const auto b = adj.begin() + cnt[(size_t)i], e = adj.begin() + cnt[(size_t)i + 1];
            std::sort(b, e);
            const auto u = std::unique(b, e);
            for (auto it = b; it != u; ++it) adj[(size_t)w++] = *it;
            sptr[(size_t)i + 1] = w;
        }
        adj.resize((size_t)w);
    }
    rcm_order(n, sptr, adj, p.perm);
    p.iperm.assign((size_t)n, 0);
    for (int64_t r = 0; r < n; ++r) p.iperm[(size_t)p.perm[(size_t)r]] = (int32_t)r;
    // profile of the ordered matrix
    p.lower.assign((size_t)n, 0);
    p.upper.assign((size_t)n, 0);
    for (int64_t i = 0; i < n; ++i) {
        const int32_t r = p.iperm[(size_t)i];
        for (int64_t e = (int64_t)ptr[i]; e < (int64_t)ptr[i + 1]; ++e) {
            const int32_t c = p.iperm[(size_t)col[e]];
            if (c < r) p.lower[(size_t)r] = std::max(p.lower[(size_t)r], r - c);
            if (c > r) p.upper[(size_t)c] = std::max(p.upper[(size_t)c], c - r);
        }
    }
    p.bl = 0; p.bu = 0;
    for (int64_t i = 0; i < n; ++i) {
        p.bl = std::max(p.bl, p.lower[(size_t)i]);
        p.bu = std::max(p.bu, p.upper[(size_t)i]);
    }
    // tiles: L panel of tile k from the first column its rows reach; U panel of tile k up to the
    // last column whose first row (c - upper[c]) lies in tile k or before
    const int64_t T = kLuTile;
    p.ntiles = (n + T - 1) / T;
    p.lfirst.assign((size_t)p.ntiles, 0);
    p.ulast.assign((size_t)p.ntiles, 0);
    std::vector<int64_t> reach((size_t)p.ntiles, -1);
    for (int64_t k = 0; k < p.ntiles; ++k) {
        int64_t f = k * T;
        for (int64_t r = k * T; r < std::min(n, (k + 1) * T); ++r) f = std::min(f, r - p.lower[(size_t)r]);
        p.lfirst[(size_t)k] = f / T;
    }
    for (int64_t c = 0; c < n; ++c) {
        const int64_t g = (c - p.upper[(size_t)c]) / T;
        reach[(size_t)g] = std::max(reach[(size_t)g], c / T);
    }
    int64_t m = -1;
    for (int64_t k = 0; k < p.ntiles; ++k) {
        m = std::max(m, reach[(size_t)k]);
        p.ulast[(size_t)k] = std::max(m, k);
    }
    p.offL.assign((size_t)p.ntiles + 1, 0);
    p.offU.assign((size_t)p.ntiles + 1, 0);
    for (int64_t k = 0; k < p.ntiles; ++k) {
        p.offL[(size_t)k + 1] = p.offL[(size_t)k] + (k - p.lfirst[(size_t)k]);
        p.offU[(size_t)k + 1] = p.offU[(size_t)k] + (p.ulast[(size_t)k] - k);
    }
    const size_t chunk = (size_t)kLuChunk * sizeof(double);
    p.factor_bytes = (size_t)(p.offL[(size_t)p.ntiles] + p.offU[(size_t)p.ntiles] + 2 * p.ntiles) * chunk +
                     (size_t)n * sizeof(int) + 2 * ((size_t)p.ntiles + 1) * sizeof(int64_t) +
                     (size_t)p.ntiles * T * sizeof(double) + (2 + 2 * (size_t)p.ntiles) * sizeof(unsigned long long);
    p.setup_bytes = (size_t)n * ((size_t)p.bl + p.bu + 1) * sizeof(double) +
                    ((size_t)n + 1 + (size_t)nnz + (size_t)n) * sizeof(int) + (size_t)nnz * sizeof(double);
    return B200_OK;
}

void coarse_lu_destroy(CoarseLu *L) {
    if (!L) return;
    cudaFree(L->perm); cudaFree(L->offL); cudaFree(L->offU); cudaFree(L->panL); cudaFree(L->panU);
    cudaFree(L->Linv); cudaFree(L->Uinv); cudaFree(L->z); cudaFree(L->sync);
    delete L;
}

int coarse_lu_create(b200_ctx_t ctx, int64_t n, const std::vector<int32_t> &hptr,
                     const std::vector<int32_t> &hcol, const std::vector<double> &hval,
                     b200_coarse_s *S) {
    LuPlan p;
    int rc = lu_plan(n, hptr.data(), hcol.data(), p);
    if (rc) return rc;
    size_t free_b = 0, total_b = 0;
    B200_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (p.factor_bytes + p.setup_bytes > free_b)
        return fail(B200_ENOMEM, "coarse solver: the banded LU factor of this level needs " +
                                     std::to_string((p.factor_bytes + p.setup_bytes) >> 20) +
                                     " MiB of device memory (bandwidth " + std::to_string(std::max(p.bl, p.bu)) +
                                     " after reordering), " + std::to_string(free_b >> 20) + " MiB are free");
    const int N = (int)n, W = p.bl + p.bu + 1;
    const int64_t nnz = (int64_t)hptr[(size_t)n];
    CoarseLu *L = new (std::nothrow) CoarseLu();
    if (!L) return fail(B200_ENOMEM, "out of host memory");
    L->ntiles = p.ntiles; L->bl = p.bl; L->bu = p.bu;
    L->chunks = p.offL[(size_t)p.ntiles] + p.offU[(size_t)p.ntiles] + 2 * p.ntiles;
    int *dptr = nullptr, *dcol = nullptr, *diperm = nullptr;
    double *dval = nullptr, *B = nullptr;
    auto scratch_free = [&]() { cudaFree(dptr); cudaFree(dcol); cudaFree(diperm); cudaFree(dval); cudaFree(B); };
#define LU_CUDA(call)                                                          \
    do {                                                                       \
        cudaError_t rc__ = (call);                                             \
        if (rc__ != cudaSuccess) {                                             \
            scratch_free();                                                    \
            coarse_lu_destroy(L);                                              \
            return cuda_fail(rc__, #call, __FILE__, __LINE__);                 \
        }                                                                      \
    } while (0)
    const size_t chunk = (size_t)kLuChunk * sizeof(double);
    const size_t Bbytes = (size_t)N * W * sizeof(double);
    const int64_t T = p.ntiles;
    LU_CUDA(cudaMalloc(&dptr, ((size_t)N + 1) * sizeof(int)));
    LU_CUDA(cudaMalloc(&dcol, std::max<size_t>(1, (size_t)nnz) * sizeof(int)));
    LU_CUDA(cudaMalloc(&dval, std::max<size_t>(1, (size_t)nnz) * sizeof(double)));
    LU_CUDA(cudaMalloc(&diperm, (size_t)N * sizeof(int)));
    LU_CUDA(cudaMalloc(&B, Bbytes));
    LU_CUDA(cudaMalloc(&L->perm, (size_t)N * sizeof(int)));
    LU_CUDA(cudaMalloc(&L->offL, ((size_t)T + 1) * sizeof(int64_t)));
    LU_CUDA(cudaMalloc(&L->offU, ((size_t)T + 1) * sizeof(int64_t)));
    LU_CUDA(cudaMalloc(&L->panL, std::max<size_t>(1, (size_t)p.offL[(size_t)T]) * chunk));
    LU_CUDA(cudaMalloc(&L->panU, std::max<size_t>(1, (size_t)p.offU[(size_t)T]) * chunk));
    LU_CUDA(cudaMalloc(&L->Linv, (size_t)T * chunk));
    LU_CUDA(cudaMalloc(&L->Uinv, (size_t)T * chunk));
    LU_CUDA(cudaMalloc(&L->z, (size_t)T * kLuTile * sizeof(double)));
    LU_CUDA(cudaMalloc(&L->sync, (2 + 2 * (size_t)T) * sizeof(unsigned long long)));
    cudaStream_t st = ctx->stream;
    LU_CUDA(cudaMemcpyAsync(dptr, hptr.data(), ((size_t)N + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
    if (nnz) {
        LU_CUDA(cudaMemcpyAsync(dcol, hcol.data(), (size_t)nnz * sizeof(int), cudaMemcpyHostToDevice, st));
        LU_CUDA(cudaMemcpyAsync(dval, hval.data(), (size_t)nnz * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    LU_CUDA(cudaMemcpyAsync(diperm, p.iperm.data(), (size_t)N * sizeof(int), cudaMemcpyHostToDevice, st));
    LU_CUDA(cudaMemcpyAsync(L->perm, p.perm.data(), (size_t)N * sizeof(int), cudaMemcpyHostToDevice, st));
    LU_CUDA(cudaMemcpyAsync(L->offL, p.offL.data(), ((size_t)T + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    LU_CUDA(cudaMemcpyAsync(L->offU, p.offU.data(), ((size_t)T + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    LU_CUDA(cudaMemsetAsync(L->sync, 0, (2 + 2 * (size_t)T) * sizeof(unsigned long long), st));
    LU_CUDA(cudaMemsetAsync(B, 0, Bbytes, st));
    lu_scatter_kernel<<<(N + 127) / 128, 128, 0, st>>>(N, p.bl, W, dptr, dcol, dval, diperm, B);
    LU_CUDA(cudaGetLastError());
    ctx->launches++;
    // right-looking elimination, one launch per pivot column
    const dim3 sblk(32, 8);
    for (int k = 0; k + 1 < N; ++k) {
        const int nc = std::min(p.bu, N - 1 - k), nr = std::min(p.bl, N - 1 - k);
        if (nc <= 0 || nr <= 0) continue;
        lu_step_kernel<<<dim3((nc + 31) / 32, (nr + 7) / 8), sblk, 0, st>>>(N, k, p.bl, p.bu, W, B);
        ctx->launches++;
    }
    LU_CUDA(cudaGetLastError());
    if (p.bl > 0) {
        const size_t tot = (size_t)N * p.bl;
        lu_scale_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(N, p.bl, W, B);
        LU_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    // pivots back to the host for the singularity test
    std::vector<double> hpiv((size_t)N);
    LU_CUDA(cudaMemcpy2DAsync(hpiv.data(), sizeof(double), B + p.bl, (size_t)W * sizeof(double),
                              sizeof(double), (size_t)N, cudaMemcpyDeviceToHost, st));
    lu_panels_kernel<<<dim3((unsigned)T, 2), 256, 0, st>>>(N, p.bl, p.bu, W, B, L->offL, L->offU,
                                                          L->panL, L->panU);
    LU_CUDA(cudaGetLastError());
    const size_t dsm = 2 * chunk;
    LU_CUDA(cudaFuncSetAttribute(lu_diag_inverse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm));
    lu_diag_inverse_kernel<<<(unsigned)T, kLuTile, dsm, st>>>(N, p.bl, p.bu, W, B, L->Linv, L->Uinv);
    LU_CUDA(cudaGetLastError());
    ctx->launches += 2;
    LU_CUDA(cudaStreamSynchronize(st));
#undef LU_CUDA
    scratch_free();
    double pmax = 0.0, pmin = std::numeric_limits<double>::infinity();
    for (double v : hpiv) {
        const double a = std::fabs(v);
        if (!(a == a)) { pmin = 0.0; break; }   // NaN
        pmax = std::max(pmax, a);
        pmin = std::min(pmin, a);
    }
    if (!(pmin > 0.0) || pmin < pmax * 1e-14 || !std::isfinite(pmax)) {
        coarse_lu_destroy(L);
        return fail(B200_ESINGULAR, "coarse matrix is numerically singular (or has a zero pivot "
                                    "without pivoting)");
    }
    cudaError_t e = cudaSuccess;
    auto smem = [&](auto kernel) {
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLuSweepSmem);
    };
    smem(coarse_lu_sweep_kernel<double, false>);
    smem(coarse_lu_sweep_kernel<double, true>);
    smem(coarse_lu_sweep_kernel<float, false>);
    smem(coarse_lu_sweep_kernel<float, true>);
    if (e != cudaSuccess) {
        coarse_lu_destroy(L);
        return cuda_fail(e, "cudaFuncSetAttribute(coarse_lu_sweep_kernel)", __FILE__, __LINE__);
    }
    L->grid = (int)std::min<int64_t>(T, (int64_t)ctx->sm_count * kLuCtasPerSm);
    S->kind = B200_COARSE_BANDED_LU;
    S->lu = L;
    S->bytes = p.factor_bytes;
    return B200_OK;
}

template <class T>
static int lu_sweeps(b200_ctx_t ctx, CoarseLu *L, int N, const T *rhs, T *x) {
    LuSweepArgs a;
    a.n = N; a.ntiles = (int)L->ntiles; a.perm = L->perm; a.z = L->z;
    a.pan = L->panL; a.off = L->offL; a.dinv = L->Linv; a.ticket = L->sync; a.flags = L->sync + 2;
    B200_CUDA(launch_pdl(ctx, coarse_lu_sweep_kernel<T, false>, dim3(L->grid), dim3(kLuThreads),
                         kLuSweepSmem, a, rhs, (T *)nullptr));
    B200_CHECK_LAUNCH();
    a.pan = L->panU; a.off = L->offU; a.dinv = L->Uinv; a.ticket = L->sync + 1; a.flags = L->sync + 2 + L->ntiles;
    B200_CUDA(launch_pdl(ctx, coarse_lu_sweep_kernel<T, true>, dim3(L->grid), dim3(kLuThreads),
                         kLuSweepSmem, a, (const T *)nullptr, x));
    B200_CHECK_LAUNCH();
    ctx->launches += 2;
    return B200_OK;
}

int coarse_lu_solve(b200_ctx_t ctx, b200_coarse_s *S, b200_vec_t rhs, b200_vec_t x) {
    CoarseLu *L = S->lu;
    const double *pr;
    int rc = rd(rhs, &pr);
    if (rc) return rc;
    if ((rc = tail_flush(ctx))) return rc;
    ProfScope prof(ctx, B200_PROF_COARSE_LU, S->n, S->n, L->chunks * kLuChunk);
    if (rhs->dtype == B200_F32) return lu_sweeps<float>(ctx, L, (int)S->n, tp<float>(pr), tp<float>(wr(x)));
    return lu_sweeps<double>(ctx, L, (int)S->n, pr, wr(x));
}

} // namespace b200

extern "C" int b200_coarse_lu_plan_i64(int64_t n, const int64_t *ptr, const int64_t *col, int32_t *perm_out,
                                       int32_t *lower_out, int32_t *upper_out, int64_t *lfirst_out,
                                       int64_t *ulast_out, int64_t tiles_capacity, int64_t *tiles,
                                       int *tile_rows, int64_t *bandwidth, size_t *factor_bytes,
                                       size_t *setup_bytes) {
    B200_REQUIRE(n > 0 && ptr && ptr[0] == 0, "bad row pointer array");
    B200_REQUIRE(ptr[n] == 0 || col, "bad column array");
    for (int64_t i = 0; i < n; ++i) B200_REQUIRE(ptr[i + 1] >= ptr[i], "bad row pointer array");
    for (int64_t e = 0; e < ptr[n]; ++e) B200_REQUIRE(col[e] >= 0 && col[e] < n, "column index out of range");
    LuPlan p;
    const int rc = lu_plan(n, ptr, col, p);
    if (rc) return rc;
    if (perm_out) std::copy(p.perm.begin(), p.perm.end(), perm_out);
    if (lower_out) std::copy(p.lower.begin(), p.lower.end(), lower_out);
    if (upper_out) std::copy(p.upper.begin(), p.upper.end(), upper_out);
    if (lfirst_out || ulast_out) {
        B200_REQUIRE(tiles_capacity >= p.ntiles, "tile arrays too small");
        if (lfirst_out) std::copy(p.lfirst.begin(), p.lfirst.end(), lfirst_out);
        if (ulast_out) std::copy(p.ulast.begin(), p.ulast.end(), ulast_out);
    }
    if (tiles) *tiles = p.ntiles;
    if (tile_rows) *tile_rows = kLuTile;
    if (bandwidth) *bandwidth = std::max(p.bl, p.bu);
    if (factor_bytes) *factor_bytes = p.factor_bytes;
    if (setup_bytes) *setup_bytes = p.setup_bytes;
    return B200_OK;
}

extern "C" int b200_coarse_info(b200_coarse_t S, int *kind, int64_t *n, int64_t *bandwidth, int64_t *tiles) {
    B200_REQUIRE(S, "null argument");
    if (kind) *kind = S->kind;
    if (n) *n = S->n;
    if (bandwidth) *bandwidth = S->lu ? std::max(S->lu->bl, S->lu->bu) : 0;
    if (tiles) *tiles = S->lu ? S->lu->ntiles : 0;
    return B200_OK;
}
