// coarse_lu.cuh -- banded LU of the coarsest level, for levels too large for the dense inverse.
//
// The matrix arrives ordered by reverse Cuthill-McKee (api_coarse_lu.cu) and is factored
// without pivoting, like solver::skyline_lu, in a dense band of width bl + bu + 1 (row i keeps
// columns [i - bl, i + bu] at B[i * W + (j - i + bl)]).  The solve reads a tiled copy of the
// factor: the rows are cut into tiles of kLuTile rows; tile k keeps
//   * its L panel: the columns of the earlier tiles its rows reach, as kLuTile x kLuTile chunks,
//   * its U panel: the columns of the later tiles its rows reach, likewise,
//   * the inverses of its diagonal blocks of L (unit lower) and U,
// so a sweep never substitutes inside a tile: y_k = Linv_kk (b_k - sum_d L_kd y_d) and
// x_k = Uinv_kk (y_k - sum_d U_kd x_d).  DESIGN.md section 3.5 has the schedule and its
// progress argument.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kLuTile    = 64;                                  // rows per tile
constexpr int kLuChunk   = kLuTile * kLuTile;                   // doubles per chunk
constexpr int kLuThreads = 256;                                 // 8 warps x 8 rows per tile
constexpr int kLuRowsPerWarp = kLuTile / (kLuThreads / 32);
constexpr uint32_t kLuChunkBytes = kLuChunk * sizeof(double);
constexpr int kLuCtasPerSm = 1;                                // sweep grid: CTAs per SM
constexpr size_t kLuSweepSmem = 2 * (size_t)kLuChunkBytes;      // near chunk + diagonal inverse

// ---- numeric factorisation --------------------------------------------------------------------

// B[iperm[i]][iperm[col]] += val for every entry of row i (one thread per row: duplicates are
// summed in entry order)
__global__ void lu_scatter_kernel(int n, int bl, int W, const int *__restrict__ ptr,
                                  const int *__restrict__ col, const double *__restrict__ val,
                                  const int *__restrict__ iperm, double *B) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = iperm[i];
    double *row = B + (size_t)r * W + bl - r;
    for (int e = ptr[i]; e < ptr[i + 1]; ++e) row[iperm[col[e]]] += val[e];
}

// Elimination step k: B[i][j] -= (B[i][k] / B[k][k]) * B[k][j] for i in (k, k + bl],
// j in (k, k + bu].  Column k is only read here and is scaled into multipliers once at the
// end (lu_scale_kernel), so no thread of this launch reads what another one writes.
__global__ void __launch_bounds__(256)
lu_step_kernel(int n, int k, int bl, int bu, int W, double *B) {
    const int j = k + 1 + blockIdx.x * blockDim.x + threadIdx.x;
    const int i = k + 1 + blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= n || j >= n || i > k + bl || j > k + bu) return;
    const double a = B[(size_t)i * W + (k - i + bl)];
    if (a == 0.0) return;
    const double l = a / B[(size_t)k * W + bl];
    const double u = B[(size_t)k * W + (j - k + bl)];
    if (u == 0.0) return;
    double *p = B + (size_t)i * W + (j - i + bl);
    *p = fma(-l, u, *p);
}

// the strictly lower band becomes the multipliers: B[i][j] /= B[j][j]
__global__ void lu_scale_kernel(int n, int bl, int W, double *B) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)n * bl) return;
    const int i = (int)(idx / bl);
    const int j = i - bl + (int)(idx % bl);
    if (j < 0) return;
    double *p = B + (size_t)i * W + (j - i + bl);
    if (*p != 0.0) *p /= B[(size_t)j * W + bl];
}

// copy the factor out of the band into the tiled panels (one CTA per tile and triangle):
// chunk c of tile k covers the columns of tile d = dep(k, c); rows and columns past n are 0
__global__ void __launch_bounds__(256)
lu_panels_kernel(int n, int bl, int bu, int W, const double *__restrict__ B,
                 const int64_t *__restrict__ offL, const int64_t *__restrict__ offU,
                 double *panL, double *panU) {
    const int k = blockIdx.x;
    const bool upper = blockIdx.y == 1;
    const int64_t *off = upper ? offU : offL;
    double *pan = upper ? panU : panL;
    const int64_t c0 = off[k], nd = off[k + 1] - c0;
    for (int64_t c = 0; c < nd; ++c) {
        // consumption order: farthest tile first (see coarse_lu_sweep_kernel)
        const int d = upper ? (int)(k + nd - c) : (int)(k - nd + c);
        double *dst = pan + (size_t)(c0 + c) * kLuChunk;
        for (int e = threadIdx.x; e < kLuChunk; e += blockDim.x) {
            const int i = k * kLuTile + e / kLuTile, j = d * kLuTile + e % kLuTile;
            const int o = j - i;
            const bool in = i < n && j < n && (upper ? o <= bu : -o <= bl);
            dst[e] = in ? B[(size_t)i * W + (o + bl)] : 0.0;
        }
    }
}

// Inverses of the diagonal blocks of tile k (one CTA of kLuTile threads per tile; thread c
// forms column c of each inverse by substitution).  Rows past n are identity rows.
__global__ void __launch_bounds__(kLuTile)
lu_diag_inverse_kernel(int n, int bl, int bu, int W, const double *__restrict__ B,
                       double *Linv, double *Uinv) {
    extern __shared__ __align__(128) double lu_sm[];
    double *A = lu_sm;                       // [kLuTile][kLuTile] diagonal block of the factor
    double *Z = lu_sm + kLuChunk;            // [r][c]: column c of the inverse being formed
    const int k = blockIdx.x, c = threadIdx.x, r0 = k * kLuTile;
    for (int e = threadIdx.x; e < kLuChunk; e += blockDim.x) {
        const int i = r0 + e / kLuTile, j = r0 + e % kLuTile, o = j - i;
        double v;
        if (i >= n || j >= n) v = (i == j) ? 1.0 : 0.0;
        else v = (o <= bu && -o <= bl) ? B[(size_t)i * W + (o + bl)] : 0.0;
        A[e] = v;
    }
    __syncthreads();
    // L (unit lower): z_r = [r == c] - sum_{m < r} L[r][m] z_m
    for (int r = 0; r < kLuTile; ++r) {
        double s = (r == c) ? 1.0 : 0.0;
        for (int m = c; m < r; ++m) s = fma(-A[r * kLuTile + m], Z[m * kLuTile + c], s);
        Z[r * kLuTile + c] = (r < c) ? 0.0 : s;
    }
    double *Lk = Linv + (size_t)k * kLuChunk;
    for (int r = 0; r < kLuTile; ++r) Lk[r * kLuTile + c] = Z[r * kLuTile + c];
    // U: z_r = ([r == c] - sum_{m > r} U[r][m] z_m) / U[r][r]
    for (int r = kLuTile - 1; r >= 0; --r) {
        double s = (r == c) ? 1.0 : 0.0;
        for (int m = r + 1; m <= c; ++m) s = fma(-A[r * kLuTile + m], Z[m * kLuTile + c], s);
        Z[r * kLuTile + c] = (r > c) ? 0.0 : s / A[r * kLuTile + r];
    }
    double *Uk = Uinv + (size_t)k * kLuChunk;
    for (int r = 0; r < kLuTile; ++r) Uk[r * kLuTile + c] = Z[r * kLuTile + c];
}

// ---- the sweeps ------------------------------------------------------------------------------

struct LuSweepArgs {
    int n, ntiles;
    const double  *pan;          // chunks of every tile's panel, tile after tile
    const int64_t *off;          // [ntiles + 1] first chunk of each tile
    const double  *dinv;         // [ntiles][kLuTile][kLuTile] diagonal-block inverses
    const int     *perm;         // perm[new] = old
    double        *z;            // [ntiles * kLuTile] y after the forward sweep, x after the backward
    unsigned long long *flags;   // [ntiles] tile k done in epoch e <=> flags[k] >= e + 1
    unsigned long long *ticket;  // claims so far, over all launches
};

__device__ __forceinline__ unsigned long long lu_ld_acquire(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void lu_st_release(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// z is written by other CTAs of the same launch: read it from L2, never from a stale L1 line
__device__ __forceinline__ double2 lu_ld_cg2(const double *p) {
    return __ldcg(reinterpret_cast<const double2 *>(p));
}

// One sweep as a persistent kernel.  Every CTA claims tickets from a counter that is never
// reset: launch e hands out tickets [e * (ntiles + G), (e + 1) * (ntiles + G)) for a grid of G
// CTAs -- one per tile, in sweep order, and one more per CTA, which tells it to exit.  So the
// epoch e is the ticket divided by ntiles + G, and nothing per call comes from the host: the
// launch records into a CUDA graph and replays.  A tile waits only on tiles with smaller
// tickets, which CTAs that are already running hold, so the sweep needs neither a cooperative
// launch nor a grid barrier.
//
// Per tile: the diagonal-block inverse and the nearest panel chunk (the one on the critical
// path) are copied to shared memory by TMA while the farther chunks stream from HBM; warp w
// accumulates rows 8w..8w+7, lane l columns 2l, 2l+1 of every chunk, in FP64, chunks in
// consumption order (farthest tile first), then the lanes are summed by a butterfly.
template <class T, bool kBackward>
__global__ void __launch_bounds__(kLuThreads)
coarse_lu_sweep_kernel(LuSweepArgs a, const T *__restrict__ rhs, T *__restrict__ x) {
    extern __shared__ __align__(128) double lu_sm[];
    double *sNear = lu_sm;
    double *sD = lu_sm + kLuChunk;
    __shared__ double sV[kLuTile];
    __shared__ unsigned long long sTicket;
    __shared__ __align__(8) uint64_t bar;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rw = warp * kLuRowsPerWarp;       // first row of this warp inside the tile
    ptx::pdl_wait();
    if (tid == 0) {
        ptx::mbar_init(&bar, 1);
        ptx::fence_mbar_init();
    }
    uint32_t phase = 0;
    const unsigned long long per = (unsigned long long)a.ntiles + gridDim.x;
    for (;;) {
        if (tid == 0) sTicket = atomicAdd(a.ticket, 1ull);
        __syncthreads();
        const unsigned long long tk = sTicket;
        const unsigned long long done = tk / per + 1;         // flag value of this epoch
        const int loc = (int)(tk % per);
        if (loc >= a.ntiles) break;
        const int k = kBackward ? a.ntiles - 1 - loc : loc;
        const int64_t c0 = a.off[k];
        const int nd = (int)(a.off[k + 1] - c0);
        if (tid == 0) {
            ptx::fence_proxy_async();                         // shared memory reads of the last tile
            ptx::mbar_expect_tx(&bar, (nd ? 2u : 1u) * kLuChunkBytes);
            ptx::bulk_g2s(sD, a.dinv + (size_t)k * kLuChunk, kLuChunkBytes, &bar);
            if (nd) ptx::bulk_g2s(sNear, a.pan + (size_t)(c0 + nd - 1) * kLuChunk, kLuChunkBytes, &bar);
        }
        // this tile's right-hand side, loaded before any wait: it is off the critical path
        double b = 0.0;
        if (lane < kLuRowsPerWarp) {
            const int row = k * kLuTile + rw + lane;
            if (kBackward) b = __ldcg(a.z + row);
            else if (row < a.n) b = (double)rhs[a.perm[row]];
        }
        double acc[kLuRowsPerWarp];
#pragma unroll
        for (int r = 0; r < kLuRowsPerWarp; ++r) acc[r] = 0.0;
        for (int c = 0; c < nd; ++c) {
            const int d = kBackward ? k + nd - c : k - nd + c;
            if (tid == 0)
                while (lu_ld_acquire(a.flags + d) < done) {}
            __syncthreads();
            const double2 y = lu_ld_cg2(a.z + (size_t)d * kLuTile + 2 * lane);
            if (c + 1 < nd) {
                const double *ch = a.pan + (size_t)(c0 + c) * kLuChunk + 2 * lane;
                double2 v[kLuRowsPerWarp];
#pragma unroll
                for (int r = 0; r < kLuRowsPerWarp; ++r) v[r] = ptx::ld_stream2(ch + (rw + r) * kLuTile);
#pragma unroll
                for (int r = 0; r < kLuRowsPerWarp; ++r) acc[r] = fma(v[r].y, y.y, fma(v[r].x, y.x, acc[r]));
            } else {
                ptx::mbar_wait(&bar, phase);
#pragma unroll
                for (int r = 0; r < kLuRowsPerWarp; ++r) {
                    const double2 v = *reinterpret_cast<const double2 *>(sNear + (rw + r) * kLuTile + 2 * lane);
                    acc[r] = fma(v.y, y.y, fma(v.x, y.x, acc[r]));
                }
            }
        }
#pragma unroll
        for (int r = 0; r < kLuRowsPerWarp; ++r)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
        if (lane < kLuRowsPerWarp) {
            double s = acc[0];
#pragma unroll
            for (int r = 1; r < kLuRowsPerWarp; ++r) if (lane == r) s = acc[r];
            sV[rw + lane] = b - s;
        }
        if (nd == 0) ptx::mbar_wait(&bar, phase);
        phase ^= 1;
        __syncthreads();
        // diagonal block: v = Dinv_kk * sV
        const double2 sv = *reinterpret_cast<const double2 *>(sV + 2 * lane);
#pragma unroll
        for (int r = 0; r < kLuRowsPerWarp; ++r) {
            const double2 dv = *reinterpret_cast<const double2 *>(sD + (rw + r) * kLuTile + 2 * lane);
            acc[r] = fma(dv.y, sv.y, dv.x * sv.x);
        }
#pragma unroll
        for (int r = 0; r < kLuRowsPerWarp; ++r)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
        if (lane < kLuRowsPerWarp) {
            const int row = k * kLuTile + rw + lane;
            double v = acc[0];
#pragma unroll
            for (int r = 1; r < kLuRowsPerWarp; ++r) if (lane == r) v = acc[r];
            a.z[row] = v;
            if (kBackward && row < a.n) x[a.perm[row]] = (T)v;
        }
        __syncthreads();
        // the release is cumulative: it publishes every store of the CTA ordered before it by
        // the barrier
        if (tid == 0) lu_st_release(a.flags + k, done);
    }
}

} // namespace b200
