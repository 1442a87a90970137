// tail_kernels.cuh -- the coarse tail of the V-cycle as ONE kernel.
//
// amg::cycle (amg.hpp:514-553) issues ~5 backend calls per level; on the coarse levels each of
// them is a kernel that does 1-3 us of work but sits behind a dependent-launch gap of several
// microseconds, so at 256^3 the levels below 10^5 rows cost ~14 launches per cycle, and at 64^3
// they ARE the cycle.  AMGCL's host control flow stays unmodified: the C ABI DEFERS calls whose
// operator is small (api_tail.cu) into a command list and, as soon as a call that cannot be
// deferred arrives, runs the whole list as one persistent kernel -- one 1024-thread CTA per SM,
// commands separated by a device-wide barrier instead of a kernel boundary.
//
// What makes a command cheap here:
//   * the barrier is one red.release + a spin on ld.acquire of a monotonically increasing
//     64-bit counter (no reset, no fences): one per SM;
//   * matrix data is written by nobody, so BEFORE arriving at the barrier every thread already
//     loads the row pointers of its first row of the NEXT command and prefetches that row's
//     first col/val lines into L1: after the barrier only the dependent x-gather is left;
//   * gathers are issued four at a time per lane (memory-level parallelism), FMAs in entry order.
//
// Bit-compatibility: every command evaluates exactly the arithmetic of the stand-alone kernel
// it replaces -- same lanes per row, same per-lane entry order, same shuffle tree, same
// epilogue (csr_kernels.cuh: compute_staged / store_row; relax_zero_kernel;
// coarse_kernels.cuh: coarse_gemv_kernel) -- so a solve with and without the tail kernel gives
// the same bits (tests/test_gpu_solver.py::test_coarse_tail_is_bit_transparent).
//
// Memory model: vectors written by one command are read by later commands of the same kernel
// on other SMs, so vector reads go to L2 (ld.global.cg); only data no command writes (matrix
// arrays, smoother diagonal, dense inverse) use the read-only path / L1.
#pragma once
#include "common.cuh"
#include "csr_kernels.cuh"

namespace b200 {

enum { TAIL_CSR = 0, TAIL_RELAX_ZERO = 1, TAIL_GEMV = 2 };
constexpr int kTailMaxCmds = 28;
constexpr int kTailThreads = 1024;

struct TailCmd {
    int           op;       // TAIL_*
    int           mode;     // TAIL_CSR: MODE_*
    int           nrows;    // rows / vector length / dense dimension
    int           lanes;    // TAIL_CSR: lanes per row
    const int    *ptr;
    const int    *col;
    const double *val;      // TAIL_GEMV: dense inverse, row-major
    const double *x;        // gathered vector / GEMV right-hand side
    const double *f;
    const double *d;
    double       *y;
    double        alpha, beta;
};

struct TailArgs {
    int                 n;
    unsigned long long *bar;      // monotonically increasing arrival counter
    unsigned long long  bar_base; // its value when this kernel starts (host bookkeeping)
    TailCmd             cmd[kTailMaxCmds];
};

// device-wide barrier #k of this kernel (all CTAs are co-resident: cooperative launch)
__device__ __forceinline__ void tail_barrier(unsigned long long *bar, unsigned long long target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(bar) : "memory");
        unsigned long long v;
        do {
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
        } while (v < target);
    }
    __syncthreads();
}

__device__ __forceinline__ void tail_prefetch_l1(const void *p) {
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
}

struct TailRow { int beg, end; };      // row pointers of a thread's first row, loaded early

// before the barrier: row pointers of my first row of command c, its first lines into L1
template <int L, int THREADS = kTailThreads>
__device__ __forceinline__ TailRow tail_csr_peek(const TailCmd &c) {
    TailRow t = {0, 0};
    const int r = (blockIdx.x * THREADS + threadIdx.x) / L;
    if (r < c.nrows) {
        t.beg = __ldg(c.ptr + r);
        t.end = __ldg(c.ptr + r + 1);
        const int e = t.beg + (int)(threadIdx.x % L);
        if (e < t.end) {
            tail_prefetch_l1(c.col + e);
            tail_prefetch_l1(c.val + e);
        }
    }
    return t;
}
__device__ __forceinline__ TailRow tail_peek(const TailCmd &c) {
    if (c.op != TAIL_CSR) return TailRow{0, 0};
    switch (c.lanes) {
    case 1:  return tail_csr_peek<1>(c);
    case 2:  return tail_csr_peek<2>(c);
    case 4:  return tail_csr_peek<4>(c);
    case 8:  return tail_csr_peek<8>(c);
    case 16: return tail_csr_peek<16>(c);
    default: return tail_csr_peek<32>(c);
    }
}

// one CSR pass, L lanes per row: the arithmetic of compute_staged<MODE, L> + store_row<MODE>
template <int L, int THREADS = kTailThreads>
__device__ __forceinline__ void tail_csr(const TailCmd &c, const TailRow &first) {
    constexpr int U = 4;
    const int gid     = (blockIdx.x * THREADS + threadIdx.x) / L;
    const int lane    = threadIdx.x % L;
    const int ngroups = gridDim.x * THREADS / L;
    for (int base = 0; base < c.nrows; base += ngroups) {
        const int  r     = base + gid;
        const bool valid = r < c.nrows;
        double sum = 0.0;
        if (valid) {
            const int beg = base ? __ldg(c.ptr + r) : first.beg;
            const int end = base ? __ldg(c.ptr + r + 1) : first.end;
            int e = beg + lane;
            if (L >= 16) {
                // wide groups: the first entry of a lane is a plain product (csr_kernels.cuh)
                if (e < end) { sum = __ldg(c.val + e) * __ldcg(c.x + __ldg(c.col + e)); e += L; }
            }
            for (; e < end; e += U * L) {
                int    cc[U];
                double vv[U], xx[U];
                bool   p[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int eu = e + u * L;
                    p[u]  = eu < end;
                    cc[u] = p[u] ? __ldg(c.col + eu) : __ldg(c.col + e);
                    vv[u] = p[u] ? __ldg(c.val + eu) : 0.0;
                }
#pragma unroll
                for (int u = 0; u < U; ++u) xx[u] = __ldcg(c.x + cc[u]);
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (p[u]) sum = fma(vv[u], xx[u], sum);
            }
        }
        if (L > 1) {
#pragma unroll
            for (int o = L / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        }
        if (valid && lane == 0) {
            double out;
            if (c.mode == MODE_SPMV) {
                out = c.alpha * sum;
            } else if (c.mode == MODE_SPMV_ACC) {
                out = c.alpha * sum + c.beta * __ldcg(c.y + r);
            } else if (c.mode == MODE_RESID) {
                out = __ldcg(c.f + r) - sum;
            } else {
                const double t = __ldcg(c.f + r) - sum;
                const double w = c.alpha * __ldg(c.d + r);
                out = fma(w, t, __ldcg(c.x + r));
            }
            c.y[r] = out;
        }
    }
}

// ---- one small operator, one plain launch --------------------------------------------------
// The streaming ring kernel (csr_kernels.cuh) pays for its pipeline -- mbarrier set-up, bulk
// copies, shared-memory staging -- even when the whole operator is a few hundred kilobytes; on
// such operators the direct-load row reduction above (same arithmetic, bit for bit) finishes
// in the time a dependent launch takes anyway.  One row group per L lanes, rows strided over
// the grid.
template <int L>
__global__ void __launch_bounds__(kThreads) small_csr_kernel(const TailCmd c) {
    const TailRow first = tail_csr_peek<L, kThreads>(c);     // matrix data: before the dependency
    ptx::pdl_wait();
    tail_csr<L, kThreads>(c, first);
}

__global__ void __launch_bounds__(kTailThreads, 1) coarse_tail_kernel(const TailArgs a) {
    TailRow first = tail_peek(a.cmd[0]);
    for (int k = 0; k < a.n; ++k) {
        const TailCmd &c = a.cmd[k];
        if (c.op == TAIL_CSR) {
            switch (c.lanes) {
            case 1:  tail_csr<1>(c, first); break;
            case 2:  tail_csr<2>(c, first); break;
            case 4:  tail_csr<4>(c, first); break;
            case 8:  tail_csr<8>(c, first); break;
            case 16: tail_csr<16>(c, first); break;
            default: tail_csr<32>(c, first); break;
            }
        } else if (c.op == TAIL_RELAX_ZERO) {
            // x = (omega*d).*rhs (relax_zero_kernel)
            const int stride = gridDim.x * kTailThreads;
            for (int i = blockIdx.x * kTailThreads + threadIdx.x; i < c.nrows; i += stride)
                c.y[i] = fma(c.alpha * __ldg(c.d + i), __ldcg(c.f + i), 0.0);
        } else {
            // x = Ainv * rhs: one warp per row (coarse_gemv_kernel), four loads in flight
            const int lane   = threadIdx.x & 31;
            const int nwarps = gridDim.x * (kTailThreads / 32);
            for (int row = (blockIdx.x * kTailThreads + threadIdx.x) >> 5; row < c.nrows; row += nwarps) {
                const double *rowp = c.val + (size_t)row * c.nrows;
                double s = 0.0;
                int j = lane;
                for (; j + 96 < c.nrows; j += 128) {
                    const double a0 = __ldg(rowp + j), a1 = __ldg(rowp + j + 32);
                    const double a2 = __ldg(rowp + j + 64), a3 = __ldg(rowp + j + 96);
                    const double b0 = __ldcg(c.x + j), b1 = __ldcg(c.x + j + 32);
                    const double b2 = __ldcg(c.x + j + 64), b3 = __ldcg(c.x + j + 96);
                    s = fma(a0, b0, s); s = fma(a1, b1, s); s = fma(a2, b2, s); s = fma(a3, b3, s);
                }
                for (; j < c.nrows; j += 32) s = fma(__ldg(rowp + j), __ldcg(c.x + j), s);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (lane == 0) c.y[row] = s;
            }
        }
        if (k + 1 < a.n) {
            first = tail_peek(a.cmd[k + 1]);          // matrix data only: safe before the barrier
            tail_barrier(a.bar, a.bar_base + (unsigned long long)(k + 1) * gridDim.x);
        }
    }
}

} // namespace b200
