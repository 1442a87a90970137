// csr_kernels.cuh -- the streaming CSR kernels of the V-cycle.
//
// One kernel template covers every pass over a CSR operator in the AMGCL solve
// phase (SURVEY.md section 8a, rows a1, a2, a9, a10):
//
//   MODE_SPMV   y = alpha*A*x (+ beta*y)      backend::spmv      matrix_ops.hpp:47-83
//   MODE_RESID  y = f - A*x                   backend::residual  matrix_ops.hpp:85-115
//   MODE_RELAX  y = x + (alpha*d).*(f - A*x)  damped_jacobi / spai0 sweep
//                                             damped_jacobi.hpp:103-132, spai0.hpp:86-109
//
// Data movement.  The matrix is cut (on the host, once, at upload) into row
// blocks: runs of consecutive rows starting at a multiple of four whose
// non-zeros fit a shared-memory stage.  A block's slice of `val`, `col` and
// `ptr16` (row pointers relative to the block's first non-zero) is contiguous in
// global memory, so one elected thread fetches it with one 1-D TMA bulk copy each (cp.async.bulk -> SASS UBLKCP) that complete on an
// mbarrier; the matrix stream never passes through registers and is tagged
// L2::evict_first so it does not displace the gathered x-vector.  Rows are
// then reduced out of shared memory by groups of L lanes (L = 1..32, chosen
// from the average row length) with a shuffle tree; with L == 1 the summation
// order is exactly the reference's sequential `sum += a.value()*x[a.col()]`.
//
// Two schedulers over the same stage code:
//   variant 0: one row block per CTA, latency hidden by several CTAs per SM;
//   variant 1: persistent CTAs walking the block list with an S-deep ring of
//              stages, so S*CTAs/SM bulk copies are always in flight per SM.
//
// Column formats (template parameter FMT): how the kernel learns the column of an entry.  The
// arithmetic (entry order, lanes, shuffle tree, epilogue) is shared, so every format gives the
// bits of the plain one (tests/test_gpu_formats.py, tests/test_gpu_window.py); measurements in
// DESIGN.md section 3.1b.
//
// Windowed operators (FMT_WINDOW; opt-in: measured slower than the plain path).  For an operator
// whose row blocks gather from few distinct places the upload also stores, per block, the runs
// of x it reads and, per entry, the 16-bit position of its column inside the block's window.
// The kernel fills the window into shared memory with coalesced loads (one 32-byte sector is
// fetched once per block, not once per scattered 8-byte gather that misses the small L1 left
// beside the stages) and reduces the rows entirely out of shared memory; the column stream
// shrinks from 4 to 2 bytes per entry.
//
// Offset-indexed columns (FMT_OFFSET).  In a matrix assembled on a structured grid every entry
// sits on one of a few diagonals: col - row takes a handful of distinct values (7 for the
// Poisson stencil, a few more on a partitioned operator where halo columns are renumbered).  If
// there are at most 256 of them, the upload also stores one BYTE per entry -- the index of its
// offset in a table -- and the kernel streams 1 instead of 4 bytes of column per entry
// (9 instead of 12 bytes per FP64 entry, 5 instead of 8 per FP32 entry), rebuilding the column
// as row + table[index] from shared memory.
//
// Pattern-indexed rows (FMT_PATTERN).  On such a matrix whole ROWS repeat: the tuple of offsets
// (col - row of every entry, in entry order) of a row is one of a few patterns (27 for the
// Poisson problem: interior + boundary combinations).  With at most 256 patterns the upload
// stores one byte per ROW and no column information per entry at all: the kernel streams the
// values (8 or 4 bytes per entry), the row pointers and the pattern ids, and rebuilds
// col = row + pattern[k] for the k-th entry of the row from a table in shared memory -- one
// shared-memory load per entry, as many as the plain path needs for its staged column.  The
// default for every operator that qualifies (the finest level of a structured-grid problem).
//
// Value-keyed patterns (FMT_PATVAL).  Where the pairs (offset, value) repeat as well -- a stencil
// operator with constant coefficients, again 27 patterns for the Poisson problem -- the pattern
// also fixes the row's values and its length: the operator streams one byte per row and nothing
// else, and the k-th entry of row r is (col = row + off[pstart[pid] + k], value = pval[pstart[pid] + k])
// from tables in shared memory (built by patterns.cuh).  With nothing per entry to stage, these
// operators run csr_patval_kernel instead of the ring: it loads the ids directly and keeps several
// rows per thread in flight.  Same entries in the same order, on the same threads, as FMT_PATTERN
// on the ring: the bits of the streamed values.  Single-GPU only.
//
// Narrow columns (FMT_COL16 / FMT_COL24).  Every other operator (no long blocks, <= 8 lanes per
// row) stores, per block, its smallest column and, per entry, the low 16 bits of col - base, plus
// the high 8 bits in an array of their own where some block spans more than 16 bits
// (narrow.cuh): 2 or 3 instead of 4 bytes of column per entry.
//
// The rows of the blocks a CTA walks form one stream over its warps.  Between blocks the CTA
// synchronises with a barrier (windowed; plain and narrow operators whose blocks give every warp
// rows) or not at all (the last warp done with a stage refills it) -- see the ring kernel.
//
// Precision.  Every kernel is a template over the element types of the matrix
// values, the gathered vector, the right-hand side, the output and the smoother
// diagonal (struct Prec).  FP64 throughout is the default; the other
// combinations are the ones AMGCL's mixed-precision composition produces (FP32
// hierarchy under an FP64 Krylov solver, tutorial/1.poisson3Db/poisson3Db.cpp:45-51):
// as in the reference (matrix_ops.hpp:57) a row sum is accumulated in the value
// type of the OUTPUT vector.  An FP64 operator whose every value converts to FP32 and back
// with the same bits also streams them as FP32 (PrecSD): the widened value is the same double,
// so every product, row sum and epilogue is that of PrecDD.  An FP64 operator with at most 4,096
// distinct values streams an 8- or 16-bit index per entry instead (PrecI8D / PrecI16D, built by
// values.cuh): the kernel reads the double the index names from a table in shared memory, so it
// too multiplies the very same doubles as PrecDD.
#pragma once
#include "common.cuh"
#include "reduce.cuh"
#include <type_traits>

namespace b200 {

// storage format of the column indices the kernel streams
enum { FMT_PLAIN = 0,     // int32 column per entry
       FMT_WINDOW = 1,    // 16-bit position in the block's shared-memory window of x
       FMT_OFFSET = 2,    // 8-bit index into a table of (col - row) offsets
       FMT_PATTERN = 3,   // no per-entry column: 8-bit pattern id per row, col = row + pattern[k]
       FMT_COL16 = 4,     // 16-bit column relative to the block's smallest column
       FMT_COL24 = 5,     // the same in 24 bits: a 16-bit and an 8-bit array
       FMT_PATVAL = 6 };  // no per-entry data: 8-bit pattern id per row, columns AND values from tables
static_assert(FMT_PLAIN == B200_FMT_PLAIN && FMT_WINDOW == B200_FMT_WINDOW && FMT_OFFSET == B200_FMT_OFFSET &&
              FMT_PATTERN == B200_FMT_PATTERN && FMT_COL16 == B200_FMT_COL16 && FMT_COL24 == B200_FMT_COL24 &&
              FMT_PATVAL == B200_FMT_PATVAL,
              "formats as include/amgcl_b200_formats.h reports them");

enum { MODE_SPMV = 0, MODE_SPMV_ACC = 1, MODE_RESID = 2, MODE_RELAX = 3,
       // y = f - A x with x = (alpha*d).*f formed on the fly and written to xw: the smoother's
       // first sweep from x = 0 (relax_zero_kernel) fused into the residual that follows it
       // (amg.hpp:527-534: apply_pre, then residual)
       MODE_RESID_SCALED = 4 };

#ifndef B200_GATHER_BATCH
#define B200_GATHER_BATCH 4
#endif
constexpr int kGatherBatch = B200_GATHER_BATCH;   // x-gathers issued back to back per lane

template <class TV_, class TX_, class TF_, class TY_, class TD_>
struct Prec {
    typedef TV_ TV;   // matrix values
    typedef TX_ TX;   // gathered vector x
    typedef TF_ TF;   // right-hand side f
    typedef TY_ TY;   // output y (and accumulation type of a row sum)
    typedef TD_ TD;   // smoother diagonal
};
typedef Prec<double, double, double, double, double> PrecDD;   // FP64 throughout
typedef Prec<float, float, float, float, float>      PrecFF;   // FP32 level of a mixed hierarchy
typedef Prec<float, double, double, double, float>   PrecFD;   // FP32 operator on FP64 vectors
typedef Prec<float, double, double, float, float>    PrecFDF;  // finest residual into FP32 scratch
typedef Prec<float, float, float, double, float>     PrecFFD;  // prolongation into an FP64 iterate
// FP64 operator whose values are all exact FP32 (b200_csr_s::val32): 4-byte values widened to the
// same doubles at FMA time, FP64 everything else -- the bits of PrecDD
typedef Prec<float, double, double, double, double>  PrecSD;
// FP64 operator with at most 256 / 4,096 distinct values (b200_csr_s::vidx): the stage holds an
// 8- / 16-bit index per entry, read as vtab[index] at FMA time -- the bits of PrecDD
typedef Prec<unsigned char, double, double, double, double>  PrecI8D;
typedef Prec<unsigned short, double, double, double, double> PrecI16D;

// does the stored value type index a table of values?
template <class TV> struct IndexedValues : std::false_type {};
template <> struct IndexedValues<unsigned char> : std::true_type {};
template <> struct IndexedValues<unsigned short> : std::true_type {};

// the value of a stored entry, in the type of the row sum: the entry itself or, indexed, the
// table entry it names
template <class TS, class TV>
__device__ __forceinline__ TS value_of(TV v, const double *vtab) {
    if constexpr (IndexedValues<TV>::value) return (TS)vtab[v];
    else return (TS)v;
}

template <class P>
struct CsrArgsT {
    const int    *ptr;    // (long blocks)
    const unsigned short *ptr16;   // staged blocks: ptr[r] - first non-zero of r's block
    const int    *col;
    const typename P::TV *val;
    const double *vtab;   // indexed values: the table val indexes (vtab_n entries), else nullptr
    int           vtab_n;
    const int4   *blk;    // [nblocks] in WALK ORDER: {first row (~first row if the block gathers
                          //   halo columns), end row, first non-zero, end non-zero}
    int           nrows;
    int           nblocks;
    int           rows_cap;
    int           nnz_cap;
    int           row_stream;     // plain / narrow formats: no CTA barrier between blocks (ring kernel)
    const typename P::TX *x;      // gathered vector (local columns)
    const typename P::TX *xh;     // halo values for columns >= nloc (multi-GPU), else nullptr
    int           nloc;   // number of local columns when xh is set
    // multi-GPU, peer-memory transport: the halo is pushed by the peers while this kernel
    // already works on interior rows; a block that gathers remote columns first waits for
    // the flags of the ranks in wait_mask to reach wait_seq (csrc/peer.cuh protocol)
    // (such blocks come last in the walk order, so the transfer overlaps the interior rows)
    const unsigned long long *wait_flags;  // flag row of the current parity (16 slots)
    unsigned int              wait_mask;
    unsigned long long        wait_seq;
    // ... and THIS rank's boundary values are pushed by this very kernel: right after the
    // grid dependency resolves every CTA packs a slice of x[send_idx[.]] into the halo buffers
    // of the ranks that gather them (plain stores over NVLink), the last CTA to finish
    // releases their flags; then all CTAs go on to the interior row blocks
    const int                *send_idx;
    int                       n_send;
    int                       nranks;
    typename P::TX           *push_data[kMaxRanks];   // my segment in peer q's halo buffer (or nullptr)
    unsigned long long       *push_flag[kMaxRanks];   // my flag in peer q's flag row (or nullptr)
    unsigned int             *push_ticket;
    unsigned long long        push_seq;                // 0: nothing to push / NCCL transport
    // row shares of a replicated result (R onto a small level): every row is also stored into
    // every rank's gather buffer; the last CTA releases the flags at the end of the kernel
    int                       gather_on;
    typename P::TY           *gather_data[kMaxRanks]; // my share's place in rank q's buffer
    unsigned long long       *gather_flag[kMaxRanks];
    unsigned int             *gather_ticket;
    unsigned long long        gather_seq;
    // Windowed operators: window-local column of every entry, the runs of x each block's window
    // is made of ({first column, length | first slot << 16}), and each block's range of runs
    const unsigned short *col16;
    const int2   *wrun;
    const int2   *wblk;   // [nblocks] in walk order
    int           run_cap;// most runs a block has (stage layout); 0: not a windowed launch
    // Offset-indexed operators: index of every entry's (col - row) in off_tab[256]
    const unsigned char *idx8;
    const int    *off_tab;
    // Pattern-indexed operators: pattern id of every row, first table entry of every pattern
    // ([257]), and the table of offsets itself
    const unsigned char  *pid;
    const unsigned short *pat_start;
    const int    *pat_off;
    int           pat_total;   // entries of pat_off in use (<= kPatOffCap)
    const typename P::TV *pat_val;   // FMT_PATVAL: the value of every table entry, parallel to pat_off
    // Narrow columns (FMT_COL16 / FMT_COL24): col = cbase[block] + clo16[e] (+ chi8[e] << 16)
    const unsigned short *clo16;
    const unsigned char  *chi8;
    const int    *cbase;  // [nblocks] in walk order
    typename P::TY       *y;      // output
    typename P::TX       *xw;     // RESID_SCALED: where x = (alpha*d).*f is written
    const typename P::TF *f;      // rhs          (RESID, RELAX)
    const typename P::TD *d;      // diagonal     (RELAX)
    double        alpha;  // SPMV: alpha; RELAX: omega
    double        beta;   // SPMV_ACC
    // scalars produced while the rows are in registers (reduce.cuh; FP64 outputs only):
    //   ndot >= 1: sum_r y_r * w_r  (w == nullptr: RELAX uses the rhs f, otherwise y itself)
    //   ndot == 2: additionally sum_r y_r^2
    int           ndot;
    const double *w;
    RedOut        red;
};
typedef CsrArgsT<PrecDD> CsrArgs;

// ---- shared memory layout of one stage --------------------------------------
struct StageLayout {
    int val_off, col_off, hi_off, ptr_off, run_off, pid_off, bytes;
};
// fmt: storage format of the columns (FMT_*); run_cap: FMT_WINDOW only, most runs a block has
__host__ __device__ inline StageLayout stage_layout(int rows_cap, int nnz_cap, int val_size,
                                                    int fmt = FMT_PLAIN, int run_cap = 0) {
    StageLayout s;
    s.val_off = 0;
    int val_bytes = nnz_cap * val_size + 16;        // source aligned down to 16 B
    val_bytes = (val_bytes + 15) & ~15;
    s.col_off = s.val_off + val_bytes;
    const bool narrow = fmt == FMT_COL16 || fmt == FMT_COL24;
    int col_bytes = fmt == FMT_WINDOW || narrow ? (nnz_cap + 16) * 2   // +7 align down, +7 round up
                  : fmt == FMT_OFFSET  ? (nnz_cap + 32)       // +15 align down, +15 round up
                  : fmt == FMT_PATTERN ? 0
                                       : (nnz_cap + 8) * 4;   // +3 align down, +3 round up
    col_bytes = (col_bytes + 15) & ~15;
    s.hi_off = s.col_off + col_bytes;
    int hi_bytes = fmt == FMT_COL24 ? nnz_cap + 32 : 0;       // +15 align down, +15 round up
    hi_bytes = (hi_bytes + 15) & ~15;
    s.ptr_off = s.hi_off + hi_bytes;
    int ptr_bytes = (rows_cap + 16) * 2;            // 16-bit: +7 align down, +7 round up
    ptr_bytes = (ptr_bytes + 15) & ~15;
    s.run_off = s.ptr_off + ptr_bytes;
    int run_bytes = fmt == FMT_WINDOW ? (run_cap + 2) * 8 : 0;   // +1 align down, +1 round up
    run_bytes = (run_bytes + 15) & ~15;
    s.pid_off = s.run_off + run_bytes;
    int pid_bytes = fmt == FMT_PATTERN ? rows_cap + 32 : 0;   // +15 align down, +15 round up
    pid_bytes = (pid_bytes + 15) & ~15;
    s.bytes = s.pid_off + pid_bytes;
    return s;
}
constexpr int kMaxStages   = 8;
constexpr int kHeaderBytes = 448;   // mbarriers [0,64) + reduction scratch [64,128) + descriptors [128,384)
                                    // + per-stage "warps done" counters [384,416)
constexpr int kWinRunLen   = 64;    // longest run of a window (longer ones are cut at upload)
constexpr int kOffTabLen   = 256;   // offset-indexed operators: entries of the (col - row) table
constexpr int kPatCap      = 256;   // pattern-indexed operators: most row patterns ...
constexpr int kPatOffCap   = 1024;  // ... and most offsets in all patterns together
// shared memory behind the stages: the window of x / the offset table / the pattern tables, then an
// indexed operator's table of values; FMT_PATVAL (csr_patval_kernel, no stages): the pattern tables
// and the entries' values, val_size bytes each
constexpr int kPatTabBytes = kPatOffCap * 4 + ((kPatCap + 1) * 2 + 15) / 16 * 16;
__host__ __device__ constexpr int fmt_table_bytes(int fmt, int val_size) {   // (not FMT_WINDOW: sized per operator)
    return fmt == FMT_OFFSET ? kOffTabLen * 4 : fmt == FMT_PATTERN ? kPatTabBytes
         : fmt == FMT_PATVAL ? kPatTabBytes + kPatOffCap * val_size : 0;
}

struct BlockDesc {      // written by the producer thread, read by everyone after the wait
    int r0, r1;         // row range
    int e0, e1;         // non-zero range
    int halo;           // the block gathers columns owned by other ranks
    int q0, q1;         // windowed operators: the block's runs
    int cb;             // narrow columns: the block's smallest column
};
static_assert(sizeof(BlockDesc) * kMaxStages <= 384 - 128, "descriptors overflow the header");

// ---- issue the bulk copies of one row block ----------------------------------
template <int FMT = FMT_PLAIN, class P>
__device__ __forceinline__ BlockDesc load_desc(const CsrArgsT<P> &a, int b) {
    const int4 q = __ldg(a.blk + b);       // one 16-byte load: nothing else to chase
    BlockDesc d;
    d.halo = q.x < 0;
    d.r0 = q.x < 0 ? ~q.x : q.x;
    d.r1 = q.y; d.e0 = q.z; d.e1 = q.w;
    d.q0 = d.q1 = 0; d.cb = 0;
    if (FMT == FMT_WINDOW) {
        const int2 w = __ldg(a.wblk + b);
        d.q0 = w.x; d.q1 = w.y;
    }
    if (FMT == FMT_COL16 || FMT == FMT_COL24) d.cb = __ldg(a.cbase + b);
    return d;
}

// Returns true if the block was staged (false: too long, use the strided path).
// Every slice is its own bulk copy, its source aligned down to 16 bytes (the kernel adds back the
// offset); the row pointers are the block-relative 16-bit ones of rows [r0, r1].
template <int FMT = FMT_PLAIN, class P>
__device__ __forceinline__ bool issue_block(const CsrArgsT<P> &a, const BlockDesc &d, char *stage,
                                            const StageLayout &lay, uint64_t *bar,
                                            uint64_t policy) {
    typedef typename P::TV TV;
    constexpr int VA = 16 / (int)sizeof(TV);        // values per 16 bytes
    const int nnz = d.e1 - d.e0;
    if (FMT == FMT_PLAIN && nnz > a.nnz_cap) {
        // nothing to stage: complete the phase with a plain arrive
        // (only a plain operator has long blocks)
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(ptx::smem_addr(bar))
                     : "memory");
        return false;
    }
    const int a0 = d.e0 & ~(VA - 1);
    const int nval = ((d.e1 - a0) + VA - 1) & ~(VA - 1);
    const int p0 = d.r0 & ~7;                       // 16-bit row pointers: 8 per 16 bytes
    const int nptr = ((d.r1 + 1 - p0) + 7) & ~7;    // (+ the next block's first row: 0)
    int ncol = 0, nhi = 0, nrun = 0, npid = 0;      // bytes of each slice
    const void *csrc = nullptr, *hsrc = nullptr, *psrc = nullptr;
    if (FMT == FMT_PLAIN) {
        const int c0 = d.e0 & ~3;
        ncol = (((d.e1 - c0) + 3) & ~3) * 4;
        csrc = a.col + c0;
    } else if (FMT == FMT_WINDOW || FMT == FMT_COL16 || FMT == FMT_COL24) {
        const int c0 = d.e0 & ~7;
        ncol = (((d.e1 - c0) + 7) & ~7) * 2;
        csrc = (FMT == FMT_WINDOW ? a.col16 : a.clo16) + c0;
    } else if (FMT == FMT_OFFSET) {
        const int c0 = d.e0 & ~15;
        ncol = ((d.e1 - c0) + 15) & ~15;
        csrc = a.idx8 + c0;
    }
    if (FMT == FMT_COL24) {
        const int h0 = d.e0 & ~15;
        nhi = ((d.e1 - h0) + 15) & ~15;
        hsrc = a.chi8 + h0;
    }
    if (FMT == FMT_WINDOW) {
        const int qa = d.q0 & ~1;                   // runs: 2 per 16 bytes
        nrun = (((d.q1 - qa) + 1) & ~1) * 8;
        psrc = a.wrun + qa;
    }
    if (FMT == FMT_PATTERN) {
        const int q0 = d.r0 & ~15;                  // pattern ids: 16 per 16 bytes
        npid = ((d.r1 - q0) + 15) & ~15;
        psrc = a.pid + q0;
    }
    const uint32_t bytes = nval * (int)sizeof(TV) + ncol + nhi + nptr * 2 + nrun + npid;
    ptx::mbar_expect_tx(bar, bytes);
    if (nval) ptx::bulk_g2s(stage + lay.val_off, a.val + a0, nval * (int)sizeof(TV), bar, policy);
    if (ncol) ptx::bulk_g2s(stage + lay.col_off, csrc, ncol, bar, policy);
    if (nhi) ptx::bulk_g2s(stage + lay.hi_off, hsrc, nhi, bar, policy);
    if (nptr) ptx::bulk_g2s(stage + lay.ptr_off, a.ptr16 + p0, nptr * 2, bar, policy);
    if (nrun) ptx::bulk_g2s(stage + lay.run_off, psrc, nrun, bar, policy);
    if (npid) ptx::bulk_g2s(stage + lay.pid_off, psrc, npid, bar, policy);
    return true;
}

// ---- per-row epilogue ----------------------------------------------------------
// acc: the thread's running contributions to the launch's scalars (reduce.cuh)
struct RowAcc { double s0, s1; };

// what the epilogue of a row reads besides the row sum; loaded BEFORE the row's gathers are
// issued so that it arrives with them (one memory round per row instead of two)
template <class P>
struct RowOps {
    typename P::TF f;     // rhs           (RESID, RESID_SCALED, RELAX)
    typename P::TD d;     // diagonal      (RESID_SCALED, RELAX)
    typename P::TX x;     // old iterate   (RELAX)
    typename P::TY y;     // old output    (SPMV_ACC)
    double         w;     // dot weight    (ndot with w)
};
template <int MODE, class P>
__device__ __forceinline__ RowOps<P> load_row_ops(const CsrArgsT<P> &a, int r) {
    RowOps<P> o;
    o.f = 0; o.d = 0; o.x = 0; o.y = 0; o.w = 0.0;
    if (MODE == MODE_SPMV_ACC) o.y = a.y[r];
    if (MODE == MODE_RESID || MODE == MODE_RESID_SCALED || MODE == MODE_RELAX) o.f = a.f[r];
    if (MODE == MODE_RESID_SCALED || MODE == MODE_RELAX) o.d = a.d[r];
    if (MODE == MODE_RELAX) o.x = a.x[r];
    if (a.ndot && a.w) o.w = a.w[r];
    return o;
}

template <int MODE, class P>
__device__ __forceinline__ void store_row(const CsrArgsT<P> &a, int r, typename P::TY sum, RowAcc &acc,
                                          const RowOps<P> &o) {
    typedef typename P::TY TY;
    TY out;
    double wv = 0.0;
    if (MODE == MODE_SPMV) {
        out = (TY)(a.alpha * sum);
    } else if (MODE == MODE_SPMV_ACC) {
        out = (TY)(a.alpha * sum + a.beta * o.y);
    } else if (MODE == MODE_RESID) {
        out = (TY)(o.f - sum);
    } else if (MODE == MODE_RESID_SCALED) {
        const typename P::TF fr = o.f;
        out = (TY)(fr - sum);
        a.xw[r] = fma((typename P::TX)(a.alpha * o.d), (typename P::TX)fr, (typename P::TX)0);
    } else {
        // x_new = (omega*d)*t + x with t = f - A x; same association as the
        // reference's vmul  z = a*x*y + b*z  (builtin.hpp:1238-1265)
        const typename P::TF fr = o.f;
        const TY t = (TY)(fr - sum);
        const TY w = (TY)(a.alpha * o.d);
        out = fma(w, t, (TY)o.x);
        wv = (double)fr;
    }
    a.y[r] = out;
    if (a.gather_on) {
#pragma unroll 1
        for (int q = 0; q < a.nranks; ++q)
            if (a.gather_data[q]) a.gather_data[q][r] = out;
    }
    if (a.ndot) {
        const double yv = (double)out;
        if (a.w) wv = o.w;
        else if (MODE != MODE_RELAX) wv = yv;
        acc.s0 = fma(yv, wv, acc.s0);
        if (a.ndot > 1) acc.s1 = fma(yv, yv, acc.s1);
    }
}
// (operands loaded on the spot: the paths that do not overlap them with the gathers)
template <int MODE, class P>
__device__ __forceinline__ void store_row(const CsrArgsT<P> &a, int r, typename P::TY sum, RowAcc &acc) {
    store_row<MODE>(a, r, sum, acc, load_row_ops<MODE>(a, r));
}

// ---- x[col]: local columns from the vector, remote ones from the all-gathered halo --
template <bool HALO, class P>
__device__ __forceinline__ typename P::TX gather(const CsrArgsT<P> &a,
                                                 const typename P::TX *__restrict__ x, int c) {
    if (HALO) {
        // halo values may arrive while the kernel runs: read them through L2 (ld.cg)
        if (c < a.nloc) return __ldg(x + c);
        return __ldcg(a.xh + (c - a.nloc));
    }
    return __ldg(x + c);
}

// RESID_SCALED: the gathered vector does not exist yet; its entry c is (alpha*d[c])*f[c],
// evaluated exactly as relax_zero_kernel does
template <int MODE, bool HALO, class P>
__device__ __forceinline__ typename P::TX gather_m(const CsrArgsT<P> &a,
                                                   const typename P::TX *__restrict__ x, int c) {
    typedef typename P::TX TX;
    if (MODE == MODE_RESID_SCALED)
        return fma((TX)(a.alpha * __ldg(a.d + c)), (TX)__ldg(a.f + c), (TX)0);
    return gather<HALO>(a, x, c);
}

// Block until the peers' halo pushes for this exchange have landed (thread 0 polls the
// flags with acquire semantics, the CTA follows through the barrier).
template <bool HALO, class P>
__device__ __forceinline__ void wait_for_halo(const CsrArgsT<P> &a, const BlockDesc &d) {
    if (!HALO) return;
    if (!d.halo || !a.wait_mask) return;                       // uniform per CTA
    if (threadIdx.x == 0) {
        unsigned int m = a.wait_mask;
        while (m) {
            const int q = __ffs(m) - 1;
            m &= m - 1;
            unsigned long long v;
            do {
                asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(a.wait_flags + q) : "memory");
            } while (v < a.wait_seq);
        }
    }
    __syncthreads();
}

// ---- windowed operators: bring the block's runs of x into shared memory --------------------
// One warp per run (runs are at most kWinRunLen long and start on a 32-byte boundary of x, so a
// warp's loads are whole sectors); ends with a CTA barrier.
template <int MODE, bool HALO, class P>
__device__ __forceinline__ void fill_window(const CsrArgsT<P> &a, const BlockDesc &d, const char *stage,
                                            const StageLayout &lay, typename P::TX *win) {
    const int2 *runs = reinterpret_cast<const int2 *>(stage + lay.run_off) + (d.q0 & 1);
    const int nq   = d.q1 - d.q0;
    const int lane = threadIdx.x & 31;
    const typename P::TX *__restrict__ x = a.x;
    for (int q = threadIdx.x >> 5; q < nq; q += kThreads / 32) {
        const int2 rn   = runs[q];
        const int first = rn.x;
        const int len   = rn.y & 0xffff;
        const int slot  = (int)((unsigned)rn.y >> 16);
#pragma unroll
        for (int i = lane; i < kWinRunLen; i += 32)
            if (i < len) win[slot + i] = gather_m<MODE, HALO>(a, x, first + i);
    }
    __syncthreads();
}

// ---- reduce the rows of a staged block out of shared memory ---------------------
// FMT_WINDOW: x comes from the block's window, `win`, indexed by the 16-bit columns;
// FMT_OFFSET: the column of an entry of row r is r + off[8-bit index];
// FMT_PATTERN: the column of the k-th entry of row r is r + off[pstart[pattern id of r] + k];
// FMT_COL16 / FMT_COL24: the column is the block's smallest column + the stored 16 (+ 8) bits
//
// Rows go to warps in chunks of 32 / L rows: chunk j of the block (rows [j*32/L, (j+1)*32/L)) is
// reduced by warp (k0 + j) % 8, one row per group of L lanes.  k0 is the block's first chunk in
// the CTA's stream of rows (csr_ring_kernel); with k0 = 0 warp w takes chunks w, w + 8, ...
template <int MODE, int L, bool HALO, class P, int FMT = FMT_PLAIN>
__device__ __forceinline__ void compute_staged(const CsrArgsT<P> &a, const BlockDesc &d,
                                               const char *stage, const StageLayout &lay, RowAcc &acc,
                                               const typename P::TX *win = nullptr, const int *off = nullptr,
                                               const unsigned short *pstart = nullptr, int k0 = 0,
                                               const double *vtab = nullptr) {
    constexpr bool WIN = FMT == FMT_WINDOW;
    constexpr bool OFF = FMT == FMT_OFFSET;
    constexpr bool PAT = FMT == FMT_PATTERN;
    constexpr bool NAR = FMT == FMT_COL16 || FMT == FMT_COL24;
    typedef typename P::TV TV;
    typedef typename P::TX TX;
    typedef typename P::TY TS;                       // row sums live in the output's type
    typedef typename std::conditional<WIN || NAR, unsigned short,
                                      typename std::conditional<OFF, unsigned char, int>::type>::type CI;
    static_assert(!((WIN || OFF || PAT || NAR) && L >= 16), "compressed column formats use at most 8 lanes per row");
    const unsigned char *pid_s = reinterpret_cast<const unsigned char *>(stage + lay.pid_off) + (d.r0 & 15);
    constexpr int VA = 16 / (int)sizeof(TV);
    const TV *val_s = reinterpret_cast<const TV *>(stage + lay.val_off);
    const CI     *col_s = reinterpret_cast<const CI *>(stage + lay.col_off);
    const unsigned char  *hi_s  = reinterpret_cast<const unsigned char *>(stage + lay.hi_off);
    const unsigned short *ptr_s = reinterpret_cast<const unsigned short *>(stage + lay.ptr_off) + (d.r0 & 7);
    const int vo = d.e0 & ~(VA - 1);
    const int nr = d.r1 - d.r0;
    const int co = WIN || NAR ? (d.e0 & ~7) : OFF ? (d.e0 & ~15) : (d.e0 & ~3);
    const int ho = d.e0 & ~15;
    // what the stage holds for entry e: the column (plain, narrow) or its index (window, offset)
    auto stored_col = [&](int e) -> int {
        if (!NAR) return col_s[e - co];
        if (FMT == FMT_COL24) return d.cb + ((int)col_s[e - co] | (int)hi_s[e - ho] << 16);
        return d.cb + (int)col_s[e - co];
    };
    // row rr's entries, from the block-relative row pointers; the slot after the last row is
    // the next block's first row, always 0: the last row ends at e1 = e0 + 0 + (e1 - e0)
    auto row_beg = [&](int rr) -> int { return d.e0 + (int)ptr_s[rr]; };
    auto row_end = [&](int rr) -> int { return d.e0 + (int)ptr_s[rr + 1] + (rr + 1 == nr ? d.e1 - d.e0 : 0); };
    constexpr int G = kThreads / L;
    const int c0   = (((int)threadIdx.x >> 5) - k0) & (kThreads / 32 - 1);   // this warp's first chunk
    const int g    = (threadIdx.x & 31) / L;                                   // its row in a chunk
    const int lane = threadIdx.x % L;
    const TX *__restrict__ x = a.x;

    if (L >= 16) {
        // Wide groups (a half or a full warp per row): consecutive lanes read consecutive
        // entries, so the shared-memory reads are bank-conflict free and the gathers of one
        // row coalesce.  Memory-level parallelism comes from working on RU rows at once
        // instead of batching along one (short) row.
        constexpr int RU = kGatherBatch;
        for (int base = c0 * (32 / L); base < nr; base += G * RU) {
            int  beg[RU], end[RU], c[RU];
            TV   v[RU];
            TX   xv[RU];
            TS   sum[RU];
            bool rowok[RU], p[RU];
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                const int rr = base + u * G + g;
                rowok[u] = rr < nr;
                beg[u] = rowok[u] ? row_beg(rr) : 0;
                end[u] = rowok[u] ? row_end(rr) : 0;
                sum[u] = 0;
            }
            // first L entries of each of the RU rows: all loads first, then the gathers
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                const int e = beg[u] + lane;
                p[u] = e < end[u];
                c[u] = p[u] ? stored_col(e) : 0;
                v[u] = p[u] ? val_s[e - vo] : (TV)0;
            }
#pragma unroll
            for (int u = 0; u < RU; ++u) xv[u] = p[u] ? gather_m<MODE, HALO>(a, x, c[u]) : (TX)0;
#pragma unroll
            for (int u = 0; u < RU; ++u)
                if (p[u]) sum[u] = value_of<TS>(v[u], vtab) * (TS)xv[u];
            // rows longer than L: the rest, row by row
#pragma unroll
            for (int u = 0; u < RU; ++u)
                for (int e = beg[u] + lane + L; e < end[u]; e += L)
                    sum[u] = fma(value_of<TS>(val_s[e - vo], vtab), (TS)gather_m<MODE, HALO>(a, x, stored_col(e)),
                                 sum[u]);
#pragma unroll
            for (int o = L / 2; o > 0; o >>= 1) {
#pragma unroll
                for (int u = 0; u < RU; ++u) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
            }
#pragma unroll
            for (int u = 0; u < RU; ++u)
                if (rowok[u] && lane == 0) store_row<MODE>(a, d.r0 + base + u * G + g, sum[u], acc);
        }
    } else
    for (int base = c0 * (32 / L); base < nr; base += G) {
        const int  rr    = base + g;
        const bool valid = rr < nr;
        TS sum = 0;
        RowOps<P> ops;
        ops.f = 0; ops.d = 0; ops.x = 0; ops.y = 0; ops.w = 0.0;
        if (valid) {
            // the epilogue's operands travel with the row's gathers
            if (lane == 0) ops = load_row_ops<MODE>(a, d.r0 + rr);
            const int beg = row_beg(rr);
            const int end = row_end(rr);
            // PAT: the row's pattern starts at off[pb + beg], so entry e sits at off[pb + e]
            int pb = 0;
            if (PAT) pb = (int)pstart[pid_s[rr]] - beg;
            // U independent gathers in flight per lane, then the FMAs in entry order (one lane per
            // row: short rows, a whole row of up to 8 entries goes out in one round)
            constexpr int U = (L == 1) ? 2 * kGatherBatch : kGatherBatch;
            for (int e = beg + lane; e < end; e += U * L) {
                int  c[U];
                TX   xv[U];
                bool p[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int eu = e + u * L;
                    p[u] = eu < end;
                    if (PAT) c[u] = d.r0 + rr + off[pb + (p[u] ? eu : e)];
                    else c[u] = stored_col(p[u] ? eu : e);
                }
                if (OFF) {
#pragma unroll
                    for (int u = 0; u < U; ++u) c[u] = d.r0 + rr + off[c[u]];
                }
#pragma unroll
                for (int u = 0; u < U; ++u)
                    xv[u] = !p[u] ? (TX)0 : WIN ? win[c[u]] : gather_m<MODE, HALO>(a, x, c[u]);
                // (the values come from shared memory when they are needed: no registers held
                //  across the gathers)
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (p[u]) sum = fma(value_of<TS>(val_s[e + u * L - vo], vtab), (TS)xv[u], sum);
            }
        }
        if (L > 1) {
#pragma unroll
            for (int o = L / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        }
        if (valid && lane == 0) store_row<MODE>(a, d.r0 + rr, sum, acc, ops);
    }
}

// ---- rows too long to stage: whole CTA strides over each row -----------------------
template <int MODE, bool HALO, class P>
__device__ __forceinline__ void compute_long(const CsrArgsT<P> &a, const BlockDesc &d,
                                             double *red_s /* >= 8 doubles */, RowAcc &acc) {
    typedef typename P::TX TX;
    typedef typename P::TY TS;
    const TX *__restrict__ x = a.x;
    for (int r = d.r0; r < d.r1; ++r) {
        const int beg = __ldg(a.ptr + r), end = __ldg(a.ptr + r + 1);
        TS sum = 0;
        for (int e = beg + threadIdx.x; e < end; e += kThreads)
            sum = fma(value_of<TS>(__ldg(a.val + e), a.vtab), (TS)gather_m<MODE, HALO>(a, x, __ldg(a.col + e)), sum);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        __syncthreads();                       // red_s free from the previous row
        if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = (double)sum;
        __syncthreads();
        if (threadIdx.x == 0) {
            TS tot = 0;
#pragma unroll
            for (int w = 0; w < kThreads / 32; ++w) tot += (TS)red_s[w];
            store_row<MODE>(a, r, tot, acc);
        }
    }
}

// ---- multi-GPU: this rank's side of the exchanges, done by the consumer kernel itself --------
__device__ __forceinline__ void xchg_st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// all CTAs: pack + push a slice of the boundary values; last CTA: release the consumers' flags
template <class P>
__device__ __forceinline__ void halo_push(const CsrArgsT<P> &a) {
    if (!a.push_seq) return;
    const typename P::TX *__restrict__ x = a.x;
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < a.n_send; i += gridDim.x * kThreads) {
        const typename P::TX v = x[a.send_idx[i]];
#pragma unroll 1
        for (int q = 0; q < a.nranks; ++q)
            if (a.push_data[q]) a.push_data[q][i] = v;
    }
    __threadfence_system();                   // my peer stores are visible system-wide ...
    __shared__ bool push_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(a.push_ticket, 1u);    // ... before the ticket moves
        push_last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (push_last) {
        // (st.release.sys orders everything that happens-before it -- all CTAs' stores, via
        // their fences and the ticket -- before the flag)
        if (threadIdx.x < a.nranks && a.push_flag[threadIdx.x])
            xchg_st_release_sys(a.push_flag[threadIdx.x], a.push_seq);
        if (threadIdx.x == 0) *a.push_ticket = 0;
    }
}
// end of a kernel that stored row shares into the peers' gather buffers
template <class P>
__device__ __forceinline__ void gather_finish(const CsrArgsT<P> &a) {
    __threadfence_system();
    __shared__ bool gather_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(a.gather_ticket, 1u);
        gather_last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (gather_last) {
        if (threadIdx.x < a.nranks && a.gather_flag[threadIdx.x])
            xchg_st_release_sys(a.gather_flag[threadIdx.x], a.gather_seq);
        if (threadIdx.x == 0) *a.gather_ticket = 0;
    }
}

// ---- variant 0: one row block per CTA -----------------------------------------------
template <int MODE, int L, bool HALO, class P>
__global__ void __launch_bounds__(kThreads, 4) csr_block_kernel(const CsrArgsT<P> a) {
    extern __shared__ __align__(128) char smem[];
    uint64_t *bar   = reinterpret_cast<uint64_t *>(smem);
    double   *red_s = reinterpret_cast<double *>(smem + 64);
    char     *stage = smem + kHeaderBytes;
    const StageLayout lay = stage_layout(a.rows_cap, a.nnz_cap, (int)sizeof(typename P::TV));

    const int b = blockIdx.x;
    const BlockDesc d = load_desc(a, b);          // broadcast loads, uniform
    const bool staged = (d.e1 - d.e0) <= a.nnz_cap;
    RowAcc acc = {0.0, 0.0};                      // (this variant produces no scalars)

    if (staged) {
        if (threadIdx.x == 0) {
            ptx::mbar_init(bar, 1);
            ptx::fence_mbar_init();
            issue_block(a, d, stage, lay, bar, ptx::policy_evict_first());
        }
        __syncthreads();
        ptx::mbar_wait(bar, 0);
        wait_for_halo<HALO>(a, d);
        compute_staged<MODE, L, HALO>(a, d, stage, lay, acc);
    } else {
        wait_for_halo<HALO>(a, d);
        compute_long<MODE, HALO>(a, d, red_s, acc);
    }
}

// ---- variant 1: persistent CTAs, S-deep ring of stages ----------------------------------
// FMT: storage format of the columns (FMT_*, see the top of the file)
template <int MODE, int L, bool HALO, class P, int FMT = FMT_PLAIN>
__global__ void __launch_bounds__(kThreads, 4) csr_ring_kernel(const CsrArgsT<P> a, const int nstages) {
    extern __shared__ __align__(128) char smem[];
    uint64_t  *bars  = reinterpret_cast<uint64_t *>(smem);                 // [<=8]
    double    *red_s = reinterpret_cast<double *>(smem + 64);              // [8]
    BlockDesc *descs = reinterpret_cast<BlockDesc *>(smem + 128);          // [<=8]
    unsigned  *done  = reinterpret_cast<unsigned *>(smem + 384);           // [<=8] warps done with a stage
    const StageLayout lay = stage_layout(a.rows_cap, a.nnz_cap, (int)sizeof(typename P::TV), FMT, a.run_cap);
    char *stages = smem + kHeaderBytes;
    // behind the stages: the window of x (FMT_WINDOW), the offset table (FMT_OFFSET), or the
    // patterns' offsets followed by the patterns' first entries (FMT_PATTERN)
    typename P::TX *win = reinterpret_cast<typename P::TX *>(stages + (size_t)nstages * lay.bytes);
    int *off_s = reinterpret_cast<int *>(stages + (size_t)nstages * lay.bytes);
    unsigned short *pstart_s = reinterpret_cast<unsigned short *>(off_s + kPatOffCap);
    // ... and behind those an indexed operator's table of values
    constexpr bool IDX = IndexedValues<typename P::TV>::value;
    static_assert(FMT != FMT_PATVAL, "value-keyed patterns run csr_patval_kernel");
    static_assert(!(IDX && (HALO || FMT == FMT_WINDOW)), "indexed values: single-GPU, fixed-size tables only");
    double *vtab_s = reinterpret_cast<double *>(stages + (size_t)nstages * lay.bytes +
                                                fmt_table_bytes(FMT, (int)sizeof(typename P::TV)));

    const int first = blockIdx.x;
    const int step  = gridDim.x;
    const int mine  = (a.nblocks - first + step - 1) / step;   // blocks this CTA owns
    const uint64_t policy = ptx::policy_evict_first();     // (any warp's first lane may issue a refill)

    // PDL: the prologue below only reads matrix data (never written by a kernel), so it may
    // run before the predecessor's writes are visible
    if (threadIdx.x == 0) {
        for (int s = 0; s < nstages; ++s) { ptx::mbar_init(bars + s, 1); done[s] = 0; }
        ptx::fence_mbar_init();
        const int pre = mine < nstages ? mine : nstages;
        for (int i = 0; i < pre; ++i) {
            const BlockDesc d = load_desc<FMT>(a, first + i * step);
            descs[i] = d;
            issue_block<FMT>(a, d, stages + (size_t)i * lay.bytes, lay, bars + i, policy);
        }
    }
    if constexpr (FMT == FMT_OFFSET) {
        static_assert(kOffTabLen == kThreads, "one table entry per thread");
        off_s[threadIdx.x] = __ldg(a.off_tab + threadIdx.x);
    }
    if constexpr (FMT == FMT_PATTERN) {
        for (int i = threadIdx.x; i < a.pat_total; i += kThreads) off_s[i] = __ldg(a.pat_off + i);
        for (int i = threadIdx.x; i <= kPatCap; i += kThreads) pstart_s[i] = __ldg(a.pat_start + i);
    }
    if constexpr (IDX) {
        for (int i = threadIdx.x; i < a.vtab_n; i += kThreads) vtab_s[i] = __ldg(a.vtab + i);
    }
    __syncthreads();
    ptx::pdl_wait();         // vectors (x, f, d, y) come from earlier kernels: from here on
    if (HALO) halo_push(a);  // multi-GPU: my boundary values go out before anything else

    // The rows of the blocks a CTA walks form one stream, cut into chunks of one warp's worth of
    // rows (32 / L); chunk k of the stream goes to warp k % 8 (compute_staged), a fixed function of
    // the blocks' row counts, so the in-kernel scalars stay deterministic.
    // Decoupled: no CTA barrier between blocks.  A warp that is done with its chunks of a block
    // moves on to the next stage at once, and the LAST warp to finish refills the stage.  Warps
    // thus stay busy when a block has fewer rows than the CTA has row groups (long-row operators:
    // about 68 rows per block for 128 groups at 2 lanes per row, DESIGN.md section 3.1b).
    // Every warp waits on and arrives for every block, also one it has no chunk of: it reads the
    // block's descriptor, and no warp may fall a whole phase of a stage's mbarrier behind.
    // A long block (plain format) takes the whole CTA: the barriers of compute_long drain the
    // stream up to it.  Offset- and pattern-indexed operators always run decoupled; plain and
    // narrow ones where most blocks leave a warp without rows (a.row_stream, set at upload):
    // where every warp has rows anyway (the prolongation of the finest level, 256 rows of about 4
    // entries per block) the block-synchronous release measured faster.  The windowed format fills
    // its window with the whole CTA: block-synchronous.
    const bool decoupled = FMT == FMT_OFFSET || FMT == FMT_PATTERN ||
                           (FMT != FMT_WINDOW && a.row_stream);
    constexpr int LS = FMT == FMT_PLAIN || L < 16 ? L : 8;   // (compressed formats: at most 8 lanes)
    RowAcc acc = {0.0, 0.0};
    int k0 = 0;                    // the current block's first chunk in the CTA's stream of rows
    int s = 0, parity = 0;
    for (int i = 0; i < mine; ++i) {
        ptx::mbar_wait(bars + s, parity);
        const BlockDesc d = descs[s];
        wait_for_halo<HALO>(a, d);
        const char *stage = stages + (size_t)s * lay.bytes;
        if constexpr (FMT == FMT_WINDOW) {
            fill_window<MODE, HALO>(a, d, stage, lay, win);
            compute_staged<MODE, LS, HALO, P, FMT_WINDOW>(a, d, stage, lay, acc, win);
        } else if (FMT != FMT_PLAIN || (d.e1 - d.e0) <= a.nnz_cap) {
            compute_staged<MODE, LS, HALO, P, FMT>(a, d, stage, lay, acc, nullptr, off_s, pstart_s, k0, vtab_s);
            k0 += (d.r1 - d.r0 + 32 / LS - 1) / (32 / LS);
        } else {
            compute_long<MODE, HALO>(a, d, red_s, acc);
        }
        if (decoupled) {
            // its arrive.expect_tx (release) / the others' wait (acquire) on the stage's mbarrier
            // publish the new descriptor; the counter orders everyone's reads of the stage before
            // the refill
            __syncwarp();
            if ((threadIdx.x & 31) == 0) {
                __threadfence_block();
                const unsigned arrived = atomicAdd(done + s, 1u);
                if (arrived == kThreads / 32 - 1) {
                    done[s] = 0;
                    __threadfence_block();
                    if (i + nstages < mine) {
                        const BlockDesc n = load_desc<FMT>(a, first + (i + nstages) * step);
                        descs[s] = n;
                        issue_block<FMT>(a, n, stages + (size_t)s * lay.bytes, lay, bars + s, policy);
                    }
                }
            }
        } else {
            __syncthreads();             // every thread is done with stage s, descs[s], the window
            if (threadIdx.x == 0 && i + nstages < mine) {
                const BlockDesc n = load_desc<FMT>(a, first + (i + nstages) * step);
                descs[s] = n;
                issue_block<FMT>(a, n, stages + (size_t)s * lay.bytes, lay, bars + s, policy);
            }
        }
        if (++s == nstages) { s = 0; parity ^= 1; }
    }
    if (HALO && a.gather_on) gather_finish(a);
    if (a.ndot) {
        double v[2] = {acc.s0, acc.s1};
        red_finish<2>(a.red, v);
    }
}

// ---- value-keyed patterns (FMT_PATVAL): persistent CTAs without a ring ---------------------------
// Such an operator streams one pattern id per row and nothing per entry, so there is nothing to
// stage: each thread loads the ids of its rows itself and keeps several rows in flight.
//
// Same rows per thread, in the same order, as csr_ring_kernel on FMT_PATTERN (hence the same bits):
// the same grid, CTA b walks the blocks b, b + grid, ..., chunk j of a block goes to warp (k0 + j) % 8
// with k0 the CTA's running chunk count, and lane l of a group takes the entries l, l + L, ... of
// its row.  A thread's rows form a software pipeline, R at a time (normally from R consecutive
// blocks): the ids of the next batch are requested before the gathers of the current one.

// rows a thread reduces together; RESID_SCALED forms every gathered value from two loads
template <int MODE> struct PatvalBatch { static constexpr int R = MODE == MODE_RESID_SCALED ? 1 : 2; };

// pattern id of a row: read once per pass, so not kept in L1 and first out of L2 (policy:
// ptx::policy_evict_first())
__device__ __forceinline__ int ld_pid(const unsigned char *p, uint64_t policy) {
    unsigned v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(policy));
    return (int)v;
}

template <int MODE, int L, class P>
__global__ void __launch_bounds__(kThreads, 4) csr_patval_kernel(const CsrArgsT<P> a) {
    typedef typename P::TV TV;
    typedef typename P::TX TX;
    typedef typename P::TY TS;                       // row sums live in the output's type
    static_assert(L == 1 || L == 2 || L == 4, "value-keyed patterns: 1, 2 or 4 lanes per row");
    static_assert(!IndexedValues<TV>::value, "value-keyed patterns keep the values themselves");
    constexpr int R  = PatvalBatch<MODE>::R;
    constexpr int K  = L == 1 ? 2 * kGatherBatch : kGatherBatch;   // entries per lane and row per round
    constexpr int CR = 32 / L;                       // rows per chunk
    constexpr int NW = kThreads / 32;
    extern __shared__ __align__(128) char smem[];
    int *off_s = reinterpret_cast<int *>(smem);      // the patterns' offsets,
    unsigned short *pstart_s = reinterpret_cast<unsigned short *>(off_s + kPatOffCap);   // first entries
    TV *pval_s = reinterpret_cast<TV *>(smem + kPatTabBytes);   // and the entries' values

    const int first = blockIdx.x;
    const int step  = gridDim.x;
    const int mine  = (a.nblocks - first + step - 1) / step;   // blocks this CTA owns
    const int warp  = threadIdx.x >> 5;
    const int wl    = threadIdx.x & 31;
    const int g     = wl / L;                        // the thread's row in a chunk
    const int lane  = threadIdx.x % L;

    // The walk.  Lane t of every warp holds the rows [r0, r1) of the CTA's blocks wb + t and
    // wb + 32 + t, wb a multiple of 32: a block's rows come from a shuffle, and the next 32 are
    // requested 32 blocks before they are needed.
    auto block_rows = [&](int i) -> int2 {
        if (i >= mine) return make_int2(0, 0);
        const int4 q = __ldg(a.blk + first + i * step);   // (single GPU: never a halo block)
        return make_int2(q.x, q.y);
    };
    int2 win_n = block_rows(wl), win_c = make_int2(0, 0);
    int i = -1, r0 = 0, r1 = 0, k0 = 0, j = 0;       // current block, its rows, its first chunk, my next chunk
    // this thread's next row: -1 if its group has none in the warp's next chunk, -2 at the end of
    // the walk (both warp-uniform but the -1)
    auto next_row = [&]() -> int {
        while (j * CR >= r1 - r0) {                  // no chunk of the current block left for this warp
            k0 += (r1 - r0 + CR - 1) / CR;
            if (++i >= mine) return -2;
            if ((i & 31) == 0) { win_c = win_n; win_n = block_rows(i + 32 + wl); }
            r0 = __shfl_sync(0xffffffffu, win_c.x, i & 31);
            r1 = __shfl_sync(0xffffffffu, win_c.y, i & 31);
            j = (warp - k0) & (NW - 1);
        }
        const int r = r0 + j * CR + g;
        j += NW;
        return r < r1 ? r : -1;
    };

    // PDL: the tables and the first batch's ids are matrix data, never written by a kernel
    const uint64_t policy = ptx::policy_evict_first();
    for (int e = threadIdx.x; e < a.pat_total; e += kThreads) {
        off_s[e] = __ldg(a.pat_off + e);
        pval_s[e] = __ldg(a.pat_val + e);
    }
    for (int e = threadIdx.x; e <= kPatCap; e += kThreads) pstart_s[e] = __ldg(a.pat_start + e);
    int row[R], pid[R];
#pragma unroll
    for (int u = 0; u < R; ++u) row[u] = next_row();
#pragma unroll
    for (int u = 0; u < R; ++u) pid[u] = row[u] >= 0 ? ld_pid(a.pid + row[u], policy) : 0;
    __syncthreads();
    ptx::pdl_wait();         // vectors (x, f, d, y) come from earlier kernels: from here on

    const TX *__restrict__ x = a.x;
    RowAcc acc = {0.0, 0.0};
    while (row[0] != -2) {
        // the next batch's ids travel with this batch's gathers
        int nrow[R], npid[R];
#pragma unroll
        for (int u = 0; u < R; ++u) nrow[u] = next_row();
#pragma unroll
        for (int u = 0; u < R; ++u) npid[u] = nrow[u] >= 0 ? ld_pid(a.pid + nrow[u], policy) : 0;
        RowOps<P> ops[R];
        int beg[R], end[R], len = 0;
        TS sum[R];
#pragma unroll
        for (int u = 0; u < R; ++u) {
            const bool valid = row[u] >= 0;
            ops[u] = valid && lane == 0 ? load_row_ops<MODE>(a, row[u]) : RowOps<P>{};
            beg[u] = valid ? (int)pstart_s[pid[u]] : 0;
            end[u] = valid ? (int)pstart_s[pid[u] + 1] : 0;
            len = max(len, end[u] - beg[u]);
            sum[u] = 0;
        }
        // K entries of every row per round, all the rows' gathers back to back, then the FMAs of
        // each row in entry order (the values from shared memory when they are needed)
        for (int k = lane; k < len; k += K * L) {
            TX xv[R][K];
#pragma unroll
            for (int u = 0; u < R; ++u)
#pragma unroll
                for (int q = 0; q < K; ++q) {
                    const int e = beg[u] + k + q * L;
                    xv[u][q] = e < end[u] ? gather_m<MODE, false>(a, x, row[u] + off_s[e]) : (TX)0;
                }
#pragma unroll
            for (int u = 0; u < R; ++u)
#pragma unroll
                for (int q = 0; q < K; ++q) {
                    const int e = beg[u] + k + q * L;
                    if (e < end[u]) sum[u] = fma((TS)pval_s[e], (TS)xv[u][q], sum[u]);
                }
        }
        if (L > 1) {
#pragma unroll
            for (int o = L / 2; o > 0; o >>= 1) {
#pragma unroll
                for (int u = 0; u < R; ++u) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
            }
        }
#pragma unroll
        for (int u = 0; u < R; ++u)
            if (row[u] >= 0 && lane == 0) store_row<MODE>(a, row[u], sum[u], acc, ops[u]);
#pragma unroll
        for (int u = 0; u < R; ++u) { row[u] = nrow[u]; pid[u] = npid[u]; }
    }
    if (a.ndot) {
        double v[2] = {acc.s0, acc.s1};
        red_finish<2>(a.red, v);
    }
}

// ---- x == 0 shortcut of the smoother sweep: x = (omega*d).*rhs ---------------------------
template <class TD, class TF, class TX>
__global__ void __launch_bounds__(kThreads) relax_zero_kernel(size_t n, double omega,
                                                              const TD *__restrict__ d,
                                                              const TF *__restrict__ f,
                                                              TX *__restrict__ x) {
    ptx::pdl_wait();
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        // (omega*d)*(f - 0) + 0, written as the reference evaluates it
        x[i] = fma((TX)(omega * d[i]), (TX)f[i], (TX)0);
    }
}

} // namespace b200
