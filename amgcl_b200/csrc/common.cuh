// common.cuh -- shared definitions for the H100 solve-phase backend.
//
// Device objects behind the opaque C handles of include/amgcl_b200.h, error
// plumbing, and the sm_90a PTX helpers (mbarrier + 1-D TMA bulk copies) the
// streaming kernels are built from.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <string>
#include <vector>

#include "../../include/amgcl_b200.h"
#include "../../include/amgcl_b200_formats.h"
#include "../../include/amgcl_b200_coarse.h"

namespace b200 {

// ---------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------
void set_error(const std::string &msg);
int  fail(int code, const std::string &msg);
int  cuda_fail(cudaError_t rc, const char *what, const char *file, int line);

#define B200_CUDA(call)                                                        \
    do {                                                                       \
        cudaError_t rc__ = (call);                                             \
        if (rc__ != cudaSuccess)                                               \
            return ::b200::cuda_fail(rc__, #call, __FILE__, __LINE__);         \
    } while (0)

#define B200_CHECK_LAUNCH()                                                    \
    do {                                                                       \
        cudaError_t rc__ = cudaGetLastError();                                 \
        if (rc__ != cudaSuccess)                                               \
            return ::b200::cuda_fail(rc__, "kernel launch", __FILE__, __LINE__); \
    } while (0)

#define B200_REQUIRE(cond, msg)                                                \
    do {                                                                       \
        if (!(cond)) return ::b200::fail(B200_EINVAL, msg);                    \
    } while (0)

// ---------------------------------------------------------------------------
// hardware constants (H100: 132 SMs, 227 KB smem / CTA)
// ---------------------------------------------------------------------------
constexpr int kThreads      = 256;    // threads per CTA in every streaming kernel
constexpr int kRowsCapMax   = 1024;   // most rows a row block may hold
constexpr int kNnzCapMax    = 6144;   // most non-zeros a staged row block may hold
constexpr int kDotMaxBlocks = 2048;   // upper bound on partial sums of one dot product
constexpr int kMaxRed       = 3;      // scalars one launch may produce (reduce.cuh)
constexpr int kScalSlots    = 256;    // device scalar table of a context (reduce.cuh)
struct ScalExchange;                  // multi-GPU exchange buffer of the scalar table

// multi-GPU peer-memory exchange buffers (peer.cuh): [flags 256 B | parity 0 | parity 1]
constexpr int kMaxRanks   = 16;
constexpr int kFlagStride = 16;                 // flag slots per parity (>= kMaxRanks)
constexpr size_t kFlagBytes = 2 * kFlagStride * sizeof(unsigned long long);   // 256 B header

} // namespace b200

// ---------------------------------------------------------------------------
// objects behind the opaque handles
// ---------------------------------------------------------------------------
struct b200_graph_s;

struct b200_ctx_s {
    int          device      = 0;
    int          sm_count    = 132;
    cudaStream_t own_stream  = nullptr;
    cudaStream_t stream      = nullptr;   // stream in use (own or external)
    uint64_t     launches    = 0;

    // dot product scratch: per-CTA partial sums, completion ticket, result
    double       *dot_partial = nullptr;  // [kDotMaxBlocks] device
    unsigned int *dot_ticket  = nullptr;  // device, self-resetting
    double       *dot_result_h = nullptr; // pinned + mapped host scalar(s)
    double       *dot_result_d = nullptr; // device alias of dot_result_h

    // device scalar table (reduce.cuh): results of reductions done inside the streaming
    // kernels stay on the device for the next kernel; the host reads the mapped mirror
    double       *scal_d  = nullptr;      // [kScalSlots] device
    double       *scal_h  = nullptr;      // [kScalSlots] pinned + mapped host mirror
    double       *scal_hd = nullptr;      // device alias of scal_h
    unsigned long long *scal_ready_h  = nullptr;   // [kScalSlots] mapped: seq of the value in scal_h
    unsigned long long *scal_ready_hd = nullptr;   // device alias
    double       *red_partial = nullptr;  // [kMaxRed * kDotMaxBlocks] per-CTA partial sums
    unsigned int *red_ticket  = nullptr;  // device, self-resetting
    bool          scal_used[b200::kScalSlots] = {};
    unsigned long long scal_seq[b200::kScalSlots] = {};   // uses of each slot so far (multi-GPU parity)
    b200::ScalExchange  *scal_x_local = nullptr;    // multi-GPU: exchange buffer (peer-mapped)
    void                *scal_x_peer[16] = {};
    b200::ScalExchange **scal_x_table = nullptr;    // device array [nranks] of the mapped buffers

    // products left behind by a producer kernel (the fused smoother sweep leaves <rhs, x_new>):
    // b200_dot / the Krylov steps take them instead of launching a reduction when the operands
    // are exactly the producer's and unmodified since (generation counters of the vectors)
    struct Product { b200_vec_t a = nullptr, b = nullptr; uint64_t gen_a = 0, gen_b = 0; int slot = -1; };
    Product       products[4];
    int           product_next = 0;
    int           product_slot0 = -1;     // first of the 4 table slots the products rotate through
    std::vector<size_t> krylov_sizes;     // sizes of the live Krylov workspaces (b200_krylov_*)

    b200_vec_t    lazy_vec = nullptr;     // the (single) vector with a pending lazy first sweep
    int64_t       opt_fuse_first_sweep = 1;   // b200_relax from x = 0 + b200_residual -> one pass
    uint64_t      fused_first_sweeps = 0;

    // coarse tail of the V-cycle (tail_kernels.cuh): calls on small operators are deferred into
    // a command list and run as ONE kernel when the next non-deferrable call arrives
    void         *tail = nullptr;         // TailArgs (host): the pending commands
    unsigned long long *tail_bar = nullptr;   // device: arrival counter of coarse_tail_kernel's barriers
    unsigned long long  tail_bar_count = 0;   // ... its value once everything launched so far has run
    uint64_t      tail_flushes = 0, tail_commands = 0;
    bool          tail_hold = false;      // the current call touches caller-owned memory: do not defer

    // pinned staging for uploads (csr_upload): two buffers, ping-pong
    void        *stage_host[2]  = {};
    cudaEvent_t  stage_event[2] = {};

    // optional per-launch timing of the CSR streaming kernels (b200_profile_*)
    bool                      profiling = false;
    std::vector<cudaEvent_t>  prof_events;      // pool, used pairwise
    size_t                    prof_used = 0;
    struct ProfRec { int64_t nrows, ncols, nnz; int mode; size_t ev; int fmt, vbytes; };
    std::vector<ProfRec>      prof_recs;

    // multi-GPU (dist.cuh): one process per GPU, this context's share of the job
    bool     dist          = false;
    int      rank          = 0;
    int      nranks        = 1;
    void    *comm          = nullptr;       // ncclComm_t
    int64_t  dist_min_rows = 0;             // dimensions >= this are partitioned
    double  *dot_dev       = nullptr;       // device scalar for the all-reduced dot product
    // peer-memory exchange (peer.cuh): enabled when CUDA IPC between the ranks works
    bool     p2p           = false;
    unsigned int *push_ticket = nullptr;    // device, self-resetting
    unsigned int *gather_ticket = nullptr;  // device, self-resetting (row-share gathers)
    void    *ipc_dev       = nullptr;       // device staging for IPC handle exchange
    void    *probe_pb_local = nullptr;      // small peer-mapped allocation that proves CUDA IPC works
    void    *probe_pb_peer[16] = {};
    std::vector<void *> deferred_free;      // IPC-exported allocations, freed with the context

    // tuning
    int64_t opt_spmv_variant  = 1;
    int64_t opt_fuse_relax    = 1;
    int64_t opt_zero_shortcut = 1;
    int64_t opt_nnz_cap       = 2048;
    int64_t opt_lanes         = 0;        // 0 = choose from average row length
    int64_t opt_ctas_per_sm   = 4;        // persistent variant: CTAs per SM
    int64_t opt_stages        = 2;        // persistent variant: ring depth
    int64_t opt_p2p           = 1;        // multi-GPU: exchange through mapped peer memory
    int64_t opt_pdl           = 1;        // programmatic dependent launch of the solve kernels
    int64_t opt_cycle_graph   = 1;        // the shim's preconditioner wrapper may record CUDA graphs
    int64_t opt_graph_pdl     = 1;        // keep the PDL attribute on launches recorded into a graph
    int64_t opt_coarse_tail   = 0;        // defer calls on small operators into one cooperative kernel
                                          // (opt-in: measured no faster than separate launches, DESIGN.md)
    int64_t opt_tail_max_nnz  = 1500000;  // ... "small": at most this many non-zeros
    int64_t opt_tail_max_vec  = 262144;   // ... element-wise x = 0 sweeps: at most this many entries
    int64_t opt_poll_scalars  = 1;        // host reads in-kernel reduction results by polling mapped memory
    int64_t big_nnz = -1;                 // the largest operator uploaded so far and the column
    int     big_fmt = 0;                  // format it is stored in (FMT_*; for the bench's roofline)
    int64_t opt_patterns      = 1;        // operators with <= 256 distinct row patterns: no per-entry columns
    int64_t opt_patterns_min_nnz = 1000000;// ... from this many non-zeros on (decided at upload)
    int64_t opt_pattern_values = 1;       // ... keyed on (offset, value) pairs where they fit: no per-entry
                                          //   values or row pointers either (single GPU; patterns.cuh)
    int64_t opt_offsets       = 1;        // operators with <= 256 distinct (col - row): 8-bit column indices
    int64_t opt_offsets_min_nnz = 1000000;// ... from this many non-zeros on (decided at upload)
    int64_t opt_narrow        = 1;        // other operators: 16- or 24-bit block-relative columns (narrow.cuh)
    int64_t opt_narrow_values = 1;        // FP64 operators whose values are all exact FP32: stream 4-byte values
    int64_t opt_narrow_values_min_nnz = 1000000;   // ... from this many non-zeros on (decided at upload)
    int64_t opt_window        = 0;        // operators that qualify gather x through shared-memory windows
    int64_t opt_window_min_nnz = 1000000; // ... "qualify": at least this many non-zeros (decided at upload),
    int64_t opt_window_ratio  = 75;       // ... windows no larger than this percentage of the entries,
    int64_t opt_window_gap    = 2;        // ... runs are merged across holes of (gap - 1) sectors
    int64_t opt_window_lanes  = 15;       // ... lanes per row in this set (bit k: 2^k lanes)
    int64_t opt_small_kernel_max_nnz = 0;         // FP64 operators up to this size: direct-load kernel
                                                  // (opt-in: measured slower than the ring kernel, DESIGN.md)
    int64_t opt_fused_krylov  = 1;        // the C++ binding's cg / bicgstab use the fused b200_cg_* / b200_bicg_* steps

    // CUDA-graph recording of a call sequence (b200_graph_*)
    b200_graph_s *recording   = nullptr;  // non-null between b200_graph_begin and _end / _abort
    std::vector<void *> graph_deferred;   // storage of vectors destroyed while recording
    uint64_t     destroy_epoch = 0;       // bumped when an object a graph refers to is destroyed
    uint64_t     option_epoch  = 0;       // bumped by b200_ctx_set_option / set_stream
};

// LOCAL: the whole vector lives on this GPU (single GPU, or a replicated level of a multi-GPU
// context); DIST: this rank's block of a partitioned vector
enum { B200_VK_LOCAL = 0, B200_VK_DIST = 1 };

struct b200_vec_s {
    b200_ctx_t ctx   = nullptr;
    double    *ptr   = nullptr;   // device storage; holds floats when dtype == B200_F32
    int        dtype = B200_F64;
    size_t     esz   = sizeof(double);
    size_t     n     = 0;         // global length
    size_t     len   = 0;         // elements stored on this rank (== n unless distributed)
    size_t     off   = 0;         // global index of ptr[0]
    size_t     cap   = 0;         // allocated elements (distributed: the uniform block)
    int        kind  = B200_VK_LOCAL;
    bool       owned = true;
    // Lazy clear: the vector is logically zero but the memset has not been
    // issued.  Set by b200_clear, consumed by b200_relax (which then skips the
    // A-pass), dropped by any full overwrite, materialised by any other read.
    bool       zero_pending = false;
    bool       in_graph     = false;   // some recorded graph refers to this vector
    // Lazy first sweep: the vector is logically x = (omega*d).*f (the smoother sweep from x = 0)
    // but nothing has been written.  Set by b200_relax, consumed by the b200_residual that
    // normally follows (which then forms x on the fly and writes it along with the residual:
    // one pass instead of two); ANY other call on the context materialises it first.
    bool       scale_pending = false;
    const double *sc_d = nullptr, *sc_f = nullptr;
    b200_vec_t sc_fvec = nullptr;
    double     sc_omega = 0.0;
    uint64_t   gen          = 0;       // bumped by every write through the library
    bool       escaped      = false;   // raw pointer handed out / external storage: contents
                                       // may change behind the library's back
};

// operators on a multi-GPU context (dist.cuh): LOCAL needs no exchange, HALO gathers remote
// columns from the all-gathered boundary values of a partitioned vector
enum { B200_CK_LOCAL = 0, B200_CK_HALO = 1 };

struct b200_csr_s {
    b200_ctx_t ctx   = nullptr;
    int64_t    nrows = 0, ncols = 0, nnz = 0;   // shape of the matrix the kernels see (local part)
    // distributed operators (dist.cuh)
    int        kind    = B200_CK_LOCAL;
    int64_t    gl_rows = 0, gl_cols = 0, gl_nnz = 0;   // global shape (what the API reports)
    bool       rows_dist = false;     // y is a partitioned vector (else replicated / single GPU)
    bool       cols_dist = false;     // x is a partitioned vector
    bool       gather_rows = false;   // y replicated but x partitioned: this rank computes a share
                                      //   of the rows, the shares are all-gathered
    int64_t    row_off = 0, row_B = 0;//   ... first row and uniform size of a share
    int64_t    n_loc   = 0;       // HALO: length of this rank's block of x (local columns)
    int64_t    S       = 0;       // HALO: halo slots per rank
    int64_t    n_send  = 0;       // HALO: entries this rank contributes
    int       *send_idx = nullptr;// HALO: [n_send] local indices to pack
    void      *halo    = nullptr; // HALO: [nranks*S] boundary values (x's element type) the kernel gathers from
    void      *halo_owned = nullptr; //     NCCL transport: private buffer (peer transport: inside pb)
    double    *ybuf    = nullptr; // gather_rows, NCCL transport: [nranks*row_B] all-gather buffer
    // peer-memory exchange state (peer.cuh); layout: [flags 256 B | parity 0 | parity 1]
    void      *pb_local = nullptr;    // halo of x
    void      *pb_peer[16] = {};
    size_t     pb_half  = 0;          // bytes of one parity buffer
    void      *gb_local = nullptr;    // gather_rows: the shares of y
    void      *gb_peer[16] = {};
    size_t     gb_half  = 0;
    unsigned long long seq = 0;       // halo exchanges done so far (same on every rank)
    unsigned long long gseq = 0;      // row gathers done so far
    bool       xchg[16] = {};         // ranks this rank exchanges halo values with (symmetric)
    int       *ptr   = nullptr;   // [nrows+1] (+ padding) device
    int       *col   = nullptr;   // [nnz]     (+ padding) device
    void      *val   = nullptr;   // [nnz]     (+ padding) device, FP64 or FP32
    float     *val32 = nullptr;   // [nnz]     (+ padding) FP64 operator whose every value is exactly an FP32:
                                  //   the values the ring kernel streams (same bits once widened)
    void      *vidx  = nullptr;   // [nnz]     (+ padding) FP64 operator with few distinct values: 8- or
    double    *vtab  = nullptr;   //   16-bit index of every value in vtab [vtab_n], the distinct values
    int        vidx_bytes = 0;    //   sorted by bit pattern (values.cuh); the values the ring kernel
    int        vtab_n     = 0;    //   streams where the table fits beside the ring
    int        dtype = B200_F64;
    double    *scratch64 = nullptr;   // FP32 operator swept on FP64 vectors: new iterate
    bool       in_graph  = false;     // some recorded graph refers to this operator
    // row-block plan
    int        lanes    = 1;      // lanes cooperating on one row (power of two <= 32)
    int        rows_cap = 256;    // rows per block   (multiple of kThreads / lanes)
    int        nnz_cap  = 2048;   // staged non-zeros per block
    int64_t    nblocks  = 0;
    int64_t    nlong    = 0;      // blocks too long to stage (handled by the strided path)
    bool       row_stream = false;// most blocks leave warps without rows: no CTA barrier between
                                  //   blocks (csr_ring_kernel)
    // windowed operators (csr_kernels.cuh): blocks gather x from a shared-memory window
    unsigned short *col16 = nullptr;  // [nnz] (+ padding) window-local column of every entry
    int2      *wrun     = nullptr;// runs of x the windows are made of {first column, len | slot << 16}
    int2      *wblk     = nullptr;// [nblocks] walk order: {first run, end run}
    int        win_slots = 0;     // largest window (elements of x)
    int        win_runs  = 0;     // most runs a block has
    int64_t    win_total = 0;     // sum of the window sizes (elements): traffic of the fills
    // offset-indexed columns (csr_kernels.cuh): col = row + off_tab[idx8]
    unsigned char *idx8 = nullptr;    // [nnz] (+ padding)
    int       *off_tab  = nullptr;    // [256] device
    int        off_count = 0;         // distinct (col - row) offsets
    // pattern-indexed rows (csr_kernels.cuh): col of the k-th entry of row r = r + pat_off[pat_start[pid[r]] + k]
    unsigned char  *pid       = nullptr;  // [nrows] (+ padding)
    unsigned short *pat_start = nullptr;  // [257] device
    int            *pat_off   = nullptr;  // [1024] device
    int        pat_count = 0, pat_total = 0;
    // value-keyed patterns (FMT_PATVAL): the value of the k-th entry of row r = pat_val[pat_start[pid[r]] + k]
    double         *pat_val   = nullptr;  // [1024] device (an FP32 operator's values widened)
    float          *pat_val32 = nullptr;  // [1024] device, the same values as FP32 where every one is exact
    // block-relative row pointers of every staged format: ptr16[r] = ptr[r] - first non-zero of r's block
    unsigned short *ptr16 = nullptr;  // [nrows] (+ padding)
    // block-relative columns (narrow.cuh): col = cbase[block] + clo16 (+ chi8 << 16)
    int        narrow   = 0;          // 16 / 24: width of the stored columns; 0: not narrowed
    unsigned short *clo16 = nullptr;  // [nnz] (+ padding) low 16 bits of col - base
    unsigned char  *chi8  = nullptr;  // [nnz] (+ padding) high 8 bits (width 24 only)
    int       *cbase    = nullptr;    // [nblocks] walk order: smallest column of the block
    int4      *blk      = nullptr;// [nblocks] device, walk order: {first row (~r if the block gathers halo
                                  //   columns), end row, first nnz, end nnz}; HALO: interior blocks first
    // every device array above, with the bytes allocated for it (csr_array): freed by csr_free,
    // summed into `bytes`
    std::vector<std::pair<void *, size_t>> arrays;
    size_t     bytes    = 0;
};

struct b200_index_s {
    b200_ctx_t ctx  = nullptr;
    size_t     n    = 0;          // number of indices
    size_t     range = 0;         // every index is < range (size of the indexed vector)
    int       *idx  = nullptr;    // [n] device
    void      *stage_d = nullptr; // [n] device staging for gathers that end on the host
    bool       in_graph = false;
};

namespace b200 { struct CoarseLu; }   // banded LU factor (api_coarse_lu.cu)

struct b200_coarse_s {
    b200_ctx_t ctx  = nullptr;
    int        kind = B200_COARSE_DENSE;  // which representation was built (from n alone)
    b200::CoarseLu *lu = nullptr;         // B200_COARSE_BANDED_LU: the factor and sweep state
    int        dtype = B200_F64;  // element type of the vectors it is applied to
    bool       replicated = false;// multi-GPU: coarsest level partitioned -> inverse on every rank
    double    *gbuf = nullptr;    // replicated: all-gathered right-hand side [nranks * block]
    int64_t    block = 0;
    int64_t    n    = 0;
    double    *Ainv = nullptr;    // [n*n] row-major device
    size_t     bytes = 0;
    bool       in_graph = false;
};

// ---------------------------------------------------------------------------
// PTX helpers: mbarrier, TMA 1-D bulk copy, L2 policies
// ---------------------------------------------------------------------------
namespace b200 {
namespace ptx {

__device__ __forceinline__ uint32_t smem_addr(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count)
                 : "memory");
}

// Make mbarrier initialisation visible to the async (TMA) proxy.
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// Order generic-proxy accesses to shared memory before subsequent async-proxy ones.
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)),
                 "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "B200_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra B200_DONE_%=;\n"
        "bra B200_WAIT_%=;\n"
        "B200_DONE_%=:\n"
        "}\n" ::"r"(smem_addr(bar)),
        "r"(parity)
        : "memory");
}

// L2 eviction policy for data streamed exactly once per kernel (matrix values
// and column indices): evict-first keeps them from displacing the gathered
// x-vector, which is reused by neighbouring rows and later kernels.
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier.
// dst and src must be 16-byte aligned and bytes a multiple of 16.  SASS: UBLKCP.
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes,
                                         uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
        "[%0], [%1], %2, [%3], %4;" ::"r"(smem_addr(dst)),
        "l"(src), "r"(bytes), "r"(smem_addr(bar)), "l"(policy)
        : "memory");
}

__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes,
                                         uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes "
        "[%0], [%1], %2, [%3];" ::"r"(smem_addr(dst)),
        "l"(src), "r"(bytes), "r"(smem_addr(bar))
        : "memory");
}

// Programmatic dependent launch (PDL): a kernel launched with
// cudaLaunchAttributeProgrammaticStreamSerialization is scheduled as soon as every CTA of its
// predecessor in the stream has exited, without waiting for the predecessor's end-of-grid
// memory flush; pdl_wait() then blocks until that flush is complete and the predecessor's
// writes are visible.  Everything a kernel does BEFORE pdl_wait() must only touch data that
// no kernel writes (matrix arrays, block descriptors): the ring kernels issue their first TMA
// bulk copies there, so the pipeline fill overlaps the flush.  A no-op for kernels launched
// without the attribute.  (An explicit early griddepcontrol.launch_dependents was measured
// and rejected: dependents that become resident early take SM resources from the running
// persistent grid; DESIGN.md section 3.3b.)
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// streaming (read-once) 16-byte global load that does not allocate in L1
__device__ __forceinline__ double2 ld_stream2(const double *p) {
    double2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];"
                 : "=d"(r.x), "=d"(r.y)
                 : "l"(p));
    return r;
}

} // namespace ptx
} // namespace b200
