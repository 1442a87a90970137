// internal.cuh -- host-side plumbing shared by the api_*.cu translation units: error
// reporting, the device guard, per-launch profiling brackets, lazy-clear bookkeeping, graph
// recording state, the launch helper and the functions one unit calls in another.
#pragma once
#include "common.cuh"
#include "dist.cuh"
#include "reduce.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <limits>
#include <new>
#include <string>
#include <vector>

namespace b200 {

// device guard: every entry point runs with the context's device current
struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
        if (prev != dev) ok = (cudaSetDevice(dev) == cudaSuccess);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

constexpr size_t kProfMaxPairs = 1 << 17;

// Bracket one launch with a pair of events on the launching stream (profiling only).
struct ProfScope {
    b200_ctx_t ctx;
    bool on = false;
    size_t ev = 0;
    int64_t nrows, ncols, nnz;
    int mode;
    int fmt;            // CSR passes: the column format streamed (FMT_*)
    int vbytes;         // ... and the bytes of one stored value (0 for the other kernels)
    ProfScope(b200_ctx_t c, int mode_, int64_t nr, int64_t nc, int64_t nz, int fmt_ = 0, int vbytes_ = 0)
        : ctx(c), nrows(nr), ncols(nc), nnz(nz), mode(mode_), fmt(fmt_), vbytes(vbytes_) {
        if (!ctx->profiling || ctx->prof_recs.size() >= kProfMaxPairs) return;
        while (ctx->prof_events.size() < ctx->prof_used + 2) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return;
            ctx->prof_events.push_back(e);
        }
        ev = ctx->prof_used;
        if (cudaEventRecord(ctx->prof_events[ev], ctx->stream) != cudaSuccess) return;
        on = true;
    }
    ~ProfScope() {
        if (!on) return;
        if (cudaEventRecord(ctx->prof_events[ev + 1], ctx->stream) != cudaSuccess) return;
        ctx->prof_used += 2;
        ctx->prof_recs.push_back({nrows, ncols, nnz, mode, ev, fmt, vbytes});
    }
};

// ---- implemented in api_tail.cu: deferred execution of calls on small operators --------------
int  tail_flush(b200_ctx_t ctx);        // run the pending commands (one launch); no-op if none
void tail_destroy(b200_ctx_t ctx);
bool tail_enabled(b200_ctx_t ctx);
bool tail_accepts_csr(b200_ctx_t ctx, b200_csr_t A);
int  tail_enqueue_relax_zero(b200_ctx_t ctx, size_t n, double omega, const double *d, const double *f, double *x);
int  tail_enqueue_gemv(b200_ctx_t ctx, int n, const double *Ainv, const double *rhs, double *x);

// Calls that touch memory the caller can see behind the library's back (wrapped external
// storage, vectors whose raw pointer was handed out) are never deferred: their effects must be
// on the stream when the call returns.
struct TailHold {
    b200_ctx_t ctx;
    bool prev;
    TailHold(b200_ctx_t c, std::initializer_list<b200_vec_t> vs) : ctx(c), prev(c->tail_hold) {
        for (b200_vec_t v : vs)
            if (v && (!v->owned || v->escaped)) ctx->tail_hold = true;
    }
    ~TailHold() { ctx->tail_hold = prev; }
};

// ---- implemented in api_coarse_lu.cu: the coarsest level above the dense inverse's size -----
constexpr int64_t kCoarseDenseMax = 16384;   // largest n the dense inverse takes
int  coarse_lu_create(b200_ctx_t ctx, int64_t n, const std::vector<int32_t> &ptr,
                      const std::vector<int32_t> &col, const std::vector<double> &val,
                      b200_coarse_s *S);
int  coarse_lu_solve(b200_ctx_t ctx, b200_coarse_s *S, b200_vec_t rhs, b200_vec_t x);
void coarse_lu_destroy(CoarseLu *lu);

// ---- implemented in api_matrices.cu: the lazy first smoother sweep ---------------------------
int  lazy_flush(b200_ctx_t ctx);        // write out the pending x = (omega*d).*f, if any

// Lazy clear bookkeeping ------------------------------------------------------
inline int materialize(b200_vec_t v) {
    if (v->scale_pending) {
        const int lrc = lazy_flush(v->ctx);
        if (lrc) return lrc;
    }
    if (v->zero_pending) {
        if (v->len) {
            const int trc = tail_flush(v->ctx);       // the memset must follow what was deferred
            if (trc) return trc;
            ProfScope prof(v->ctx, B200_PROF_MEMSET, (int64_t)v->len, 1, 0);
            B200_CUDA(cudaMemsetAsync(v->ptr, 0, v->len * v->esz, v->ctx->stream));
        }
        v->zero_pending = false;
    }
    return B200_OK;
}
// pointer for reading (or read-modify-write)
inline int rd(b200_vec_t v, const double **p) {
    int rc = materialize(v);
    *p = v->ptr;
    return rc;
}
// pointer for a full overwrite
inline double *wr(b200_vec_t v) {
    v->zero_pending = false;
    v->gen++;
    return v->ptr;
}
// pointer for an in-place update (the caller has materialised a pending clear)
inline double *mut(b200_vec_t v) {
    v->gen++;
    return v->ptr;
}
// typed views (FP32 vectors keep their floats behind the same pointer)
template <class T> inline T *tp(double *p) { return reinterpret_cast<T *>(p); }
template <class T> inline const T *tp(const double *p) { return reinterpret_cast<const T *>(p); }
inline bool all64(std::initializer_list<b200_vec_t> vs) {
    for (b200_vec_t v : vs) if (v->dtype != B200_F64) return false;
    return true;
}
inline bool all32(std::initializer_list<b200_vec_t> vs) {
    for (b200_vec_t v : vs) if (v->dtype != B200_F32) return false;
    return true;
}

// CUDA-graph recording -----------------------------------------------------------
// The library keeps two pieces of host-side state per vector that decide WHICH kernels run and
// on WHICH addresses: the storage pointer (b200_relax trades x's storage with tmp's) and the
// lazy-clear flag.  A recorded graph bakes both in, so it remembers the state every object it
// touched had on entry (the graph may only be replayed from exactly that state) and the state
// the recorded calls left behind (applied after each replay).
struct GraphSlot {
    double **slot;      // &vec->ptr or &csr->scratch64
    bool    *zp;        // &vec->zero_pending (nullptr for operator scratch)
    double  *p0; bool z0;   // on entry
    double  *p1; bool z1;   // on exit
    uint64_t *gen;      // &vec->gen (nullptr for operator scratch): bumped by every replay
};
struct GraphProduct { b200_vec_t a, b; int slot; };   // product a replay leaves in the scalar table
} // namespace b200

struct b200_graph_s {
    b200_ctx_t ctx = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    std::vector<b200::GraphSlot> slots;
    std::vector<b200::GraphProduct> products;
    uint64_t destroy_epoch = 0, option_epoch = 0;
    uint64_t launches0 = 0;     // ctx->launches when recording started
    uint64_t launches = 0;      // kernels in the graph
    size_t   nodes = 0;
    uint64_t replays = 0;
};

namespace b200 {

inline void touch_slot(b200_ctx_t ctx, double **slot, bool *zp, uint64_t *gen = nullptr) {
    b200_graph_s *g = ctx->recording;
    for (const GraphSlot &s : g->slots)
        if (s.slot == slot) return;
    g->slots.push_back({slot, zp, *slot, zp ? *zp : false, nullptr, false, gen});
}
inline void touch(b200_ctx_t ctx, std::initializer_list<b200_vec_t> vs) {
    if (!ctx->recording) return;
    for (b200_vec_t v : vs) {
        touch_slot(ctx, &v->ptr, &v->zero_pending, &v->gen);
        v->in_graph = true;
    }
}

inline int grid_for(const b200_ctx_t ctx, size_t n_items, int per_thread_items) {
    // enough CTAs to cover the range once, capped at 8 CTAs per SM (2048 threads)
    size_t want = (n_items + (size_t)kThreads * per_thread_items - 1) /
                  ((size_t)kThreads * per_thread_items);
    size_t cap = (size_t)ctx->sm_count * 8;
    if (want < 1) want = 1;
    return (int)std::min(want, cap);
}

} // namespace b200

namespace b200 {

// ---- peer-memory exchange buffers (layout: [flags 256 B | parity 0 | parity 1]) ------------
inline unsigned long long *flag_at(void *base, int parity, int slot) {
    return reinterpret_cast<unsigned long long *>(base) + parity * kFlagStride + slot;
}
inline char *data_at(void *base, int parity, size_t half_bytes) {
    return static_cast<char *>(base) + kFlagBytes + (size_t)parity * half_bytes;
}

// Launch with programmatic stream serialization (PDL) when enabled: the kernel may be
// scheduled while its predecessor drains and orders itself with griddepcontrol.wait.
template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(b200_ctx_t ctx, void (*kernel)(KArgs...), dim3 grid, dim3 block,
                              size_t smem, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed =
        (ctx->opt_pdl && (!ctx->recording || ctx->opt_graph_pdl)) ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// ---- implemented in api_krylov.cu: the device scalar table and in-kernel reductions ----------
int  scal_create(b200_ctx_t ctx);                  // allocate the table (context creation)
void scal_destroy(b200_ctx_t ctx);
int  scal_alloc(b200_ctx_t ctx, int count);        // first of `count` consecutive free slots, -1 if none
void scal_free(b200_ctx_t ctx, int first, int count);
// RedOut for one launch that leaves `nred` scalars in the given table slots
// (across_ranks: the operands are partitioned, every rank launches the same kernel and the
// finishing CTAs all-reduce over the peers)
// host_mask: bit k set = scalar k is also written to the mapped host mirror (only where the
// host reads it right after a synchronize: a write over PCIe lengthens the kernel's tail)
void red_out(b200_ctx_t ctx, int nred, const int *slots, RedOut &o, bool across_ranks,
             unsigned host_mask = 0);
// value of a table slot on the host (synchronises; copies from the device unless mirrored)
int  scal_read(b200_ctx_t ctx, int slot, bool mirrored, double *out);
// products left behind by producer kernels (see b200_ctx_s::Product)
bool product_wanted(b200_ctx_t ctx, size_t n);
int  product_take_slot(b200_ctx_t ctx);
void product_record(b200_ctx_t ctx, b200_vec_t a, b200_vec_t b, int slot);
int  product_lookup(b200_ctx_t ctx, b200_vec_t a, b200_vec_t b);   // slot or -1
// one standalone reduction launch: <x,y> (and <x,z> when z != nullptr) into table slots
int  launch_dot_slots(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y, b200_vec_t z, const int *slots,
                      unsigned host_mask = 0);
// (api_vectors.cu) stand-alone dot kernel: FP32 vectors, NCCL transport
int  dot_legacy(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y, double *result);

// ---- implemented in api_matrices.cu: streaming passes that also leave scalars behind ----------
int  spmv_with_dots(b200_ctx_t ctx, b200_csr_t A, b200_vec_t x, b200_vec_t y, b200_vec_t w, int ndot,
                    const int *slots);
int  residual_with_norm(b200_ctx_t ctx, b200_vec_t f, b200_csr_t A, b200_vec_t x, b200_vec_t r, int slot);

// ---- implemented in api_exchange.cu (multi-GPU) ----------------------------------------------
int  peer_alloc(b200_ctx_t ctx, size_t bytes, void **local, void **peers);
void peer_release(b200_ctx_t ctx, void *local, void **peers);
// what halo_exchange hands to the consumer kernel (copied into its CsrArgs)
struct HaloArgs {
    const void               *xh = nullptr;         // halo values for columns >= nloc (x's element type)
    int                       nloc = 0;
    const unsigned long long *wait_flags = nullptr;
    unsigned int              wait_mask = 0;
    unsigned long long        wait_seq = 0;
    // peer transport: this rank's boundary values are pushed by the consumer kernel itself
    const int                *send_idx = nullptr;
    int                       n_send = 0;
    int                       nranks = 0;
    void                     *push_data[kMaxRanks] = {};
    unsigned long long       *push_flag[kMaxRanks] = {};
    unsigned int             *push_ticket = nullptr;
    unsigned long long        push_seq = 0;
};
int  halo_exchange(b200_ctx_t ctx, b200_csr_t A, const void *x, size_t esz, HaloArgs &a);
// row shares of a replicated result
struct GatherArgs {
    int                 on = 0;                     // peer transport: kernel stores into the peers
    int                 nranks = 0;
    void               *data[kMaxRanks] = {};       // (y's element type)
    unsigned long long *flag[kMaxRanks] = {};
    unsigned int       *ticket = nullptr;
    unsigned long long  seq = 0;
    void               *y_local = nullptr;          // where the kernel's plain store of a row goes
};
int  gather_begin(b200_ctx_t ctx, b200_csr_t A, size_t esz, GatherArgs &g);
int  gather_end(b200_ctx_t ctx, b200_csr_t A, const GatherArgs &g, b200_vec_t y);
int  dist_dot_finish(b200_ctx_t ctx, double *result);

} // namespace b200

#define CHECK_CTX(ctx) B200_REQUIRE((ctx) != nullptr, "null context")
#define B200_NCCL(call)                                                        \
    do {                                                                       \
        ncclResult_t rc__ = (call);                                            \
        if (rc__ != ncclSuccess)                                               \
            return fail(B200_ENCCL, std::string("NCCL error in " #call ": ") + \
                                        nccl().GetErrorString(rc__));          \
    } while (0)
inline ncclComm_t comm_of(b200_ctx_t ctx) { return static_cast<ncclComm_t>(ctx->comm); }
inline bool same_layout(b200_vec_t a, b200_vec_t b) {
    return a->n == b->n && a->kind == b->kind && a->len == b->len;
}
#define NOT_RECORDING(ctx, what)                                                        \
    B200_REQUIRE(!(ctx)->recording, what ": not allowed while a graph is being recorded")
// Every entry point that touches the device runs under GUARD: the context's device is made
// current and whatever was deferred into the coarse-tail list is launched first, so effects
// reach the stream in call order.  The four entry points that may themselves be deferred
// (b200_spmv, b200_residual, b200_relax, b200_coarse_solve) use GUARD_DEFER and flush on
// every path that launches immediately.
#define GUARD_RAW(ctx)                                                         \
    DeviceGuard guard__((ctx)->device);                                        \
    if (!guard__.ok) return fail(B200_ECUDA, "cudaSetDevice failed")
#define GUARD_DEFER(ctx)                                                       \
    GUARD_RAW(ctx);                                                            \
    do {                                                                       \
        const int lrc__ = ::b200::lazy_flush(ctx);                             \
        if (lrc__) return lrc__;                                               \
    } while (0)
#define GUARD(ctx)                                                             \
    GUARD_DEFER(ctx);                                                          \
    do {                                                                       \
        const int trc__ = ::b200::tail_flush(ctx);                             \
        if (trc__) return trc__;                                               \
    } while (0)
#define B200_BAD_MIX(what) ::b200::fail(B200_EINVAL, what ": unsupported precision combination")
