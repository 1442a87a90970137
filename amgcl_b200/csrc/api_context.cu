// api_context.cu -- error state, contexts, options, profiling, graph recording
//
// Part of the implementation of the C ABI declared in include/amgcl_b200.h (host-side logic
// only: argument checking, bookkeeping, kernel launches; no CPU fallback anywhere).
#include "internal.cuh"

#include <mutex>

// ---------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------
namespace b200 {

static thread_local std::string g_last_error;

void set_error(const std::string &msg) { g_last_error = msg; }

int fail(int code, const std::string &msg) {
    g_last_error = msg;
    return code;
}

int cuda_fail(cudaError_t rc, const char *what, const char *file, int line) {
    char buf[512];
    snprintf(buf, sizeof(buf), "CUDA error %d (%s) in %s at %s:%d", (int)rc,
             cudaGetErrorString(rc), what, file, line);
    g_last_error = buf;
    cudaGetLastError();   // clear the sticky-less error state
    return rc == cudaErrorMemoryAllocation ? B200_ENOMEM : B200_ECUDA;
}

} // namespace b200

using namespace b200;

// ---------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------
extern "C" const char *b200_last_error(void) { return g_last_error.c_str(); }

extern "C" const char *b200_version(void) { return "amgcl_b200 0.1.0 sm_90a"; }

extern "C" int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

static int ctx_init(b200_ctx_t ctx, int device) {
    cudaDeviceProp prop;
    B200_CUDA(cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    // the library holds sm_90a code only, which no other compute capability can load
    if (prop.major != 9 || prop.minor != 0)
        return fail(B200_ECUDA, "amgcl_b200 needs an sm_90a (Hopper H100) device");
    B200_CUDA(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    B200_CUDA(cudaMalloc(&ctx->dot_partial, kDotMaxBlocks * sizeof(double)));
    B200_CUDA(cudaMalloc(&ctx->dot_ticket, sizeof(unsigned int)));
    B200_CUDA(cudaMemset(ctx->dot_ticket, 0, sizeof(unsigned int)));
    B200_CUDA(cudaHostAlloc(&ctx->dot_result_h, 8 * sizeof(double), cudaHostAllocMapped));
    B200_CUDA(cudaHostGetDevicePointer(&ctx->dot_result_d, ctx->dot_result_h, 0));
    B200_CUDA(cudaMalloc(&ctx->dot_dev, 2 * sizeof(double)));
    return scal_create(ctx);
}

extern "C" int b200_ctx_create(int device, b200_ctx_t *out) {
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    int ndev = 0;
    B200_CUDA(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(B200_EINVAL, "no such CUDA device");
    DeviceGuard guard(device);
    if (!guard.ok) return fail(B200_ECUDA, "cudaSetDevice failed");

    b200_ctx_s *ctx = new (std::nothrow) b200_ctx_s();
    if (!ctx) return fail(B200_ENOMEM, "out of host memory");
    ctx->device = device;
    if (const char *e = getenv("B200_PDL")) ctx->opt_pdl = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_CYCLE_GRAPH")) ctx->opt_cycle_graph = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_GRAPH_PDL")) ctx->opt_graph_pdl = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_FUSED_KRYLOV")) ctx->opt_fused_krylov = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_COARSE_TAIL")) ctx->opt_coarse_tail = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_FUSE_FIRST_SWEEP")) ctx->opt_fuse_first_sweep = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_POLL_SCALARS")) ctx->opt_poll_scalars = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_PATTERNS")) ctx->opt_patterns = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_PATTERNS_MIN_NNZ")) ctx->opt_patterns_min_nnz = atoll(e);
    if (const char *e = getenv("B200_OFFSETS")) ctx->opt_offsets = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_OFFSETS_MIN_NNZ")) ctx->opt_offsets_min_nnz = atoll(e);
    if (const char *e = getenv("B200_NARROW_COLUMNS")) ctx->opt_narrow = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_WINDOW")) ctx->opt_window = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_WINDOW_MIN_NNZ")) ctx->opt_window_min_nnz = atoll(e);
    if (const char *e = getenv("B200_WINDOW_GAP")) ctx->opt_window_gap = std::max(1, std::min(8, atoi(e)));
    if (const char *e = getenv("B200_WINDOW_RATIO")) ctx->opt_window_ratio = atoll(e);
    if (const char *e = getenv("B200_WINDOW_LANES")) ctx->opt_window_lanes = atoll(e) & 15;
    if (const char *e = getenv("B200_SMALL_KERNEL_MAX_NNZ")) ctx->opt_small_kernel_max_nnz = atoll(e);
    // any failure below releases what was created so far (b200_ctx_destroy null-checks every member)
    const int rc = ctx_init(ctx, device);
    if (rc != B200_OK) {
        const std::string msg = g_last_error;
        b200_ctx_destroy(ctx);
        g_last_error = msg;
        return rc;
    }
    *out = ctx;
    return B200_OK;
}

extern "C" int b200_ctx_destroy(b200_ctx_t ctx) {
    if (!ctx) return B200_OK;
    tail_destroy(ctx);                            // pending calls are dropped with the context
    ctx->lazy_vec = nullptr;
    GUARD(ctx);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    scal_destroy(ctx);
    tail_destroy(ctx);
    for (int k = 0; k < 2; ++k) {
        if (ctx->stage_host[k]) cudaFreeHost(ctx->stage_host[k]);
        if (ctx->stage_event[k]) cudaEventDestroy(ctx->stage_event[k]);
    }
    if (ctx->gather_ticket) cudaFree(ctx->gather_ticket);
    if (ctx->scal_x_local) {
        for (int q = 0; q < ctx->nranks; ++q)
            if (q != ctx->rank && ctx->scal_x_peer[q]) cudaIpcCloseMemHandle(ctx->scal_x_peer[q]);
        cudaFree(ctx->scal_x_local);
    }
    if (ctx->dot_partial) cudaFree(ctx->dot_partial);
    if (ctx->dot_ticket) cudaFree(ctx->dot_ticket);
    if (ctx->dot_result_h) cudaFreeHost(ctx->dot_result_h);
    if (ctx->dot_dev) cudaFree(ctx->dot_dev);
    if (ctx->push_ticket) cudaFree(ctx->push_ticket);
    if (ctx->ipc_dev) cudaFree(ctx->ipc_dev);
    if (ctx->probe_pb_local) {
        for (int q = 0; q < ctx->nranks; ++q)
            if (q != ctx->rank && ctx->probe_pb_peer[q]) cudaIpcCloseMemHandle(ctx->probe_pb_peer[q]);
        cudaFree(ctx->probe_pb_local);
    }
    for (void *ptr : ctx->deferred_free) cudaFree(ptr);
    if (ctx->comm && nccl().handle) nccl().CommDestroy(comm_of(ctx));
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    for (cudaEvent_t e : ctx->prof_events) cudaEventDestroy(e);
    delete ctx;
    return B200_OK;
}

extern "C" int b200_ctx_default(b200_ctx_t *out) {
    B200_REQUIRE(out != nullptr, "null output pointer");
    static std::mutex mtx;
    static b200_ctx_t def = nullptr;
    std::lock_guard<std::mutex> lock(mtx);
    if (!def) {
        int dev = 0;
        B200_CUDA(cudaGetDevice(&dev));
        int rc = b200_ctx_create(dev, &def);
        if (rc != B200_OK) return rc;
    }
    *out = def;
    return B200_OK;
}

extern "C" int b200_ctx_set_stream(b200_ctx_t ctx, void *cuda_stream) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "stream change");
    {
        GUARD(ctx);                               // deferred calls belong on the old stream
    }
    ctx->option_epoch++;
    ctx->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
    return B200_OK;
}

extern "C" int b200_ctx_get_stream(b200_ctx_t ctx, void **cuda_stream) {
    CHECK_CTX(ctx);
    B200_REQUIRE(cuda_stream != nullptr, "null output pointer");
    *cuda_stream = ctx->stream;
    return B200_OK;
}

extern "C" int b200_ctx_device(b200_ctx_t ctx, int *device) {
    CHECK_CTX(ctx);
    B200_REQUIRE(device != nullptr, "null output pointer");
    *device = ctx->device;
    return B200_OK;
}

extern "C" int b200_ctx_sync(b200_ctx_t ctx) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "sync");
    GUARD(ctx);
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    return B200_OK;
}

extern "C" int b200_ctx_flush(b200_ctx_t ctx) {
    CHECK_CTX(ctx);
    GUARD(ctx);
    return B200_OK;
}

extern "C" int b200_ctx_launch_count(b200_ctx_t ctx, uint64_t *count) {
    CHECK_CTX(ctx);
    B200_REQUIRE(count != nullptr, "null output pointer");
    *count = ctx->launches;
    return B200_OK;
}

extern "C" int b200_ctx_reset_launch_count(b200_ctx_t ctx) {
    CHECK_CTX(ctx);
    ctx->launches = 0;
    return B200_OK;
}

extern "C" int b200_profile_begin(b200_ctx_t ctx) {
    CHECK_CTX(ctx);
    NOT_RECORDING(ctx, "profiling");
    {
        GUARD(ctx);
    }
    ctx->prof_used = 0;
    ctx->prof_recs.clear();
    ctx->profiling = true;
    return B200_OK;
}

// per (shape, mode, format) device times of the launches since b200_profile_begin
static int profile_collect(b200_ctx_t ctx, std::vector<b200_profile_format_entry> &agg) {
    GUARD(ctx);
    ctx->profiling = false;
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    for (const auto &r : ctx->prof_recs) {
        float ms = 0.f;
        B200_CUDA(cudaEventElapsedTime(&ms, ctx->prof_events[r.ev], ctx->prof_events[r.ev + 1]));
        b200_profile_format_entry *hit = nullptr;
        for (auto &a : agg)
            if (a.entry.nrows == r.nrows && a.entry.ncols == r.ncols && a.entry.nnz == r.nnz &&
                a.entry.mode == r.mode && a.format == r.fmt) {
                hit = &a;
                break;
            }
        if (!hit) {
            agg.push_back({{r.nrows, r.ncols, r.nnz, r.mode, 0, 0.0, 1e30}, r.fmt});
            hit = &agg.back();
        }
        hit->entry.launches += 1;
        hit->entry.total_ms += ms;
        if (ms < hit->entry.min_ms) hit->entry.min_ms = ms;
    }
    ctx->prof_recs.clear();
    ctx->prof_used = 0;
    return B200_OK;
}

extern "C" int b200_profile_end(b200_ctx_t ctx, b200_profile_entry *out, int64_t capacity,
                                int64_t *count) {
    CHECK_CTX(ctx);
    B200_REQUIRE(count != nullptr, "null output pointer");
    std::vector<b200_profile_format_entry> agg;
    const int rc = profile_collect(ctx, agg);
    if (rc) return rc;
    *count = (int64_t)agg.size();
    if (out) {
        const int64_t m = std::min<int64_t>(capacity, (int64_t)agg.size());
        for (int64_t i = 0; i < m; ++i) out[i] = agg[(size_t)i].entry;
    }
    return B200_OK;
}

extern "C" int b200_profile_end_formats(b200_ctx_t ctx, b200_profile_format_entry *out, int64_t capacity,
                                        int64_t *count) {
    CHECK_CTX(ctx);
    B200_REQUIRE(count != nullptr, "null output pointer");
    std::vector<b200_profile_format_entry> agg;
    const int rc = profile_collect(ctx, agg);
    if (rc) return rc;
    *count = (int64_t)agg.size();
    if (out) {
        const int64_t m = std::min<int64_t>(capacity, (int64_t)agg.size());
        for (int64_t i = 0; i < m; ++i) out[i] = agg[(size_t)i];
    }
    return B200_OK;
}


static int64_t *option_slot(b200_ctx_t ctx, const char *key) {
    if (!key) return nullptr;
    if (!strcmp(key, "spmv_variant")) return &ctx->opt_spmv_variant;
    if (!strcmp(key, "fuse_relax")) return &ctx->opt_fuse_relax;
    if (!strcmp(key, "zero_shortcut")) return &ctx->opt_zero_shortcut;
    if (!strcmp(key, "nnz_cap")) return &ctx->opt_nnz_cap;
    if (!strcmp(key, "lanes")) return &ctx->opt_lanes;
    if (!strcmp(key, "ctas_per_sm")) return &ctx->opt_ctas_per_sm;
    if (!strcmp(key, "stages")) return &ctx->opt_stages;
    if (!strcmp(key, "p2p")) return &ctx->opt_p2p;
    if (!strcmp(key, "pdl")) return &ctx->opt_pdl;
    if (!strcmp(key, "cycle_graph")) return &ctx->opt_cycle_graph;
    if (!strcmp(key, "graph_pdl")) return &ctx->opt_graph_pdl;
    if (!strcmp(key, "fused_krylov")) return &ctx->opt_fused_krylov;
    if (!strcmp(key, "coarse_tail")) return &ctx->opt_coarse_tail;
    if (!strcmp(key, "poll_scalars")) return &ctx->opt_poll_scalars;
    if (!strcmp(key, "small_kernel_max_nnz")) return &ctx->opt_small_kernel_max_nnz;
    if (!strcmp(key, "patterns")) return &ctx->opt_patterns;
    if (!strcmp(key, "patterns_min_nnz")) return &ctx->opt_patterns_min_nnz;
    if (!strcmp(key, "offsets")) return &ctx->opt_offsets;
    if (!strcmp(key, "offsets_min_nnz")) return &ctx->opt_offsets_min_nnz;
    if (!strcmp(key, "narrow_columns")) return &ctx->opt_narrow;
    if (!strcmp(key, "window")) return &ctx->opt_window;
    if (!strcmp(key, "window_min_nnz")) return &ctx->opt_window_min_nnz;
    if (!strcmp(key, "window_ratio")) return &ctx->opt_window_ratio;
    if (!strcmp(key, "window_gap")) return &ctx->opt_window_gap;
    if (!strcmp(key, "window_lanes")) return &ctx->opt_window_lanes;
    if (!strcmp(key, "fuse_first_sweep")) return &ctx->opt_fuse_first_sweep;
    if (!strcmp(key, "tail_max_nnz")) return &ctx->opt_tail_max_nnz;
    if (!strcmp(key, "tail_max_vec")) return &ctx->opt_tail_max_vec;
    return nullptr;
}

extern "C" int b200_ctx_set_option(b200_ctx_t ctx, const char *key, int64_t value) {
    CHECK_CTX(ctx);
    int64_t *slot = option_slot(ctx, key);
    if (!slot) return fail(B200_EINVAL, std::string("unknown option: ") + (key ? key : "(null)"));
    if (slot == &ctx->opt_nnz_cap) {
        if (value < 256 || value > kNnzCapMax || (value % 8))
            return fail(B200_EINVAL, "nnz_cap must be a multiple of 8 in [256, 6144]");
    } else if (slot == &ctx->opt_lanes) {
        if (value != 0 && (value < 1 || value > 32 || (value & (value - 1))))
            return fail(B200_EINVAL, "lanes must be 0 (auto) or a power of two <= 32");
    } else if (slot == &ctx->opt_stages) {
        if (value < 1 || value > 8) return fail(B200_EINVAL, "stages must be in [1, 8]");
    } else if (slot == &ctx->opt_ctas_per_sm) {
        if (value < 1 || value > 8) return fail(B200_EINVAL, "ctas_per_sm must be in [1, 8]");
    } else if (slot == &ctx->opt_spmv_variant) {
        if (value < 0 || value > 1) return fail(B200_EINVAL, "spmv_variant must be 0 or 1");
    }
    B200_REQUIRE(!ctx->recording, "options cannot change while a graph is being recorded");
    {
        GUARD(ctx);                               // deferred calls ran under the old value
    }
    if (*slot != value) ctx->option_epoch++;      // recorded graphs were built with the old value
    *slot = value;
    return B200_OK;
}

extern "C" int b200_ctx_get_option(b200_ctx_t ctx, const char *key, int64_t *value) {
    CHECK_CTX(ctx);
    B200_REQUIRE(value != nullptr, "null output pointer");
    int64_t *slot = option_slot(ctx, key);
    if (!slot) return fail(B200_EINVAL, std::string("unknown option: ") + (key ? key : "(null)"));
    *value = *slot;
    return B200_OK;
}

// ---------------------------------------------------------------------------
// CUDA-graph recording of a call sequence (the V-cycle; SURVEY section 8(f) rank 1)
// ---------------------------------------------------------------------------
namespace b200 {
static void graph_free(b200_graph_s *g) {
    if (!g) return;
    if (g->exec) cudaGraphExecDestroy(g->exec);
    if (g->graph) cudaGraphDestroy(g->graph);
    delete g;
}
static void graph_release_deferred(b200_ctx_t ctx) {
    for (void *p : ctx->graph_deferred) cudaFree(p);     // cudaFree waits for the device
    ctx->graph_deferred.clear();
}
// put every touched object back into the state it had when recording started (nothing that
// was recorded has run).  The generations move on rather than back: products the recorded
// calls registered name table slots no executed kernel wrote, and must not match.
static void graph_rollback(b200_graph_s *g) {
    for (const GraphSlot &s : g->slots) {
        *s.slot = s.p0;
        if (s.zp) *s.zp = s.z0;
        if (s.gen) ++*s.gen;
    }
}
} // namespace b200

extern "C" int b200_graph_begin(b200_ctx_t ctx, int *recording) {
    CHECK_CTX(ctx);
    B200_REQUIRE(recording != nullptr, "null output pointer");
    B200_REQUIRE(!ctx->recording, "graph_begin: already recording");
    *recording = 0;
    // not recordable: per-launch event timing, multi-GPU exchanges (host-side sequence
    // numbers and NCCL calls), the legacy default stream
    if (ctx->profiling || ctx->dist || !ctx->opt_cycle_graph) return B200_OK;
    if (ctx->stream == nullptr || ctx->stream == cudaStreamLegacy) return B200_OK;
    GUARD(ctx);
    b200_graph_s *g = new (std::nothrow) b200_graph_s();
    if (!g) return fail(B200_ENOMEM, "out of host memory");
    g->ctx = ctx;
    g->destroy_epoch = ctx->destroy_epoch;
    g->option_epoch = ctx->option_epoch;
    g->launches0 = ctx->launches;
    const cudaError_t rc = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed);
    if (rc != cudaSuccess) {
        delete g;
        return cuda_fail(rc, "cudaStreamBeginCapture", __FILE__, __LINE__);
    }
    ctx->recording = g;
    *recording = 1;
    return B200_OK;
}

extern "C" int b200_graph_abort(b200_ctx_t ctx) {
    CHECK_CTX(ctx);
    b200_graph_s *g = ctx->recording;
    if (!g) return B200_OK;
    GUARD(ctx);
    cudaGraph_t junk = nullptr;
    cudaStreamEndCapture(ctx->stream, &junk);      // may itself report the capture as invalidated
    if (junk) cudaGraphDestroy(junk);
    cudaGetLastError();
    graph_rollback(g);
    ctx->launches = g->launches0;
    ctx->recording = nullptr;
    graph_free(g);
    graph_release_deferred(ctx);
    return B200_OK;
}

extern "C" int b200_graph_end(b200_ctx_t ctx, b200_graph_t *out) {
    CHECK_CTX(ctx);
    B200_REQUIRE(out != nullptr, "null output pointer");
    *out = nullptr;
    b200_graph_s *g = ctx->recording;
    B200_REQUIRE(g != nullptr, "graph_end: not recording");
    GUARD(ctx);
    ctx->recording = nullptr;
    cudaError_t rc = cudaStreamEndCapture(ctx->stream, &g->graph);
    if (rc == cudaSuccess) rc = cudaGraphInstantiate(&g->exec, g->graph, 0);
    if (rc == cudaSuccess) rc = cudaGraphGetNodes(g->graph, nullptr, &g->nodes);
    if (rc == cudaSuccess) rc = cudaGraphLaunch(g->exec, ctx->stream);     // the recorded calls run now
    if (rc != cudaSuccess) {
        cudaGetLastError();
        graph_rollback(g);
        ctx->launches = g->launches0;
        graph_free(g);
        graph_release_deferred(ctx);
        return cuda_fail(rc, "graph_end (capture / instantiate / launch)", __FILE__, __LINE__);
    }
    graph_release_deferred(ctx);
    for (GraphSlot &s : g->slots) {
        s.p1 = *s.slot;
        s.z1 = s.zp ? *s.zp : false;
    }
    g->launches = ctx->launches - g->launches0;
    *out = g;
    return B200_OK;
}

extern "C" int b200_graph_launch(b200_ctx_t ctx, b200_graph_t g, int *launched) {
    CHECK_CTX(ctx);
    B200_REQUIRE(g && launched, "null argument");
    *launched = 0;
    B200_REQUIRE(g->ctx == ctx, "graph belongs to another context");
    B200_REQUIRE(!ctx->recording, "graph_launch: a graph is being recorded");
    if (ctx->profiling || !ctx->opt_cycle_graph) return B200_OK;
    if (g->destroy_epoch != ctx->destroy_epoch || g->option_epoch != ctx->option_epoch)
        return B200_OK;                      // stale: the caller records a new one
    for (const GraphSlot &s : g->slots)
        if (*s.slot != s.p0 || (s.zp && *s.zp != s.z0)) return B200_OK;
    GUARD(ctx);
    B200_CUDA(cudaGraphLaunch(g->exec, ctx->stream));
    for (const GraphSlot &s : g->slots) {
        *s.slot = s.p1;
        if (s.zp) *s.zp = s.z1;
        if (s.gen) ++*s.gen;                 // the replay wrote (or may have written) the vector
    }
    // products the recorded kernels leave in the scalar table (smoother sweep -> <rhs, x>)
    for (const GraphProduct &p : g->products) product_record(ctx, p.a, p.b, p.slot);
    ctx->launches += g->launches;
    g->replays++;
    *launched = 1;
    return B200_OK;
}

extern "C" int b200_graph_info(b200_graph_t g, int64_t *kernels, int64_t *nodes, int64_t *replays,
                               int *stale) {
    B200_REQUIRE(g != nullptr, "null argument");
    if (kernels) *kernels = (int64_t)g->launches;
    if (nodes) *nodes = (int64_t)g->nodes;
    if (replays) *replays = (int64_t)g->replays;
    if (stale)
        *stale = (g->destroy_epoch != g->ctx->destroy_epoch || g->option_epoch != g->ctx->option_epoch);
    return B200_OK;
}

extern "C" int b200_graph_destroy(b200_graph_t g) {
    if (!g) return B200_OK;
    GUARD(g->ctx);
    graph_free(g);
    return B200_OK;
}

