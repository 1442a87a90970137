/*
 * amgcl_b200.h -- C ABI of the H100-native solve-phase backend for AMGCL.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Everything the AMGCL
 * solve phase asks of a backend -- amgcl::backend::{spmv, residual, vmul,
 * axpby, axpbypcz, inner_product, copy, clear} (reference:
 * amgcl/backend/interface.hpp:312-405), the damped_jacobi / spai0 smoother
 * sweeps (amgcl/relaxation/damped_jacobi.hpp:103-132, spai0.hpp:86-109) and
 * the coarsest-level direct solve (amgcl/amg.hpp:521-524,
 * amgcl/backend/cuda.hpp:61-84) -- is exported here as plain `extern "C"`
 * functions over opaque handles, plain pointers and sizes.  No C++ or torch
 * types cross this boundary.  The C++ header include/amgcl/backend/b200.hpp
 * binds these symbols to the amgcl::backend template interface.
 *
 * Conventions
 *   - every function returns 0 on success, a negative B200_E* code otherwise;
 *     b200_last_error() returns a thread-local, human readable message.
 *   - all device work is issued on the context's stream (b200_ctx_set_stream)
 *     and is asynchronous unless stated otherwise.
 *   - values are FP64, device indices are int32 (nnz < 2^31 per matrix);
 *     host CSR input may be int64 (ptrdiff_t, amgcl's default) or int32.
 *   - there is NO CPU fallback: if no CUDA device is usable every call fails.
 */
#ifndef AMGCL_B200_H
#define AMGCL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK            0
#define B200_EINVAL       -1   /* bad argument (null handle, size mismatch ...)   */
#define B200_ECUDA        -2   /* CUDA runtime error; see b200_last_error()      */
#define B200_ENOMEM       -3   /* host or device allocation failed               */
#define B200_ERANGE       -4   /* nnz or dimension does not fit int32            */
#define B200_ESINGULAR    -5   /* coarse matrix is numerically singular          */
#define B200_ENCCL        -6   /* NCCL error                                     */

/* element types: FP64 is the default everywhere; FP32 objects exist for AMGCL's mixed
 * precision composition (FP32 hierarchy under an FP64 Krylov solver,
 * tutorial/1.poisson3Db/poisson3Db.cpp:45-51, docs/tutorial/poisson3Db.rst:259-292) */
#define B200_F64           0
#define B200_F32           1

typedef struct b200_ctx_s    *b200_ctx_t;     /* device + stream + scratch            */
typedef struct b200_csr_s    *b200_csr_t;     /* device CSR matrix (+ row-block plan) */
typedef struct b200_vec_s    *b200_vec_t;     /* device FP64 vector                   */
typedef struct b200_coarse_s *b200_coarse_t;  /* coarsest-level direct solver         */
typedef struct b200_split_s  *b200_split_t;   /* host view of one rank's operator share */
typedef struct b200_graph_s  *b200_graph_t;   /* recorded call sequence (CUDA graph)    */
typedef struct b200_index_s  *b200_index_t;   /* device index list (gather / scatter)   */
typedef struct b200_krylov_s *b200_krylov_t;  /* device-resident scalars of a Krylov solver */

/* ---------------------------------------------------------------- context */

/* Thread-local message describing the last failing call. */
const char *b200_last_error(void);

/* Library version string ("amgcl_b200 <semver> sm_90a"). */
const char *b200_version(void);

/* Number of usable CUDA devices (0 if none: every other call will fail). */
int b200_device_count(void);

/* Create a context on CUDA device `device` (replaces the cusparseHandle_t that
 * amgcl::backend::cuda<>::params carries, amgcl/backend/cuda.hpp:490-507). */
int b200_ctx_create(int device, b200_ctx_t *ctx);
int b200_ctx_destroy(b200_ctx_t ctx);

/* Process-wide default context on the current device (lazily created).  Used
 * by the C++ shim when Backend::params is default constructed. */
int b200_ctx_default(b200_ctx_t *ctx);

/* Use an externally owned cudaStream_t (e.g. torch's current stream) for all
 * subsequent work; NULL selects the context's own stream again. */
int b200_ctx_set_stream(b200_ctx_t ctx, void *cuda_stream);
int b200_ctx_get_stream(b200_ctx_t ctx, void **cuda_stream);
int b200_ctx_device(b200_ctx_t ctx, int *device);

/* Block the host until all work issued on the context's stream is done. */
int b200_ctx_sync(b200_ctx_t ctx);
/* Calls on small operators may be deferred (option "coarse_tail"); they reach the stream when
 * the next call that cannot be deferred is made -- every host-synchronous call, b200_ctx_sync,
 * and this one.  Call it before handing the stream to code that does not go through this
 * library (recording an event of your own, say). */
int b200_ctx_flush(b200_ctx_t ctx);

/* Number of kernels launched through this context since creation / reset. */
int b200_ctx_launch_count(b200_ctx_t ctx, uint64_t *count);
int b200_ctx_reset_launch_count(b200_ctx_t ctx);

/* Coarse tail statistics: launches of the tail kernel and calls they executed. */
int b200_tail_stats(b200_ctx_t ctx, uint64_t *flushes, uint64_t *commands);

/* Per-launch device timing of the CSR streaming kernels (the reference's
 * cuda_clock / AMGCL_TIC hooks, cuda.hpp:809-838, only see launch time): between
 * begin and end every spmv / residual / relax launch is bracketed by a pair of
 * CUDA events on the launching stream; end() aggregates them per (matrix shape,
 * mode).  mode: 0 spmv(beta=0), 1 spmv(beta!=0), 2 residual, 3 fused relax; the
 * vector kernels report nrows = n, ncols = 1, nnz = 0 and one of the modes below. */
/* (mode 4: residual fused with the smoother's first sweep from x = 0) */
#define B200_PROF_VECTOR      10   /* element-wise, +1 per extra input stream (10..12) */
#define B200_PROF_DOT         20
#define B200_PROF_RELAX_ZERO  21   /* x = omega*diag.*rhs shortcut of the smoother     */
#define B200_PROF_COARSE      22   /* dense GEMV of the coarsest-level solve           */
#define B200_PROF_MEMSET      23   /* materialised lazy clear                          */
#define B200_PROF_TAIL        24   /* coarse tail: nrows = calls run by the one kernel  */
#define B200_PROF_COMM        30   /* multi-GPU exchange (pack + NCCL collective)      */
typedef struct {
    int64_t nrows, ncols, nnz;
    int     mode;
    int64_t launches;
    double  total_ms;
    double  min_ms;
} b200_profile_entry;
int b200_profile_begin(b200_ctx_t ctx);
int b200_profile_end(b200_ctx_t ctx, b200_profile_entry *out, int64_t capacity, int64_t *count);

/* ---------------------------------------------------------------- multi-GPU */

/* One process per GPU (SPMD): every rank runs the same AMGCL program on the same
 * host hierarchy; after b200_dist_init every vector / matrix dimension >=
 * dist_min_rows is partitioned in uniform contiguous row blocks across the ranks and
 * everything smaller is replicated (every rank holds and computes it, as mpi::amg
 * consolidates small levels, amgcl/mpi/amg.hpp:430-465).  A rank keeps WHOLE ROWS of every
 * operator, so each row sum is formed on one GPU in the reference's order.
 * Replaces amgcl::mpi::distributed_matrix / comm_pattern / mpi::inner_product
 * (amgcl/mpi/distributed_matrix.hpp:51-557, amgcl/mpi/inner_product.hpp:53-62):
 *   operator with partitioned input   local columns + halo slots; the halo (every rank's
 *                                     packed boundary values) is pushed into the peers'
 *                                     buffers and awaited INSIDE the consumer kernel
 *   replicated result, partitioned input   each rank computes a share of the rows and stores
 *                                     them into every rank's gather buffer
 *   <x, y>                            reduced and all-reduced inside the producing kernel
 * over CUDA-IPC mapped peer memory (NVLink); with option "p2p" = 0 the same exchanges run
 * as a pack kernel + ncclAllGather / ncclAllReduce.  With dist_min_rows = rows of the
 * finest matrix only the finest level is partitioned (the north-star configuration).  The
 * id comes from b200_nccl_unique_id on rank 0 and is distributed by the caller (e.g. with
 * torch.distributed). */
int b200_nccl_unique_id(char *id, size_t size /* >= 128 */);
int b200_dist_init(b200_ctx_t ctx, const char *id, size_t size, int nranks, int rank,
                   int64_t dist_min_rows);
/* p2p: 1 if the exchanges run through CUDA-IPC mapped peer memory inside our own kernels
 * (default when every rank could map its peers; option "p2p" = 0 before b200_dist_init
 * forces the NCCL collectives), 0 for NCCL. */
int b200_dist_info(b200_ctx_t ctx, int *rank, int *nranks, int64_t *dist_min_rows, int *p2p);

/* Pure host helpers (no device, no NCCL) exposing the partition logic to tests.
 * b200_partition: uniform block size and this rank's [lo, hi) for a dimension.
 * b200_dist_split_i64: rank's share of an operator = the rows of its block; kind 1: the
 * vector the operator is applied to is partitioned (columns remapped to [local | halo
 * slots]), kind 2: it is replicated (columns untouched).  slots = halo slots per rank,
 * send_idx = local indices this rank contributes to the all-gathered halo, in slot order. */
int b200_partition(int64_t n, int nranks, int rank, int64_t *block, int64_t *lo, int64_t *hi);
int b200_dist_split_i64(int kind, int nranks, int rank, int64_t nrows, int64_t ncols,
                        const int64_t *ptr, const int64_t *col, const double *val,
                        b200_split_t *out);
int b200_split_info(b200_split_t sp, int64_t *nrows, int64_t *ncols, int64_t *nnz,
                    int64_t *n_loc, int64_t *slots, int64_t *n_send);
int b200_split_copy(b200_split_t sp, int64_t *ptr, int64_t *col, double *val, int64_t *send_idx);
int b200_split_destroy(b200_split_t sp);

/* Tuning knobs (all optional; defaults are chosen for the H100).
 *   "spmv_variant"     0 = one row block per CTA, 1 = persistent multi-stage ring (default)
 *   "ctas_per_sm"      persistent variant: resident CTAs per SM (default 4)
 *   "stages"           persistent variant: ring depth per CTA (default 2)
 *   "nnz_cap"          non-zeros staged per row block (default 2048; applies to
 *                      matrices created afterwards)
 *   "lanes"            lanes per row, 0 = from the average row length (default)
 *   "p2p"              multi-GPU: 1 = peer-memory exchange kernels (default), 0 = NCCL
 *   "pdl"              1 = programmatic dependent launch of the solve kernels (default;
 *                      environment variable B200_PDL overrides the default), 0 = plain launches
 *   "cycle_graph"      1 = b200_graph_begin records (default; env B200_CYCLE_GRAPH), 0 = it
 *                      reports "not recording" and existing graphs are not replayed
 *   "graph_pdl"        1 = launches recorded into a graph keep the PDL attribute (default;
 *                      env B200_GRAPH_PDL)
 *   "coarse_tail"      1 = calls on small operators (at most "tail_max_nnz" non-zeros, default
 *                      1.5e6; x = 0 sweeps on at most "tail_max_vec" entries) are deferred and run
 *                      together as ONE cooperative kernel with device-wide barriers between them
 *                      when the next call that cannot be deferred arrives (default); 0 = every
 *                      call launches its own kernel.  Results are bit-identical either way.
 *   "fuse_first_sweep" 1 = b200_relax on an x known to be zero followed by b200_residual of the
 *                      same system (amg.hpp:527-534: pre-smoothing, then the residual to restrict)
 *                      is ONE pass over A: x = (omega*diag).*rhs is formed on the fly, written,
 *                      and r = rhs - A x with it (default; operators with short rows and tiny
 *                      levels only); 0 = two kernels.  Results are bit-identical.
 *   "small_kernel_max_nnz"  FP64 operators with at most this many non-zeros are applied by a
 *                      direct-load kernel instead of the TMA ring pipeline; same arithmetic,
 *                      bit-identical results.  Default 0 = always the ring kernel: measured, the
 *                      ring kernel wins even on tiny operators because its first bulk copies
 *                      are issued before the grid dependency resolves
 *   "poll_scalars"     1 = a host-synchronous result of an in-kernel reduction (b200_dot, the
 *                      Krylov steps) is awaited by polling the mapped host word the finishing CTA
 *                      releases (default), 0 = by cudaStreamSynchronize
 *   "fused_krylov"     1 = the C++ binding's solver::cg / solver::bicgstab specialisations run the
 *                      fused b200_cg_* / b200_bicg_* steps (default; env B200_FUSED_KRYLOV),
 *                      0 = they issue the reference's sequence of primitives
 *   "patterns"         1 = operators with at most 256 row patterns (created afterwards, at least
 *                      "patterns_min_nnz" non-zeros, default 1e6) are also stored pattern-indexed
 *                      and streamed without per-entry columns (default; env B200_PATTERNS);
 *                      0 = not built / not used.  Bit-identical either way (see below).
 *   "offsets"          the same for offset-indexed columns ("offsets_min_nnz"; env B200_OFFSETS);
 *                      used where an operator does not qualify for "patterns"
 *   "window"           1 = operators that qualify are also stored windowed ("window_min_nnz",
 *                      "window_ratio" percent, "window_gap", "window_lanes"); default 0:
 *                      measured slower than the plain path (env B200_WINDOW)
 *   "fuse_relax"       1 = single-pass fused smoother sweep (default), 0 = two kernels
 *   "zero_shortcut"    1 = skip the A-pass when x is known to be zero (default)
 * Unknown keys return B200_EINVAL. */
int b200_ctx_set_option(b200_ctx_t ctx, const char *key, int64_t value);
int b200_ctx_get_option(b200_ctx_t ctx, const char *key, int64_t *value);

/* ---------------------------------------------------------------- vectors */

/* Replaces thrust::device_vector<double> (amgcl/backend/cuda.hpp:483-484) and
 * Backend::create_vector / copy_vector (cuda.hpp:521-546). */
int b200_vec_create(b200_ctx_t ctx, size_t n, b200_vec_t *v);        /* zero filled */
int b200_vec_wrap(b200_ctx_t ctx, double *device_ptr, size_t n, b200_vec_t *v);
int b200_vec_destroy(b200_vec_t v);
int b200_vec_size(b200_vec_t v, size_t *n);
int b200_vec_bytes(b200_vec_t v, size_t *bytes);
/* Raw device pointer (materialises a pending lazy clear).  The pointer is
 * invalidated by b200_relax(), which may swap storage between x and tmp. */
int b200_vec_data(b200_vec_t v, double **device_ptr);
/* Host <-> device copies, ordered on the context's stream; both block the host
 * until the copy has completed (same semantics as thrust::copy, cuda.hpp:635-660). */
int b200_vec_upload(b200_vec_t v, const double *host, size_t n);
int b200_vec_download(b200_vec_t v, double *host, size_t n);
/* Multi-GPU contexts: the block of a partitioned vector this rank owns ([offset, offset+len) of
 * the global index range; the whole vector otherwise), and a download of only that block into
 * its place host[offset .. offset+len) of a full-size host array -- no exchange between the
 * ranks, other entries of `host` are left untouched (b200_vec_download all-gathers the complete
 * vector to every rank).  On a single GPU identical to b200_vec_download. */
int b200_vec_local_range(b200_vec_t v, size_t *offset, size_t *len);
int b200_vec_download_local(b200_vec_t v, double *host, size_t n);
/* FP32 vectors (single GPU only).  Every primitive below accepts the precision
 * combinations AMGCL's mixed-precision composition produces -- all FP64, all FP32, and an
 * FP32 matrix / diagonal applied to FP64 vectors (see DESIGN.md "Mixed precision") -- and
 * returns B200_EINVAL for any other mix. */
int b200_vec_create_f32(b200_ctx_t ctx, size_t n, b200_vec_t *v);
int b200_vec_upload_f32(b200_vec_t v, const float *host, size_t n);
int b200_vec_download_f32(b200_vec_t v, float *host, size_t n);
int b200_vec_dtype(b200_vec_t v, int *dtype);

/* ---------------------------------------------------------------- matrices */

/* Upload a host CSR matrix (deep copy), narrowing indices to int32 and building
 * the row-block plan used by the streaming kernels.  Replaces
 * cuda_matrix<double>'s constructor (amgcl/backend/cuda.hpp:219-237,310-333)
 * as called from Backend::copy_matrix (cuda.hpp:512-518). */
int b200_csr_create_i64(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                        const int64_t *ptr, const int64_t *col, const double *val,
                        b200_csr_t *A);
int b200_csr_create_i32(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                        const int32_t *ptr, const int32_t *col, const double *val,
                        b200_csr_t *A);
int b200_csr_create_i64_f32(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                            const int64_t *ptr, const int64_t *col, const float *val,
                            b200_csr_t *A);
int b200_csr_create_i32_f32(b200_ctx_t ctx, int64_t nrows, int64_t ncols,
                            const int32_t *ptr, const int32_t *col, const float *val,
                            b200_csr_t *A);
int b200_csr_dtype(b200_csr_t A, int *dtype);
int b200_csr_destroy(b200_csr_t A);
int b200_csr_rows(b200_csr_t A, size_t *n);
int b200_csr_cols(b200_csr_t A, size_t *n);
int b200_csr_nonzeros(b200_csr_t A, size_t *n);
int b200_csr_bytes(b200_csr_t A, size_t *bytes);
/* Plan introspection for tests / DESIGN.md: lanes per row and row-block count. */
int b200_csr_plan(b200_csr_t A, int *lanes_per_row, int64_t *n_blocks, int64_t *n_long_blocks);

/* Pure host helper (no device needed): the row-block plan b200_csr_create_*
 * would build for a matrix with these row pointers.  blk_out (may be NULL)
 * receives nblocks+1 pairs {first row, first non-zero}; blk_capacity is its
 * size in pairs.  lanes = 0 selects lanes-per-row from the average row length. */
int b200_plan_i64(int64_t nrows, const int64_t *ptr, int lanes, int nnz_cap,
                  int32_t *blk_out, int64_t blk_capacity, int64_t *nblocks,
                  int *lanes_out, int *rows_cap_out, int64_t *nlong_out);

/* Pattern-indexed rows.  In a matrix assembled on a structured grid whole rows repeat: the
 * tuple (col - row of every entry, in entry order) of a row is one of a few patterns (27 for
 * the 7-point Poisson problem).  With at most 256 patterns (1024 offsets in all) the upload
 * also stores one byte per ROW, and the streaming kernel reads no column information per
 * entry at all (8 instead of 12 bytes per FP64 entry), rebuilding col = row + pattern[k] from
 * a table in shared memory; same entry order and arithmetic, same bits (options "patterns",
 * "patterns_min_nnz"; decided at upload; preferred over offset-indexed columns).
 * b200_csr_patterns: whether A carries the format, its patterns and their total length.
 * b200_pattern_plan_i64: pure host helper for tests (pid_out [nrows], start_out [257],
 * off_out [1024]). */
int b200_csr_patterns(b200_csr_t A, int *pattern_indexed, int *count, int *total);
/* The largest operator (this rank's non-zeros) uploaded through ctx so far and the column
 * format it is stored in: 0 plain, 1 windowed, 2 offset-indexed, 3 pattern-indexed (what
 * bench.py needs to count the bytes the finest-level passes really stream). */
int b200_ctx_largest_operator(b200_ctx_t ctx, int64_t *nnz, int *format);
int b200_pattern_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                          uint8_t *pid_out, uint16_t *start_out, int32_t *off_out, int *count,
                          int *total, int *qualifies);

/* Offset-indexed columns.  If col - row takes at most 256 distinct values over the whole
 * operator (matrices assembled on structured grids: 7 for the Poisson stencil), the upload
 * also stores one byte per entry -- the index of its offset in a table -- and the streaming
 * kernel reads 1 instead of 4 bytes of column per entry, rebuilding col = row + table[index];
 * same entry order and arithmetic, same bits (options "offsets", "offsets_min_nnz"; decided at
 * upload).  b200_csr_offsets: whether A carries the format and how many offsets it has.
 * b200_offset_plan_i64: pure host helper for tests (idx8_out [nnz], tab_out [256]). */
int b200_csr_offsets(b200_csr_t A, int *offset_indexed, int *count);
int b200_offset_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                         uint8_t *idx8_out, int32_t *tab_out, int *count, int *qualifies);

/* Windowed operators (opt-in: measured slower than the plain path, DESIGN.md).  An
 * operator whose row blocks gather x from few contiguous places
 * (the level matrices and prolongations of a structured problem) is additionally stored with
 * 16-bit window-local columns plus, per row block, the runs of x its window is made of; the
 * streaming kernel then fills the window into shared memory with coalesced loads and reduces
 * the rows out of it -- same arithmetic, same bits, fewer bytes (options "window",
 * "window_min_nnz", "window_ratio", "window_gap", "window_lanes"; decided at upload).
 * b200_csr_window: whether A carries the format, its largest window / run list and the sum of
 * all window sizes (elements of x).
 * b200_window_plan_i64: pure host helper for tests -- plan + windows of a host matrix.
 * blk_out receives 6 ints per block {first row, end row, first nnz, end nnz, first run, end
 * run}, runs_out 2 ints per run {first column, length | first slot << 16}, col16_out one
 * window slot per entry.  *qualifies == 0: the operator would be stored plain. */
int b200_csr_window(b200_csr_t A, int *windowed, int *max_slots, int *max_runs, int64_t *total_slots);
int b200_window_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                         int lanes, int nnz_cap, int slot_cap, int max_ratio_percent, int gap,
                         uint16_t *col16_out, int32_t *runs_out, int64_t runs_capacity,
                         int32_t *blk_out, int64_t blk_capacity, int64_t *nblocks,
                         int64_t *nruns, int *max_slots, int *max_runs, int *qualifies);

/* ---------------------------------------------------------------- primitives */

/* y = alpha*A*x + beta*y.  y is never read when beta == 0.
 * (interface.hpp:312-323, builtin: backend/detail/matrix_ops.hpp:47-83) */
int b200_spmv(b200_ctx_t ctx, double alpha, b200_csr_t A, b200_vec_t x,
              double beta, b200_vec_t y);

/* r = f - A*x, one kernel (interface.hpp:329-335, matrix_ops.hpp:85-115;
 * the reference cuda backend needs copy + spmv, cuda.hpp:605-622). */
int b200_residual(b200_ctx_t ctx, b200_vec_t f, b200_csr_t A, b200_vec_t x,
                  b200_vec_t r);

/* x = 0 (interface.hpp:338-344).  Lazy: marks x as zero; the memset is only
 * issued if something later reads x element-wise. */
int b200_clear(b200_ctx_t ctx, b200_vec_t x);

/* y = x (interface.hpp:347-353). */
int b200_copy(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y);

/* *result = sum_i x_i*y_i, compensated, deterministic summation order,
 * synchronous (interface.hpp:356-371; builtin Kahan: builtin.hpp:1099-1183). */
int b200_dot(b200_ctx_t ctx, b200_vec_t x, b200_vec_t y, double *result);

/* y = a*x + b*y; y not read when b == 0 (interface.hpp:377-382, builtin.hpp:1185-1209). */
int b200_axpby(b200_ctx_t ctx, double a, b200_vec_t x, double b, b200_vec_t y);

/* z = a*x + b*y + c*z; z not read when c == 0 (interface.hpp:388-393, builtin.hpp:1211-1236). */
int b200_axpbypcz(b200_ctx_t ctx, double a, b200_vec_t x, double b, b200_vec_t y,
                  double c, b200_vec_t z);

/* z = alpha*x.*y + beta*z; z not read when beta == 0 (interface.hpp:399-405, builtin.hpp:1238-1265). */
int b200_vmul(b200_ctx_t ctx, double alpha, b200_vec_t x, b200_vec_t y,
              double beta, b200_vec_t z);

/* Index lists (Backend::gather / Backend::scatter, cuda.hpp:548-577; used by components that
 * move sub-vectors, e.g. the boundary exchange of mpi/distributed_matrix.hpp:300).  `range` is
 * the size of the vector the indices point into; indices are narrowed to int32 and checked
 * (B200_ERANGE).  Single-GPU contexts only. */
int b200_index_create_i64(b200_ctx_t ctx, const int64_t *idx, size_t n, size_t range, b200_index_t *I);
int b200_index_destroy(b200_index_t I);
int b200_index_size(b200_index_t I, size_t *n);
/* dst[k] = src[I[k]], k < n (thrust::gather, cuda.hpp:556-558) */
int b200_gather(b200_ctx_t ctx, b200_index_t I, b200_vec_t src, b200_vec_t dst);
/* host[k] = src[I[k]]: n elements of src's type; synchronous (cuda.hpp:560-563) */
int b200_gather_host(b200_ctx_t ctx, b200_index_t I, b200_vec_t src, void *host);
/* dst[I[k]] = src[k]; the other entries of dst are kept; indices must be distinct
 * (thrust::scatter, cuda.hpp:573-575) */
int b200_scatter(b200_ctx_t ctx, b200_index_t I, b200_vec_t src, b200_vec_t dst);

/* ---------------------------------------------------------------- smoothers */

/* One diagonal-smoother sweep, fused into a single pass over A:
 *     x <- x + (omega * diag) .* (rhs - A x)
 * damped_jacobi: diag = D^-1, omega = damping (damped_jacobi.hpp:103-132);
 * spai0:         diag = M,    omega = 1       (spai0.hpp:86-109).
 * tmp is scratch of the same size as x; on return its contents are unspecified
 * and x/tmp may have exchanged device storage.  If x is known to be zero
 * (b200_clear() was the last writer) the A-pass is skipped: x = (omega*diag).*rhs,
 * which is what the reference computes in that case (residual == rhs exactly). */
int b200_relax(b200_ctx_t ctx, b200_csr_t A, b200_vec_t rhs, b200_vec_t x,
               b200_vec_t tmp, b200_vec_t diag, double omega);

/* ---------------------------------------------------------------- Krylov steps */

/* The vector half of a Krylov iteration as fused passes with device-resident scalars.
 *
 * The reference's solvers issue every vector update and inner product as a separate backend
 * call and carry the scalars through the host: solver/cg.hpp:180-198 is
 *   P.apply(r,s); rho = <r,s>; p = s + (rho/rho_prev) p; q = A p; alpha = rho/<q,p>;
 *   x += alpha p; r -= alpha q; <r,r>
 * = 7 calls and 3 host synchronisations per iteration (bicgstab.hpp:198-236: 6).  The steps
 * below are what the specialisations of amgcl::solver::cg / bicgstab for backend::b200
 * (include/amgcl/backend/b200.hpp) call instead: each reads its operands once, forms its
 * coefficient (a quotient of inner products) on the device from a per-context scalar table,
 * and leaves the inner products of what it just wrote in that table for the next step.  The
 * products <q,p>, <rh,v>, <t,s>, <t,t> are reduced inside the SpMV kernel that produces q / v /
 * t; <r,s> is left behind by the fused smoother sweep that ends the V-cycle (b200_relax does
 * that whenever a workspace of the operator's size exists).  On a multi-GPU context the
 * kernel that finishes a reduction also all-reduces it over the ranks through peer memory
 * (replaces mpi/inner_product.hpp:53-62).  The host synchronises only where the algorithm
 * tests convergence: once per CG iteration, twice per BiCGStab iteration.
 *
 * All vectors are FP64 vectors of the workspace's size n; A is an FP64 or FP32 operator.
 * Functions with a `double *` result are host-synchronous. */
int b200_krylov_create(b200_ctx_t ctx, size_t n, b200_krylov_t *K);
int b200_krylov_destroy(b200_krylov_t K);
/* r = rhs - A x and *rr = <r,r> in one pass; starts a new solve (cg.hpp:176-177,
 * bicgstab.hpp:180).  If x is known to be zero the pass over A is skipped (r = rhs). */
int b200_krylov_residual(b200_krylov_t K, b200_vec_t rhs, b200_csr_t A, b200_vec_t x,
                         b200_vec_t r, double *rr);
/* The workspace's scalars as the device formed them (device -> host copy, synchronises),
 * out[0..count), count <= 9: rho of the current iteration, <q,p> | <rh,v>, alpha, <t,s>,
 * <t,t>, omega, <r,r>, <s,s>, rho of the next iteration.  For tests and diagnostics. */
int b200_krylov_scalars(b200_krylov_t K, double *out, int count);

/* CG.  b200_cg_direction: rho = <r,s> (taken from the smoother's epilogue when available),
 * p = s + (rho/rho_prev) p, p = s on the first call of a solve (cg.hpp:183-189).
 * b200_cg_step: q = A p; alpha = rho/<q,p>; x += alpha p; r -= alpha q; *rr = <r,r>
 * (cg.hpp:191-198). */
int b200_cg_direction(b200_krylov_t K, b200_vec_t r, b200_vec_t s, b200_vec_t p);
int b200_cg_step(b200_krylov_t K, b200_csr_t A, b200_vec_t p, b200_vec_t q, b200_vec_t x,
                 b200_vec_t r, double *rr);

/* BiCGStab with right preconditioning (bicgstab.hpp:176-236; T = M^-1 p resp. M^-1 s is
 * applied by the caller between the steps).
 *   b200_bicg_start      rh = r; rho = <r,rh>                                   :183,200
 *   b200_bicg_direction  p = r + beta (p - omega v), beta = (rho alpha)/(rho_prev omega);
 *                        p = r on the first call of a solve                      :202-208
 *   b200_bicg_step_s     v = A T; alpha = rho/<rh,v>; x += alpha T; s = r - alpha v;
 *                        *ss = <s,s>; *rho (optional) = this iteration's rho    :210-222
 *   b200_bicg_step_r     t = A T; omega = <t,s>/<t,t>; x += omega T; r = s - omega t;
 *                        *rr = <r,r>; next rho = <r,rh>; *omega (optional)      :223-236,200
 * rho and omega are returned for the breakdown checks of bicgstab.hpp:206,228. */
int b200_bicg_start(b200_krylov_t K, b200_vec_t r, b200_vec_t rh);
int b200_bicg_direction(b200_krylov_t K, b200_vec_t r, b200_vec_t v, b200_vec_t p);
int b200_bicg_step_s(b200_krylov_t K, b200_csr_t A, b200_vec_t rh, b200_vec_t T, b200_vec_t v,
                     b200_vec_t r, b200_vec_t s, b200_vec_t x, double *ss, double *rho);
int b200_bicg_step_r(b200_krylov_t K, b200_csr_t A, b200_vec_t rh, b200_vec_t T, b200_vec_t t,
                     b200_vec_t s, b200_vec_t r, b200_vec_t x, double *rr, double *omega);

/* ---------------------------------------------------------------- coarse solve */

/* Coarsest-level direct solver (replaces solver::cuda_skyline_lu,
 * cuda.hpp:61-84): the n x n inverse is formed on the device once
 * (Gauss-Jordan, partial pivoting, FP64) and applied as a dense GEMV per
 * cycle, so nothing leaves the device inside the V-cycle. */
int b200_coarse_create_i64(b200_ctx_t ctx, int64_t n, const int64_t *ptr,
                           const int64_t *col, const double *val, b200_coarse_t *S);
int b200_coarse_create_i32(b200_ctx_t ctx, int64_t n, const int32_t *ptr,
                           const int32_t *col, const double *val, b200_coarse_t *S);
/* FP32 hierarchy: the coarse matrix arrives in FP32, the inverse is formed and kept in
 * FP64, and it is applied to FP32 vectors. */
int b200_coarse_create_i64_f32(b200_ctx_t ctx, int64_t n, const int64_t *ptr,
                               const int64_t *col, const float *val, b200_coarse_t *S);
int b200_coarse_create_i32_f32(b200_ctx_t ctx, int64_t n, const int32_t *ptr,
                               const int32_t *col, const float *val, b200_coarse_t *S);
int b200_coarse_destroy(b200_coarse_t S);
int b200_coarse_bytes(b200_coarse_t S, size_t *bytes);
/* x = A^-1 rhs */
int b200_coarse_solve(b200_ctx_t ctx, b200_coarse_t S, b200_vec_t rhs, b200_vec_t x);

/* ---------------------------------------------------------------- recorded call sequences */

/* CUDA-graph recording of a sequence of the calls above (SURVEY section 8(f) rank 1: "whole-cycle
 * CUDA graph").  The reference issues the V-cycle (amg.hpp:514-553) as ~10 library calls per
 * level from the host on every preconditioner application; between b200_graph_begin and
 * b200_graph_end the same calls are recorded instead of executed, b200_graph_end runs them once
 * and returns a graph that b200_graph_launch replays with a single launch.
 *
 * The library's host-side vector state (storage exchanged by b200_relax, pending lazy clears)
 * is part of what was recorded: b200_graph_launch compares the current state of every vector
 * the graph touches with the state at recording time and sets *launched = 0 WITHOUT doing
 * anything when they differ (or when an object the graph refers to has been destroyed, an
 * option or the stream changed, or profiling is on); the caller then records another graph or
 * issues the calls directly.  Scalars (alpha, beta, omega) and the handles passed to the recorded
 * calls are baked in: a graph recorded for apply(r, s) computes on r and s, so a caller that
 * applies the same sequence to several vector pairs keeps one graph per pair.
 *
 * While recording, host-synchronous and allocating calls (b200_dot, uploads / downloads,
 * b200_ctx_sync, object creation / destruction) fail with B200_EINVAL -- except b200_vec_destroy
 * of a vector the recording does not use (a garbage-collected handle, say), whose storage is
 * released when the recording ends; after any failure call
 * b200_graph_abort, which drops the recording and restores the vector state of
 * b200_graph_begin (nothing recorded has run).  *recording = 0 from b200_graph_begin means the
 * context cannot record right now (profiling, multi-GPU context, legacy default stream, option
 * "cycle_graph" = 0): issue the calls directly. */
int b200_graph_begin(b200_ctx_t ctx, int *recording);
int b200_graph_end(b200_ctx_t ctx, b200_graph_t *graph);     /* instantiate + run once */
int b200_graph_abort(b200_ctx_t ctx);
int b200_graph_launch(b200_ctx_t ctx, b200_graph_t graph, int *launched);
/* kernels per replay, graph nodes (kernels + memsets + copies), replays so far, staleness */
int b200_graph_info(b200_graph_t graph, int64_t *kernels, int64_t *nodes, int64_t *replays,
                    int *stale);
int b200_graph_destroy(b200_graph_t graph);

#ifdef __cplusplus
}
#endif
#endif /* AMGCL_B200_H */
