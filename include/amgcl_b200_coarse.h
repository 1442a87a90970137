/* amgcl_b200_coarse.h -- coarsest levels above the dense inverse's 16384 rows: the banded LU
 * behind b200_coarse_t, how to tell which representation a handle holds, and the host-side
 * plan of the banded LU.
 *
 * Kept apart from amgcl_b200.h for the reason amgcl_b200_formats.h gives: the drop-in library
 * and the tutorial program are compiled from amgcl_b200.h together with AMGCL's headers, and a
 * machine without AMGCL's headers can only install a kept build of them whose recorded source
 * hash still matches.  The AMGCL backend needs nothing from here: b200_coarse_create_* chooses
 * the representation itself.
 *
 * b200_coarse_create_* (amgcl_b200.h) chooses from n alone:
 *   n <= 16384  the n x n inverse, formed once on the device (Gauss-Jordan, partial pivoting,
 *               FP64) and applied as a dense GEMV per cycle;
 *   n >  16384  banded LU: the matrix is ordered by reverse Cuthill-McKee, factored on the
 *               device without pivoting (as solver::skyline_lu does, skyline_lu.hpp:74-95) in
 *               FP64 into tiles of 64 rows, and each solve is one forward and one backward
 *               sweep.  The limit is device memory: the factor takes about
 *               8 * n * (lower + upper bandwidth) bytes after the ordering, and B200_ENOMEM is
 *               returned before anything is allocated when factor and factorisation scratch
 *               would not fit.  Multi-GPU contexts keep the 16384-row limit.
 * Both give B200_ESINGULAR when a pivot is non-finite or below 1e-14 of the largest (on the
 * banded path also for a zero pivot of a non-singular matrix, as skyline_lu would divide by it). */
#ifndef AMGCL_B200_COARSE_H
#define AMGCL_B200_COARSE_H

#include "amgcl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* profile mode of the banded-LU sweeps (b200_profile_end; see B200_PROF_COARSE for the GEMV) */
#define B200_PROF_COARSE_LU    25

/* Which representation S holds (B200_COARSE_*), its size, and for the banded LU the larger of
 * the lower and upper bandwidths of the ordered matrix and the number of 64-row tiles (both 0
 * for the dense inverse). */
#define B200_COARSE_DENSE      0
#define B200_COARSE_BANDED_LU  1
int b200_coarse_info(b200_coarse_t S, int *kind, int64_t *n, int64_t *bandwidth, int64_t *tiles);

/* Pure host helper (no device needed): the symbolic phase of the banded LU for a host matrix.
 * perm_out [n] (may be NULL): perm_out[new] = old row (reverse Cuthill-McKee of the
 * symmetrised pattern).  lower_out [n] / upper_out [n] (may be NULL): per-row lower and
 * per-column upper bandwidth of the permuted matrix.  lfirst_out / ulast_out [tiles] (may be
 * NULL, tiles_capacity entries): per tile of *tile_rows rows, the first tile its L panel
 * reaches and the last tile its U panel reaches.  *factor_bytes is what the solver keeps on
 * the device, *setup_bytes the extra device memory the factorisation needs while it runs. */
int b200_coarse_lu_plan_i64(int64_t n, const int64_t *ptr, const int64_t *col, int32_t *perm_out,
                            int32_t *lower_out, int32_t *upper_out, int64_t *lfirst_out,
                            int64_t *ulast_out, int64_t tiles_capacity, int64_t *tiles,
                            int *tile_rows, int64_t *bandwidth, size_t *factor_bytes,
                            size_t *setup_bytes);

#ifdef __cplusplus
}
#endif
#endif /* AMGCL_B200_COARSE_H */
