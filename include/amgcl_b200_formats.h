/* amgcl_b200_formats.h -- the column formats of the CSR operators: which one each operator and
 * each profiled pass uses, and the host-side plan of the narrow format.
 *
 * Kept apart from amgcl_b200.h on purpose: the drop-in library and the tutorial program are
 * compiled from amgcl_b200.h together with AMGCL's headers, and a machine without AMGCL's
 * headers can only install a kept build of them whose recorded source hash still matches.
 * Nothing here is used by the AMGCL backend itself. */
#ifndef AMGCL_B200_FORMATS_H
#define AMGCL_B200_FORMATS_H

#include "amgcl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Column formats, as b200_ctx_largest_operator and b200_profile_end_formats report them. */
#define B200_FMT_PLAIN    0   /* int32 column per entry                                     */
#define B200_FMT_WINDOW   1   /* 16-bit slot in a per-block shared-memory window of x       */
#define B200_FMT_OFFSET   2   /* 8-bit index of col - row                                   */
#define B200_FMT_PATTERN  3   /* no per-entry column: 8-bit row pattern id                  */
#define B200_FMT_COL16    4   /* 16-bit column relative to the block's smallest column      */
#define B200_FMT_COL24    5   /* the same in 24 bits (a 16-bit and an 8-bit array)          */
#define B200_FMT_PATVAL   6   /* no per-entry data: 8-bit row pattern id, values in the     */
                              /* pattern table as well                                      */

/* Value-keyed patterns.  Where the pairs (col - row, value) of the rows also take at most 256
 * patterns of at most 1024 entries in all (a stencil operator with constant coefficients: 27
 * patterns for the 7-point Poisson problem), a single-GPU operator that qualifies for the
 * pattern-indexed format keeps each entry's value in the pattern table too.  The streaming
 * passes then read one byte per row and nothing per entry: the row's pattern id gives its
 * length, columns and values.  Values are compared bit for bit (-0.0, +0.0 and NaN payloads
 * are distinct).  The table is kept in FP64 and, where every table value is exact in FP32 and
 * "narrow_values" applies, in FP32; the passes multiply the same doubles either way, so every
 * result keeps its bits.  Such an operator keeps no FP32 copy and no value index.  Context
 * option "pattern_values" (b200_ctx_set_option; env B200_PATTERN_VALUES): 1 = built at upload
 * and used where the tables fit beside the ring of stages (default), 0 = not built / not used
 * (the passes stream the FP64 values, format B200_FMT_PATTERN).  A pass on such an operator
 * reports B200_FMT_PATVAL, and as value_bytes the width of the table it reads (4 or 8).
 * b200_pattern_value_plan_i64: pure host helper for tests, the value-keyed plan b200_csr_create
 * tries first (pid_out [nrows], start_out [257], off_out / val_out [1024]; qualifies 0: too
 * many patterns; exact_f32 1: every table value survives double -> float -> double). */
int b200_pattern_value_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col,
                                const double *val, uint8_t *pid_out, uint16_t *start_out, int32_t *off_out,
                                double *val_out, int *count, int *total, int *exact_f32, int *qualifies);

/* Narrow columns.  Inside one row block the columns of an operator span far less than the
 * int32 range.  An operator that is neither pattern- nor offset-indexed (nor windowed), has no
 * long row blocks and at most 8 lanes per row stores, per row block, its smallest column and,
 * per entry, the low 16 bits of (column - that base) plus, if some block spans more than
 * 2^16 - 1 columns, the high 8 bits in a second array; the streaming kernel reads 2 or 3
 * instead of 4 bytes of column per entry.  Same entry order and arithmetic, same bits.
 * Context option "narrow_columns" (b200_ctx_set_option; env B200_NARROW_COLUMNS): 1 = built at
 * upload and used (default), 0 = not built / not used.
 * Every staged format streams 16-bit row pointers relative to the first non-zero of the row's
 * block.
 * b200_csr_narrow: 16 or 24, or 0 when A is not stored that way.
 * b200_narrow_plan_i64: pure host helper for tests, the plan b200_csr_create builds for a
 * single-GPU operator (base_out [nblocks], lo16_out / hi8_out [nnz], ptr16_out [nrows];
 * width_out 0: stays plain). */
int b200_csr_narrow(b200_csr_t A, int *width);
int b200_narrow_plan_i64(int64_t nrows, int64_t ncols, const int64_t *ptr, const int64_t *col, int lanes,
                         int nnz_cap, int32_t *base_out, int64_t base_capacity, uint16_t *lo16_out,
                         uint8_t *hi8_out, uint16_t *ptr16_out, int64_t *nblocks_out, int *width_out);

/* Narrow values.  An FP64 operator with at least "narrow_values_min_nnz" non-zeros (default 1e6)
 * whose every value has the same bits after double -> float -> double (integer and dyadic
 * stencils, graph Laplacians, matrices assembled from FP32 data) also stores its values as FP32,
 * and the streaming passes read 4 instead of 8 bytes per value.  The widened value is the same
 * double, so every product, row sum and result keeps its bits.  The FP64 values stay: the
 * one-block-per-CTA variant (spmv_variant 0), the small-operator kernel and the coarse tail read
 * them.  Context option "narrow_values" (b200_ctx_set_option; env B200_NARROW_VALUES): 1 = built
 * at upload and used (default), 0 = not built / not used.
 * Indexed values.  Otherwise an FP64 operator of that size whose values take at most 4,096
 * distinct 64-bit patterns (the prolongation, restriction and first coarse operator of smoothed
 * aggregation on a structured grid) also stores, per entry, the 8-bit (at most 256 values) or
 * 16-bit index of its value in a table of the distinct values sorted by bit pattern; the
 * streaming passes read 1 or 2 bytes per value and take the double from the table, the same
 * double, so again every result keeps its bits.  Only on a single-GPU context, for an operator
 * without long row blocks that is not windowed, and only where the table fits in shared memory
 * beside the configured ring of stages (checked at upload and at every launch; otherwise the
 * passes read the FP64 values).  Same option and threshold.
 * b200_csr_value_bytes: 1, 2, 4 or 8, the bytes per value the streaming passes read from A.
 * b200_values_fit_f32: pure host helper for tests, the rule b200_csr_create applies to n values
 * (qualifies 1: every value survives the round trip).
 * b200_value_index_plan_i64: pure host helper for tests, the index b200_csr_create builds from n
 * values: width_out 8 or 16, or 0 when there are more than 4,096 distinct values (count_out is
 * then 4097); count_out distinct values into table_out (capacity >= count_out, may be NULL);
 * idx_out (may be NULL) receives n uint8_t (width 8) or n uint16_t (width 16). */
int b200_csr_value_bytes(b200_csr_t A, int *bytes);
int b200_values_fit_f32(const double *val, int64_t n, int *qualifies);
int b200_value_index_plan_i64(const double *val, int64_t n, double *table_out, int64_t table_capacity,
                              void *idx_out, int *count_out, int *width_out);

/* b200_profile_end with the column format (B200_FMT_*) and the bytes per stored value (1 to 8)
 * each CSR pass streamed (0 and 0 for the other kernels).  Entries are aggregated per
 * (shape, mode, format, value width). */
typedef struct {
    b200_profile_entry entry;
    int                format;
    int                value_bytes;
} b200_profile_format_entry;
int b200_profile_end_formats(b200_ctx_t ctx, b200_profile_format_entry *out, int64_t capacity,
                             int64_t *count);

#ifdef __cplusplus
}
#endif

#endif /* AMGCL_B200_FORMATS_H */
