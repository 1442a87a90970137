// api_col16.cu -- the narrow-column (16-bit) launches of the streaming CSR kernel (csr_kernels.cuh,
// FMT_COL16; format built by narrow.cuh at upload): every pass of csr_launch.cuh's table on 1..8
// lanes per row, with and without the multi-GPU halo, and its indexed passes without it.  A
// translation unit of its own: the units compile concurrently.
#include "csr_launch.cuh"

B200_RING_UNIT(FMT_COL16, 8, 1)
