// api_patterns.cu -- the pattern-indexed launches of the streaming CSR kernel (csr_kernels.cuh,
// FMT_PATTERN; format built by patterns.cuh at upload): every pass of csr_launch.cuh's table on
// 1..4 lanes per row, with and without the multi-GPU halo, and its indexed passes without it.  A
// translation unit of its own: the units compile concurrently.
#include "csr_launch.cuh"

B200_RING_UNIT(FMT_PATTERN, 4, 1)
