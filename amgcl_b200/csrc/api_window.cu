// api_window.cu -- the windowed launches of the streaming CSR kernel (csr_kernels.cuh, FMT_WINDOW;
// format built by window.cuh at upload): every pass of csr_launch.cuh's table on 1..8 lanes per
// row, with and without the multi-GPU halo.  A translation unit of its own: the units compile
// concurrently.
#include "csr_launch.cuh"

B200_RING_UNIT(FMT_WINDOW, 8, 0)
