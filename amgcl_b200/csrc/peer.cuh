// peer.cuh -- exchange kernels over NVLink peer memory (multi-GPU, one process per GPU).
//
// The collectives of the partitioned solve are tiny (a halo plane, one coarse
// vector, one scalar) and sit on the critical path ~200 times per solve, so their
// cost is latency, not bandwidth: an NCCL call costs tens of microseconds each on NVSwitch.
// Here every rank maps its peers'
// exchange buffers once (CUDA IPC) and the data moves with plain stores from our own
// kernels:
//
//   producer side      lives in the CONSUMER kernel of the same exchange (csr_kernels.cuh,
//                      halo_push): right after its grid dependency resolves, every CTA of
//                      the streaming kernel packs a slice of this rank's boundary values
//                      straight into each consumer's buffer over NVLink (st.global on mapped
//                      peer pointers); the last CTA done -- after a system-scope fence --
//                      releases one 64-bit flag per consumer (st.release.sys).  No launch of
//                      its own, and the transfer overlaps the interior rows.
//   consumer side      the same kernel: row blocks that gather remote columns are walked
//                      last and spin (ld.acquire.sys) until the flags of the producers they
//                      depend on carry the expected sequence number (wait_for_halo).
//   gather_copy_kernel row shares of a replicated result: waits for every rank's flag, then
//                      copies the all-gathered shares into the result vector.
//
// Buffers are double-buffered by the parity of a per-object sequence number.  That suffices
// against write-after-read because every pair of ranks that exchanges data exchanges flags in
// BOTH directions (the dependency pattern is made symmetric at set-up, api_matrices.cu): a rank
// can only pass exchange k+1 after its partner started exchange k+1, i.e. after the partner's
// exchange-k consumer finished (stream order), so nobody writes parity k&1 again (exchange
// k+2) while a partner still reads it.
#pragma once
#include "common.cuh"

namespace b200 {

// (kMaxRanks, kFlagStride, kFlagBytes: common.cuh)

struct WaitList {
    const unsigned long long *flag[kMaxRanks];   // local flags to wait on (nullptr: skip)
};

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// dst[i] = staged[i], i < count, once the shares of all ranks have landed: the row shares of a
// replicated result (R onto a small level) were stored straight into every rank's gather
// buffer by the kernels that computed them (csr_kernels.cuh: gather_data / gather_finish).
template <class T>
__global__ void __launch_bounds__(kThreads)
gather_copy_kernel(int64_t count, const T *staged, WaitList w, int nranks,
                   unsigned long long seq, T *__restrict__ dst) {
    if (threadIdx.x < nranks && w.flag[threadIdx.x]) {
        while (ld_acquire_sys(w.flag[threadIdx.x]) < seq) { __nanosleep(20); }
    }
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
        dst[i] = __ldcv(staged + i);
}

// ---- device helper: pack this rank's boundary values into its halo segment ----------
template <class T>
__global__ void __launch_bounds__(kThreads)
halo_pack_kernel(int64_t count, const int *__restrict__ send_idx, const T *__restrict__ x,
                 T *__restrict__ segment) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) segment[i] = x[send_idx[i]];
}

} // namespace b200
