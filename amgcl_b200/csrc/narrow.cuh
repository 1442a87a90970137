// narrow.cuh -- host-side construction of the narrow column format (csr_kernels.cuh,
// FMT_COL16 / FMT_COL24) and of the block-relative row pointers every staged format streams.
//
// Inside one row block the columns span far less than the int32 range: on every operator of a
// smoothed-aggregation hierarchy of a structured problem a block's largest column minus its
// smallest fits 16 bits (prolongations, coarse levels) or 24 bits (restrictions, the first
// coarse operator).  Such an operator stores, per block, its smallest column and, per entry, the
// low 16 bits of (column - base) and -- width 24 only -- the high 8 bits in an array of their
// own, so the kernel streams 2 or 3 bytes of column per entry instead of 4.  One width holds
// for the whole operator: the narrowest that every block fits.
//
// Pure host logic (exported as b200_narrow_plan_i64 for the CPU tests), on all host threads.
#pragma once
#include "common.cuh"
#include "csr_kernels.cuh"

#include <algorithm>
#include <cstdint>
#include <vector>

namespace b200 {

struct NarrowPlan {
    int width = 0;                        // 16 or 24
    std::vector<int>            base;     // [nblocks] walk order: smallest column of the block (0 if empty)
    std::vector<unsigned short> lo16;     // [nnz] low 16 bits of col - base
    std::vector<unsigned char>  hi8;      // [nnz] high 8 bits (width 24 only)
};

// blk4: the block descriptors in walk order ({r0 or ~r0, r1, e0, e1}).  Returns false when some
// block's columns span more than 2^24 - 1.
template <class Col>
inline bool build_narrow(const int4 *blk4, int64_t nblocks, const Col *col, int64_t nnz, NarrowPlan &o) {
    o.width = 0;
    if (nblocks <= 0 || nnz <= 0) return false;
    o.base.assign((size_t)nblocks, 0);
    int64_t widest = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(max : widest)
    for (int64_t b = 0; b < nblocks; ++b) {
        const int e0 = blk4[b].z, e1 = blk4[b].w;
        if (e0 == e1) continue;
        int64_t lo = (int64_t)col[e0], hi = lo;
        for (int e = e0 + 1; e < e1; ++e) {
            const int64_t c = (int64_t)col[e];
            lo = std::min(lo, c);
            hi = std::max(hi, c);
        }
        o.base[(size_t)b] = (int)lo;
        widest = std::max(widest, hi - lo);
    }
    if (widest > 0xffffff) return false;
    o.width = widest <= 0xffff ? 16 : 24;
    o.lo16.assign((size_t)nnz, 0);
    if (o.width == 24) o.hi8.assign((size_t)nnz, 0);
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t b = 0; b < nblocks; ++b) {
        const int base = o.base[(size_t)b];
        for (int e = blk4[b].z; e < blk4[b].w; ++e) {
            const unsigned rel = (unsigned)((int64_t)col[e] - base);
            o.lo16[(size_t)e] = (unsigned short)(rel & 0xffff);
            if (o.width == 24) o.hi8[(size_t)e] = (unsigned char)(rel >> 16);
        }
    }
    return true;
}

// Block-relative row pointers: ptr16[r] = ptr[r] - e0 of the block that holds row r.  A staged
// block has at most nnz_cap (<= kNnzCapMax) entries, so they fit 16 bits; the rows of a long
// block (never staged) get 0.
inline void build_ptr16(const int4 *blk4, int64_t nblocks, const int32_t *ptr, int nnz_cap,
                        std::vector<unsigned short> &ptr16) {
    static_assert(kNnzCapMax <= 0xffff, "a staged block's row pointers must fit 16 bits");
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t b = 0; b < nblocks; ++b) {
        const int4 q = blk4[b];
        const int r0 = q.x < 0 ? ~q.x : q.x;
        const bool staged = q.w - q.z <= nnz_cap;
        for (int r = r0; r < q.y; ++r) ptr16[(size_t)r] = staged ? (unsigned short)(ptr[r] - q.z) : 0;
    }
}

} // namespace b200
