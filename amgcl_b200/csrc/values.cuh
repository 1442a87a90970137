// values.cuh -- host-side construction of indexed values (csr_kernels.cuh, PrecI8D / PrecI16D):
// an FP64 operator with at most 4,096 distinct values stores, per entry, the 8-bit (at most 256
// values) or 16-bit index of its value in a table sorted by bit pattern.  The kernel reads the
// double from the table in shared memory, so it multiplies exactly the double it is given.
//
// Smoothed aggregation builds such operators on every structured-grid problem: P = (I - w D^-1 A)
// P_tent of a stencil operator, its transpose and the first coarse operator R A P take a few
// hundred to a few thousand distinct values (DESIGN.md section 3.1b).
//
// Values are compared as 64-bit patterns: -0.0 and +0.0, every NaN payload, infinities and
// subnormals are distinct values and come back bit for bit.
//
// Pure host logic (exported as b200_value_index_plan_i64 for the CPU tests), on all host threads.
#pragma once
#include "common.cuh"

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <vector>
#include <omp.h>

namespace b200 {

constexpr int kValTabCap = 4096;   // most distinct values of an indexed operator

struct ValueIndexPlan {
    int width = 0;                       // 8 or 16 bits per entry; 0: more than kValTabCap values
    int count = 0;                       // distinct values (kValTabCap + 1: more than kValTabCap)
    std::vector<uint64_t>       tab;     // [count] the distinct bit patterns, ascending
    std::vector<unsigned char>  idx8;    // [n] width 8: index of every value in tab
    std::vector<unsigned short> idx16;   // [n] width 16
};

// open-addressing set / map of 64-bit patterns, large enough for kValTabCap + 1 keys
struct BitsTable {
    static constexpr int kSlots = 16384;
    std::vector<uint64_t> key;
    std::vector<int>      val;           // -1: empty slot
    BitsTable() : key(kSlots, 0), val(kSlots, -1) {}
    static unsigned slot(uint64_t b) { return (unsigned)((b * 0x9E3779B97F4A7C15ull) >> 50); }
    // the slot holding b, or the empty slot where it would go
    unsigned find(uint64_t b) const {
        unsigned s = slot(b);
        while (val[s] >= 0 && key[s] != b) s = (s + 1) & (kSlots - 1);
        return s;
    }
};

inline uint64_t value_bits(const double *v) {
    uint64_t b;
    memcpy(&b, v, 8);
    return b;
}

// Returns false when the n values take more than kValTabCap distinct bit patterns (counting stops
// as soon as one thread has seen that many).
inline bool build_value_index(const double *val, int64_t n, ValueIndexPlan &o) {
    o.width = 0; o.count = 0;
    o.tab.clear(); o.idx8.clear(); o.idx16.clear();
    if (n < 0 || (n > 0 && !val)) return false;
    const int nth = std::max(1, omp_get_max_threads());
    std::vector<std::vector<uint64_t>> seen((size_t)nth);
    std::atomic<int> over(0);
    int used = 1;
#pragma omp parallel num_threads(nth)
    {
        const int tid = omp_get_thread_num(), nt = omp_get_num_threads();
#pragma omp single
        used = nt;
        BitsTable set;
        std::vector<uint64_t> &mine = seen[(size_t)tid];
        const int64_t lo = n * tid / nt, hi = n * (tid + 1) / nt;
        uint64_t last = 0;
        bool have_last = false;
        for (int64_t e0 = lo; e0 < hi && !over.load(std::memory_order_relaxed); e0 += 65536) {
            const int64_t e1 = std::min(hi, e0 + 65536);
            for (int64_t e = e0; e < e1; ++e) {
                const uint64_t b = value_bits(val + e);
                if (have_last && b == last) continue;           // runs of one value are common
                last = b; have_last = true;
                const unsigned s = set.find(b);
                if (set.val[s] >= 0) continue;
                if ((int)mine.size() == kValTabCap) { over.store(1, std::memory_order_relaxed); break; }
                set.key[s] = b; set.val[s] = 0;
                mine.push_back(b);
            }
        }
    }
    if (over.load()) { o.count = kValTabCap + 1; return false; }
    std::vector<uint64_t> all;
    for (int t = 0; t < used; ++t) all.insert(all.end(), seen[(size_t)t].begin(), seen[(size_t)t].end());
    std::sort(all.begin(), all.end());
    all.erase(std::unique(all.begin(), all.end()), all.end());
    if ((int)all.size() > kValTabCap) { o.count = kValTabCap + 1; return false; }
    o.count = (int)all.size();
    o.tab = all;
    o.width = o.count <= 256 ? 8 : 16;
    BitsTable map;
    for (int i = 0; i < o.count; ++i) {
        const unsigned s = map.find(o.tab[(size_t)i]);
        map.key[s] = o.tab[(size_t)i]; map.val[s] = i;
    }
    if (o.width == 8) o.idx8.assign((size_t)n, 0);
    else o.idx16.assign((size_t)n, 0);
#pragma omp parallel num_threads(nth)
    {
        const int tid = omp_get_thread_num(), nt = omp_get_num_threads();
        const int64_t lo = n * tid / nt, hi = n * (tid + 1) / nt;
        uint64_t last = 0;
        int k = -1;
        for (int64_t e = lo; e < hi; ++e) {
            const uint64_t b = value_bits(val + e);
            if (k < 0 || b != last) { last = b; k = map.val[map.find(b)]; }
            if (o.width == 8) o.idx8[(size_t)e] = (unsigned char)k;
            else o.idx16[(size_t)e] = (unsigned short)k;
        }
    }
    return true;
}

} // namespace b200
