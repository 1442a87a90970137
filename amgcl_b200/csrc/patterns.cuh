// patterns.cuh -- host-side construction of the pattern-indexed row format (csr_kernels.cuh,
// FMT_PATTERN): the tuple (col - row of every entry, in entry order) of a row is its pattern; if
// the operator has at most 256 distinct patterns whose offsets total at most 1024, every row is
// stored as the 8-bit id of its pattern and the entries carry no column information at all.
//
// Value-keyed patterns (FMT_PATVAL).  Keyed on the pairs (col - row, bit pattern of the value) of
// its entries instead, a pattern also fixes the row's values: on a stencil operator every row
// with a given offset pattern has the same values (27 patterns for the Poisson problem either
// way).  Within the same caps every row is then one byte -- the kernel takes columns, values and
// the row length from the tables.  Values are compared as bit patterns (values.cuh): -0.0 and
// +0.0 and every NaN payload are distinct and come back bit for bit.
//
// Pure host logic (exported as b200_pattern_plan_i64 / b200_pattern_value_plan_i64 for the CPU
// tests).  One pass over the entries on all host threads: a row usually repeats the pattern of
// the row before it, which is checked first; only a row that differs is looked up in the
// thread's pattern list.
#pragma once
#include "common.cuh"
#include "csr_kernels.cuh"

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <utility>
#include <vector>
#include <omp.h>

namespace b200 {

struct PatternPlan {
    std::vector<unsigned char>  pid;       // [nrows] pattern of every row
    std::vector<unsigned short> start;     // [kPatCap + 1] first table entry of every pattern
    std::vector<int>            off;       // [kPatOffCap] the patterns' offsets, one after the other
    int count = 0, total = 0;
    // value-keyed plans only: the value of every table entry, parallel to off
    bool                        values = false;
    std::vector<double>         val;       // [kPatOffCap] (an FP32 operator's values, widened)
    std::vector<float>          val32;     // [kPatOffCap] the same values as FP32 where exact
    bool                        val_f32 = false;   // every table value survives double -> float -> double
};

inline uint64_t pattern_value_bits(const double *v) { uint64_t b; memcpy(&b, v, 8); return b; }
inline uint64_t pattern_value_bits(const float *v) { uint32_t b; memcpy(&b, v, 4); return b; }

// Returns false when the operator has too many patterns.  val == nullptr: patterns of offsets
// only; otherwise of (offset, value) pairs, and the plan carries the table of values.
template <class Col, class Val = double>
inline bool build_patterns(int64_t nrows, const int32_t *ptr, const Col *col, PatternPlan &o,
                           const Val *val = nullptr) {
    const int64_t nnz = nrows ? ptr[nrows] : 0;
    if (nrows <= 0 || nnz <= 0) return false;
    const int nth = std::max(1, omp_get_max_threads());
    typedef std::vector<std::pair<int, uint64_t>> Pat;             // (col - row, value bits or 0)
    auto entry = [&](int64_t r, int64_t e) -> std::pair<int, uint64_t> {
        return std::make_pair((int)((int64_t)col[e] - r), val ? pattern_value_bits(val + e) : (uint64_t)0);
    };
    std::vector<std::vector<Pat>> lists((size_t)nth);          // each thread's patterns, in order of appearance
    std::vector<int> local((size_t)nrows);                      // row -> index in its thread's list
    int bad = 0, used = 1;
#pragma omp parallel num_threads(nth)
    {
        const int tid = omp_get_thread_num(), nt = omp_get_num_threads();
#pragma omp single
        used = nt;
        std::vector<Pat> &list = lists[(size_t)tid];
        std::map<Pat, int> index;
        Pat cur;
        int prev = -1;
        bool fail = false;
        const int64_t lo = nrows * tid / nt, hi = nrows * (tid + 1) / nt;
        for (int64_t r = lo; r < hi && !fail; ++r) {
            const int64_t e0 = ptr[r], e1 = ptr[r + 1];
            const int len = (int)(e1 - e0);
            // the pattern of the row above?
            bool same = prev >= 0 && (int)list[(size_t)prev].size() == len;
            if (same) {
                const Pat &p = list[(size_t)prev];
                for (int k = 0; k < len && same; ++k) same = p[(size_t)k] == entry(r, e0 + k);
            }
            if (!same) {
                if (len > kPatOffCap) { fail = true; break; }
                cur.resize((size_t)len);
                for (int k = 0; k < len; ++k) cur[(size_t)k] = entry(r, e0 + k);
                std::map<Pat, int>::iterator it = index.find(cur);
                if (it == index.end()) {
                    if ((int)list.size() >= kPatCap) { fail = true; break; }
                    prev = (int)list.size();
                    list.push_back(cur);
                    index[cur] = prev;
                } else {
                    prev = it->second;
                }
            }
            local[(size_t)r] = prev;
        }
        if (fail) {
#pragma omp atomic write
            bad = 1;
        }
    }
    if (bad) return false;
    // global pattern list + every thread's local -> global translation
    std::map<Pat, int> gindex;
    std::vector<const Pat *> gl;
    std::vector<std::vector<unsigned char>> xlat((size_t)used);
    int total = 0;
    for (int t = 0; t < used; ++t) {
        xlat[(size_t)t].resize(lists[(size_t)t].size());
        for (size_t i = 0; i < lists[(size_t)t].size(); ++i) {
            const Pat &p = lists[(size_t)t][i];
            std::map<Pat, int>::iterator it = gindex.find(p);
            int g;
            if (it == gindex.end()) {
                if ((int)gl.size() >= kPatCap || total + (int)p.size() > kPatOffCap) return false;
                g = (int)gl.size();
                gl.push_back(&p);
                gindex[p] = g;
                total += (int)p.size();
            } else {
                g = it->second;
            }
            xlat[(size_t)t][i] = (unsigned char)g;
        }
    }
    o.count = (int)gl.size();
    o.total = total;
    o.start.assign((size_t)kPatCap + 1, (unsigned short)total);
    o.off.assign((size_t)kPatOffCap, 0);
    o.values = val != nullptr;
    o.val.assign(o.values ? (size_t)kPatOffCap : 0, 0.0);
    o.val32.assign(o.values ? (size_t)kPatOffCap : 0, 0.0f);
    o.val_f32 = o.values;
    int pos = 0;
    for (int g = 0; g < o.count; ++g) {
        o.start[(size_t)g] = (unsigned short)pos;
        for (const std::pair<int, uint64_t> &p : *gl[(size_t)g]) {
            o.off[(size_t)pos] = p.first;
            if (o.values) {
                // the table's values, bit for bit: the stored ones, and their FP32 twins where exact
                if (sizeof(Val) == 8) {
                    double d;
                    memcpy(&d, &p.second, 8);
                    const float f = (float)d;
                    const double w = (double)f;
                    o.val[(size_t)pos] = d;
                    o.val32[(size_t)pos] = f;
                    o.val_f32 = o.val_f32 && memcmp(&w, &d, 8) == 0;
                } else {
                    const uint32_t b = (uint32_t)p.second;
                    float f;
                    memcpy(&f, &b, 4);
                    o.val[(size_t)pos] = (double)f;
                    o.val32[(size_t)pos] = f;
                }
            }
            ++pos;
        }
    }
    o.pid.resize((size_t)nrows);
#pragma omp parallel for schedule(static, 1)
    for (int t = 0; t < used; ++t) {                   // (the row ranges of the first pass)
        const int64_t lo = nrows * t / used, hi = nrows * (t + 1) / used;
        const std::vector<unsigned char> &x = xlat[(size_t)t];
        for (int64_t r = lo; r < hi; ++r) o.pid[(size_t)r] = x[(size_t)local[(size_t)r]];
    }
    return true;
}

} // namespace b200
