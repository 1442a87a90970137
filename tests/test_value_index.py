"""Host-side planner behind indexed values (b200_value_index_plan_i64, csrc/values.cuh): an FP64
operator with at most 4,096 distinct 64-bit value patterns is also stored as the 8-bit (<= 256
values) or 16-bit index of every value in a table of the distinct patterns, ascending.  The
streaming passes read table[index], so every pattern must come back bit for bit."""
import struct

import numpy as np
import pytest

import amgcl_b200 as ab
import oracle


def from_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def check(val):
    """Plan val; if indexed, the table is the sorted distinct patterns and table[index] == val
    bit for bit."""
    o = ab.value_index_plan(val)
    want = np.unique(bits(val))
    if want.size > 4096:
        assert o == {"width": 0, "count": 4097}
        return o
    assert o["count"] == want.size
    assert o["width"] == (8 if want.size <= 256 else 16)
    assert o["index"].dtype == (np.uint8 if o["width"] == 8 else np.uint16)
    np.testing.assert_array_equal(bits(o["table"]), want)
    np.testing.assert_array_equal(bits(o["table"][o["index"]]), bits(val))
    return o


def distinct(k, n, seed):
    """n values taking exactly k distinct patterns, shuffled."""
    rng = np.random.default_rng(seed)
    pool = rng.standard_normal(k) * np.exp2(rng.integers(-30, 30, k))
    assert np.unique(bits(pool)).size == k
    v = np.concatenate([pool, rng.choice(pool, n - k)])
    rng.shuffle(v)
    return v


@pytest.mark.parametrize("k,width", [(1, 8), (255, 8), (256, 8), (257, 16), (4095, 16), (4096, 16), (4097, 0)])
def test_width_at_the_boundaries(k, width):
    o = check(distinct(k, 300_000, k))
    assert o["width"] == width


def test_many_distinct_values_are_refused():
    o = check(np.random.default_rng(3).standard_normal(2_000_000))
    assert o["width"] == 0


SPECIAL = {
    "+0": 0.0,
    "-0": -0.0,
    "+inf": float("inf"),
    "-inf": float("-inf"),
    "quiet NaN": from_bits(0x7FF8000000000000),
    "NaN with payload 1": from_bits(0x7FF8000000000001),
    "negative NaN with payload": from_bits(0xFFF80000DEADBEEF),
    "signalling NaN": from_bits(0x7FF0000000000001),
    "smallest double subnormal": 5e-324,
    "largest double subnormal": from_bits(0x000FFFFFFFFFFFFF),
    "negative subnormal": -from_bits(0x0000000000001234),
    "1/9": 1.0 / 9.0,
}


def test_special_patterns_are_distinct_and_round_trip():
    rng = np.random.default_rng(11)
    # (built from the bit patterns: a NaN payload need not survive a trip through Python floats)
    pool = np.array([struct.unpack("<Q", struct.pack("<d", v))[0] for v in SPECIAL.values()],
                    dtype=np.uint64).view(np.float64)
    v = pool[rng.integers(0, pool.size, 100_000)]
    o = check(v)
    assert o["count"] == len(SPECIAL)


def test_table_order_does_not_depend_on_entry_order():
    v = distinct(1000, 500_000, 7)
    a = ab.value_index_plan(v)
    w = v[::-1].copy()
    b = ab.value_index_plan(w)
    np.testing.assert_array_equal(bits(a["table"]), bits(b["table"]))
    np.testing.assert_array_equal(a["index"][::-1], b["index"])
    assert np.all(np.diff(bits(a["table"]).astype(np.uint64)) > 0)


def test_empty_input():
    o = ab.value_index_plan(np.zeros(0))
    assert o["width"] == 8 and o["count"] == 0


@pytest.mark.skipif(not oracle.have_ref(), reason="reference build (oracle/_ref) not available")
@pytest.mark.parametrize("n", [64, 128])
def test_reference_hierarchy_widths(n):
    """Smoothed aggregation on Poisson: A0 is exact in FP32 (which takes precedence), P0 and R0
    take at most 256 distinct values, A1 at most 4,096; every other operator stays FP64."""
    ptr, col, val, _ = ab.poisson3d(n)
    S = oracle.RefSolver(ptr, col, val, "damped_jacobi", "cg")
    got = {}
    for lvl in range(S.nlevels - 1):
        for w in "APR":
            _, _, (_, _, v) = S.level_matrix(lvl, w)
            fp32 = ab.values_fit_f32(v)
            o = check(v)
            got[(lvl, w)] = 32 if fp32 else o["width"]
    want = {k: 0 for k in got}
    want.update({(0, "A"): 32, (0, "P"): 8, (0, "R"): 8, (1, "A"): 16})
    assert got == want
