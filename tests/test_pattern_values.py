"""CPU checks of the value-keyed pattern plan (amgcl_b200/csrc/patterns.cuh through
b200_pattern_value_plan_i64): row + off[start[pid] + k] must reproduce the column and
val[start[pid] + k] the bits of the value of every entry, within the caps of the pattern format
(256 patterns, 1024 entries in all)."""
import numpy as np

import amgcl_b200 as ab
from test_offsets import diag_matrix


def bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)


def decode(o, ptr):
    """(column, value) of every entry as the kernel rebuilds them from the tables."""
    nr = ptr.size - 1
    lens = np.diff(ptr)
    assert (o["start"][o["pid"].astype(np.int64) + 1] - o["start"][o["pid"]] == lens).all()
    rows = np.repeat(np.arange(nr, dtype=np.int64), lens)
    k = np.arange(ptr[-1]) - np.repeat(ptr[:-1], lens)
    e = np.repeat(o["start"][o["pid"]].astype(np.int64), lens) + k
    return rows + o["off"][e], o["val"][e]


def check(o, ptr, col, val):
    c, v = decode(o, ptr)
    assert (c == col).all()
    assert (bits(v) == bits(val)).all()
    assert o["start"][o["count"]] == o["total"]


def diagonal(values):
    """Square operator of one entry per row: row r holds values[r] on the diagonal."""
    n = len(values)
    return np.arange(n + 1, dtype=np.int64), np.arange(n, dtype=np.int64), np.asarray(values, dtype=np.float64)


def test_poisson_keeps_its_27_patterns_and_an_exact_fp32_table():
    for n in (6, 12):
        ptr, col, val, rhs = ab.poisson3d(n)
        nr = ptr.size - 1
        o = ab.pattern_value_plan(nr, nr, ptr, col, val)
        assert o is not None and o["count"] == 27 and o["total"] == 135 and o["exact_f32"]
        check(o, ptr, col, val)
        p = ab.pattern_plan(nr, nr, ptr, col)
        assert (o["pid"] == p["pid"]).all() and (o["start"] == p["start"]).all() and (o["off"] == p["off"]).all()


def test_anisotropic_poisson_qualifies_with_an_inexact_table():
    ptr, col, val, rhs = ab.poisson3d(10, anisotropy=0.3)
    nr = ptr.size - 1
    assert not ab.values_fit_f32(val)
    o = ab.pattern_value_plan(nr, nr, ptr, col, val)
    assert o is not None and o["count"] == 27 and not o["exact_f32"]
    check(o, ptr, col, val)


def test_random_values_decline_but_the_offsets_still_qualify():
    ptr, col, val = diag_matrix(3001, 3001, [-50, -1, 0, 1, 50], seed=3, keep=1.0)
    val = np.random.default_rng(3).uniform(-1, 1, col.size)
    assert ab.pattern_value_plan(3001, 3001, ptr, col, val) is None
    assert ab.pattern_plan(3001, 3001, ptr, col) is not None


def test_pattern_cap():
    """256 distinct one-entry rows are accepted, 257 are not."""
    ptr, col, val = diagonal(np.arange(1, 257) / 7.0)
    o = ab.pattern_value_plan(256, 256, ptr, col, val)
    assert o is not None and o["count"] == 256 and o["total"] == 256
    check(o, ptr, col, val)
    ptr, col, val = diagonal(np.arange(1, 258) / 7.0)
    assert ab.pattern_value_plan(257, 257, ptr, col, val) is None
    # the same 257 values repeated over many rows are still 257 patterns
    ptr, col, val = diagonal(np.tile(np.arange(1, 258) / 7.0, 20))
    assert ab.pattern_value_plan(val.size, val.size, ptr, col, val) is None


def rows_of(lens, seed):
    """Rows of the given lengths on the first diagonals, every entry a distinct value: each row
    its own pattern."""
    nr = len(lens)
    ptr = np.zeros(nr + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    rows = np.repeat(np.arange(nr, dtype=np.int64), lens)
    col = rows + (np.arange(ptr[-1]) - np.repeat(ptr[:-1], lens))
    val = np.random.default_rng(seed).uniform(1, 2, ptr[-1])
    return ptr, col, val, nr, int(col.max()) + 1


def test_entry_cap():
    """Patterns of 1024 entries in all are accepted, 1025 are not."""
    ptr, col, val, nr, nc = rows_of([4] * 256, 1)
    o = ab.pattern_value_plan(nr, nc, ptr, col, val)
    assert o is not None and o["count"] == 256 and o["total"] == 1024
    check(o, ptr, col, val)
    ptr, col, val, nr, nc = rows_of([4] * 255 + [5], 2)
    assert ab.pattern_value_plan(nr, nc, ptr, col, val) is None
    ptr, col, val, nr, nc = rows_of([1024], 3)
    o = ab.pattern_value_plan(nr, nc, ptr, col, val)
    assert o is not None and o["count"] == 1 and o["total"] == 1024
    ptr, col, val, nr, nc = rows_of([1025], 4)
    assert ab.pattern_value_plan(nr, nc, ptr, col, val) is None


def test_signed_zeros_and_nan_payloads_stay_distinct():
    qnan1 = np.array([0x7FF8000000000001], dtype=np.uint64).view(np.float64)[0]
    qnan2 = np.array([0x7FF8000000000002], dtype=np.uint64).view(np.float64)[0]
    vals = np.tile([0.0, -0.0, 1.0], 40)
    ptr, col, val = diagonal(vals)
    o = ab.pattern_value_plan(val.size, val.size, ptr, col, val)
    assert o is not None and o["count"] == 3 and o["exact_f32"]
    check(o, ptr, col, val)
    vals = np.tile([0.0, -0.0, qnan1, qnan2, np.nan, np.inf, -np.inf, 5e-324], 40)
    ptr, col, val = diagonal(vals)
    o = ab.pattern_value_plan(val.size, val.size, ptr, col, val)
    assert o is not None and o["count"] == 8
    assert not o["exact_f32"]                  # the payloads and the FP64 subnormal do not survive FP32
    check(o, ptr, col, val)


def test_empty_rows_and_rectangular_shapes():
    for nr, nc, offs, keep in ((2000, 2600, [0, 3, 4, 90, 300, 600], 0.4),
                               (2600, 2000, [-600, -3, 0, 5, 9], 1.0)):
        ptr, col, _ = diag_matrix(nr, nc, offs, seed=nr, keep=keep)
        assert (np.diff(ptr) == 0).any() == (keep == 0.4)
        # values that depend on the offset only: as many patterns as the offset plan
        val = (col - np.repeat(np.arange(nr), np.diff(ptr))) * 0.5 + 3.0
        o = ab.pattern_value_plan(nr, nc, ptr, col, val)
        p = ab.pattern_plan(nr, nc, ptr, col)
        assert o is not None and o["count"] == p["count"] and o["exact_f32"]
        check(o, ptr, col, val)
    # all rows empty: nothing to index
    assert ab.pattern_value_plan(5, 5, np.zeros(6, dtype=np.int64), np.zeros(0, dtype=np.int64),
                                 np.zeros(0)) is None
