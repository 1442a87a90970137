"""Host-side plan of the narrow column format and of the block-relative row pointers
(narrow.cuh, exported as b200_narrow_plan_i64): every column must come back as
base[block] + lo16 (+ hi8 << 16), every row pointer as e0(block) + ptr16, and the width must be
the narrowest that holds every block's column span."""
import numpy as np
import pytest

import _accuracy as acc
import amgcl_b200 as ab
import oracle


def blocks(ptr, p):
    """(first row, end row) of every block of plan p."""
    ends = list(p["starts"][1:]) + [ptr.size - 1]
    return list(zip((int(r) for r in p["starts"]), (int(r) for r in ends)))


def rebuild_cols(ptr, p, o):
    """Columns from the plan, block by block (the blocks are acc.plan's, in row order)."""
    out = np.empty(int(ptr[-1]), dtype=np.int64)
    hi = o.get("hi8")
    for b, (r0, r1) in enumerate(blocks(ptr, p)):
        e0, e1 = int(ptr[r0]), int(ptr[r1])
        rel = o["lo16"][e0:e1].astype(np.int64)
        if hi is not None:
            rel |= hi[e0:e1].astype(np.int64) << 16
        out[e0:e1] = o["base"][b] + rel
    return out


def check_roundtrip(ptr, col, ncols, lanes=0, cap=2048):
    nr = ptr.size - 1
    o = ab.narrow_plan(nr, ncols, ptr, col, lanes=lanes, nnz_cap=cap)
    p = acc.plan(ptr, lanes, cap)
    assert o["nblocks"] == p["nblocks"]
    # row pointers: e0 of the row's block + ptr16, for every row of every staged block
    for r0, r1 in blocks(ptr, p):
        e0 = int(ptr[r0])
        if int(ptr[r1]) - e0 <= cap:
            np.testing.assert_array_equal(o["ptr16"][r0:r1].astype(np.int64) + e0, ptr[r0:r1])
    if o["width"]:
        np.testing.assert_array_equal(rebuild_cols(ptr, p, o), col)
    return o, p


def span_matrix(span, nr=4000, seed=0):
    """A matrix whose widest row block spans exactly `span` columns (one row holds column 0
    and column `span`), every other block much less."""
    ptr, col, _, _ = acc.band_csr(nr, nr, [-3, 0, 3], seed=seed, keep=1.0)
    rows = np.repeat(np.arange(nr), np.diff(ptr))
    r = nr // 2 & ~3                                    # first row of some block
    extra = np.array([[r, 0], [r, span]], dtype=np.int64)
    rows = np.concatenate([rows, extra[:, 0]])
    cols = np.concatenate([col, extra[:, 1]])
    key = np.unique(rows * (span + nr + 1) + cols)
    rows, cols = key // (span + nr + 1), key % (span + nr + 1)
    ptr = np.zeros(nr + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=nr), out=ptr[1:])
    return ptr, cols, max(nr, span + 1)


@pytest.mark.parametrize("span,width", [(65535, 16), (65536, 24), ((1 << 24) - 1, 24), (1 << 24, 0)])
def test_width_at_the_span_limits(span, width):
    ptr, col, nc = span_matrix(span, seed=span & 0xff)
    o, p = check_roundtrip(ptr, col, nc)
    assert o["width"] == width
    if width:
        spans = [int(col[ptr[a]:ptr[b]].max() - col[ptr[a]:ptr[b]].min()) for a, b in blocks(ptr, p) if ptr[b] > ptr[a]]
        assert max(spans) == span
        assert o["base"][[i for i, (a, b) in enumerate(blocks(ptr, p)) if ptr[b] > ptr[a]]].min() >= 0


def test_ragged_matrices_roundtrip():
    """The edge catalogue of the accuracy generator (empty-row runs, exact-cap quads, duplicate
    and extreme columns); with long blocks the columns stay plain but the row pointers of every
    staged block still round-trip."""
    for seed, long_blocks in ((0, True), (1, False), (2, False)):
        nr, nc = 20001 + seed, 19000 + 37 * seed
        ptr, col = acc.ragged_csr(nr, nc, seed=seed, long_blocks=long_blocks)[:2]
        for lanes in (0, 1, 2, 8):
            o, p = check_roundtrip(ptr, col, nc, lanes=lanes)
            if long_blocks and p["long"].any():
                assert o["width"] == 0
            elif p["lanes"] <= 8:
                assert o["width"] in (16, 24)


def test_operators_with_more_than_8_lanes_stay_plain():
    ptr, col, _, _ = acc.band_csr(3000, 3000, list(range(-200, 200)), seed=4, keep=1.0)
    o, p = check_roundtrip(ptr, col, 3000, cap=6144)
    assert p["lanes"] > 8 and o["width"] == 0


def test_empty_blocks_single_columns_and_empty_matrix():
    nr = 64
    ptr = np.zeros(nr + 1, dtype=np.int64)              # no entries at all
    o = ab.narrow_plan(nr, 10, ptr, np.zeros(0, dtype=np.int64))
    assert o["width"] == 0 and not o["ptr16"].any()
    ptr = np.arange(nr + 1, dtype=np.int64) * (np.arange(nr + 1) > 32)   # rows 0..31 empty
    ptr[33:] = np.arange(1, nr - 31)
    col = np.full(int(ptr[-1]), 12345, dtype=np.int64)  # one column everywhere
    o, _ = check_roundtrip(ptr, col, 20000)
    assert o["width"] == 16 and not o["lo16"].any()


def test_halo_renumbered_columns():
    """A partitioned operator's local part: columns >= n_loc are halo slots n_loc + o * S + slot
    (dist.cuh), far from the local ones; the span rule sees them like any column."""
    n_loc, S, nranks = 5000, 700, 4
    rng = np.random.default_rng(5)
    ptr, col, _, _ = acc.band_csr(n_loc, n_loc, [-1, 0, 1], seed=5, keep=1.0)
    rows = np.repeat(np.arange(n_loc), np.diff(ptr))
    halo_rows = np.arange(0, n_loc, 97)
    halo_cols = n_loc + rng.integers(0, nranks, halo_rows.size) * S + rng.integers(0, S, halo_rows.size)
    rows = np.concatenate([rows, halo_rows])
    cols = np.concatenate([col, halo_cols])
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    ptr = np.zeros(n_loc + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n_loc), out=ptr[1:])
    o, _ = check_roundtrip(ptr, cols, n_loc + nranks * S)
    assert o["width"] == 16


@pytest.mark.skipif(not oracle.have_ref(), reason="reference build (oracle/_ref) not available")
def test_hierarchy_widths_at_64():
    """Every operator of the reference hierarchy at 64^3 gets the width its widest block span
    asks for; the finest-level prolongation P0 is 16-bit."""
    ptr, col, val, _ = ab.poisson3d(64)
    S = oracle.RefSolver(ptr, col, val, "damped_jacobi", "cg")
    seen = {}
    for lvl in range(S.nlevels - 1):
        for w in "APR":
            if lvl == 0 and w == "A":
                continue                                  # (pattern-indexed)
            nr, nc, (p, c, _) = S.level_matrix(lvl, w)
            o, pl = check_roundtrip(p.astype(np.int64), c.astype(np.int64), nc)
            spans = [int(c[p[a]:p[b]].max() - c[p[a]:p[b]].min()) for a, b in blocks(p, pl) if p[b] > p[a]]
            want = 0 if pl["lanes"] > 8 or pl["long"].any() else 16 if max(spans) <= 0xffff else 24
            assert o["width"] == want, (lvl, w, max(spans), pl["lanes"])
            seen[(lvl, w)] = o["width"]
    assert seen[(0, "P")] == 16
