"""CPU: the per-row error bounds of tests/_accuracy.py are tight enough to catch a subtly wrong
kernel.  A numpy model of the row reduction that follows the kernels' documented evaluation
order (per-lane fma sums, xor butterfly, the long path's warp partials; csr_kernels.cuh) must
pass assert_rows on the generators the GPU tests use, and each mutant -- a row reduction that
is wrong in one small way -- must be rejected, at the row it broke."""
import math

import numpy as np
import pytest

import _accuracy as acc

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


@pytest.fixture(autouse=True)
def _extended():
    acc.require_longdouble()


def _fma(a, b, s, ty):
    """fl_ty(a*b + s): the product and sum are formed in longdouble (error 2^-64 relative), so
    the model rounds once in ty, as the hardware fma does (to within the reference slack)."""
    return (a.astype(acc.LD) * b.astype(acc.LD) + s.astype(acc.LD)).astype(ty)


def _butterfly(v, ty):
    n = v.size
    idx = np.arange(n)
    o = n // 2
    while o:
        v = (v + v[idx ^ o]).astype(ty)
        o //= 2
    return v[0]


def model_row_sums(ptr, col, val, x, p, ty=np.float64):
    """Row sums in the order the kernels evaluate them (module docstring of _accuracy)."""
    nr = ptr.size - 1
    out = np.zeros(nr, dtype=ty)
    L = p["lanes"]
    lrow = p["long"][acc.block_of(p, np.arange(nr))]
    v = val.astype(ty)
    xs = x.astype(ty)
    for r in range(nr):
        b, e = int(ptr[r]), int(ptr[r + 1])
        if b == e:
            continue
        W = 256 if lrow[r] else L
        k = e - b
        steps = -(-k // W)
        a = np.zeros(steps * W, dtype=ty)
        g = np.zeros(steps * W, dtype=ty)
        a[:k] = v[b:e]
        g[:k] = xs[col[b:e]]
        a, g = a.reshape(steps, W), g.reshape(steps, W)
        s = np.zeros(W, dtype=ty)
        for t in range(steps):
            s = _fma(a[t], g[t], s, ty)
        if lrow[r]:
            warps = [_butterfly(s[w * 32:(w + 1) * 32], ty) for w in range(8)]
            tot = ty(0)
            for w in warps:
                tot = ty(tot + w)
            out[r] = tot
        else:
            out[r] = _butterfly(s, ty)
    return out


def _case(name):
    if name == "ragged_long":
        ptr, col, val, x = acc.ragged_csr(4097, 3001, nnz_cap=512, seed=5)
        return ptr, col, val, x, 4, 512
    if name == "ragged_staged":
        ptr, col, val, x = acc.ragged_csr(3803, 4400, nnz_cap=2048, seed=6, long_blocks=False)
        return ptr, col, val, x, 1, 2048
    if name == "ragged_wide":
        ptr, col, val, x = acc.ragged_csr(3802, 3000, nnz_cap=2048, seed=7)
        return ptr, col, val, x, 32, 2048
    ptr, col, val, x = acc.band_csr(3001, 3200, [-40, -3, -1, 0, 1, 3, 40, 150], seed=8)
    return ptr, col, val, x, 2, 2048


CASES = ["ragged_long", "ragged_staged", "ragged_wide", "band"]


def _check(ptr, col, val, x, got, p, what):
    S, M = acc.row_sums(ptr, col, val, x)
    m, k = acc.roundings(ptr, p)
    acc.assert_rows(got, S, acc.bound("spmv", m, k, acc.U64, M), what, ptr, p)


def test_generator_covers_its_edge_catalogue():
    for nr, nc in ((4097, 3001), (4098, 5000), (4099, 4099)):
        for cap in (256, 2048, 6144):
            ptr, col, val, x = acc.ragged_csr(nr, nc, nnz_cap=cap, seed=nr + cap)
            p = acc.plan(ptr, 0, cap)
            lens = np.diff(ptr)
            assert lens[0] == 0 and lens[-1] == 0 and (lens == cap).any()
            assert p["long"][0] and (p["long"][-1] or p["long"][-2])
            assert set(p["estarts"] % 4) == {0, 1, 2, 3}
            empty_blocks = np.flatnonzero(np.diff(np.append(p["estarts"], ptr[-1])) == 0)
            assert empty_blocks.size > 0                      # a whole block of empty rows
            assert (col == 0).any() and (col == nc - 1).any()
            S, M = acc.row_sums(ptr, col, val, x)
            assert ((np.abs(S) < 1e-8 * M) & (M > 0)).any()   # cancelling rows
            quad = np.add.reduceat(lens, np.arange(0, nr, 4))
            assert (quad == cap + 1).sum() >= 2


@pytest.mark.parametrize("case", CASES)
def test_model_of_the_documented_order_passes(case):
    ptr, col, val, x, lanes, cap = _case(case)
    p = acc.plan(ptr, lanes, cap)
    _check(ptr, col, val, x, model_row_sums(ptr, col, val, x, p), p, case)


def test_model_passes_in_fp32():
    ptr, col, val, x, lanes, cap = _case("ragged_long")
    p = acc.plan(ptr, lanes, cap)
    v32, x32 = val.astype(np.float32), x.astype(np.float32)
    got = model_row_sums(ptr, col, v32, x32, p, np.float32)
    S, M = acc.row_sums(ptr, col, v32, x32)
    m, k = acc.roundings(ptr, p)
    acc.assert_rows(got, S, acc.bound("spmv", m, k, acc.U32, M), "fp32", ptr, p)


def _target_row(ptr, col, val, x, min_len=3):
    """A row whose every entry matters: at least min_len entries, no cancellation."""
    S, M = acc.row_sums(ptr, col, val, x)
    lens = np.diff(ptr)
    ok = np.flatnonzero((lens >= min_len) & (np.abs(S) > 0.5 * M))
    return int(ok[len(ok) // 2])


def _expect_reject(fn, row):
    with pytest.raises(AssertionError) as e:
        fn()
    assert ("row %d " % row) in str(e.value), str(e.value)


@pytest.mark.parametrize("case", CASES)
def test_rejects_a_dropped_last_entry(case):
    ptr, col, val, x, lanes, cap = _case(case)
    p = acc.plan(ptr, lanes, cap)
    r = _target_row(ptr, col, val, x)
    bad = val.copy()
    bad[ptr[r + 1] - 1] = 0.0                      # the model never sees the row's last entry
    got = model_row_sums(ptr, col, bad, x, p)
    _expect_reject(lambda: _check(ptr, col, val, x, got, p, "dropped"), r)


@pytest.mark.parametrize("case", CASES)
def test_rejects_an_entry_counted_twice(case):
    ptr, col, val, x, lanes, cap = _case(case)
    p = acc.plan(ptr, lanes, cap)
    r = _target_row(ptr, col, val, x)
    bad = val.copy()
    bad[ptr[r]] *= 2.0
    got = model_row_sums(ptr, col, bad, x, p)
    _expect_reject(lambda: _check(ptr, col, val, x, got, p, "twice"), r)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("shift", [-1, 1])
def test_rejects_a_gather_from_the_next_column(case, shift):
    ptr, col, val, x, lanes, cap = _case(case)
    p = acc.plan(ptr, lanes, cap)
    r = _target_row(ptr, col, val, x)
    bad = col.copy()
    e = int(np.argmax(np.abs(val[ptr[r]:ptr[r + 1]] * x[col[ptr[r]:ptr[r + 1]]]))) + int(ptr[r])
    bad[e] = col[e] + shift if 0 <= col[e] + shift < x.size else col[e] - shift
    got = model_row_sums(ptr, bad, val, x, p)
    _expect_reject(lambda: _check(ptr, col, val, x, got, p, "column"), r)


@pytest.mark.parametrize("case", CASES)
def test_rejects_rows_swapped_at_a_block_boundary(case):
    ptr, col, val, x, lanes, cap = _case(case)
    p = acc.plan(ptr, lanes, cap)
    got = model_row_sums(ptr, col, val, x, p)
    S, M = acc.row_sums(ptr, col, val, x)
    # the first block boundary whose two rows differ by far more than their bounds
    for b in range(1, p["nblocks"]):
        r = int(p["starts"][b])
        if abs(float(S[r] - S[r - 1])) > 1e-6 * float(M[r] + M[r - 1]) > 0:
            break
    bad = got.copy()
    bad[[r - 1, r]] = bad[[r, r - 1]]
    with pytest.raises(AssertionError) as e:
        _check(ptr, col, val, x, bad, p, "swap")
    msg = str(e.value)
    assert ("row %d " % r) in msg or ("row %d " % (r - 1)) in msg, msg


def _ctas_scalar(y, w, grid):
    """In-kernel scalar in the kernels' order: per-CTA partials (rows strided over CTAs), then
    the finishing CTA adds them; returns the per-CTA partials too."""
    prods = y * w
    parts = np.array([math.fsum(prods[c::grid]) for c in range(grid)])
    return parts


def test_rejects_a_scalar_missing_one_cta():
    rng = np.random.default_rng(3)
    n, grid = 200000, 528
    y, w = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    S, A = acc.dot_ref(y, w)
    parts = _ctas_scalar(y, w, grid)
    nb = -(-n // 256)
    bnd = acc.csr_scalar_bound(A, nb, 256, 1, 132, 4)
    acc.assert_scalar(float(parts.sum()), S, bnd, "all CTAs")
    acc.assert_scalar(float(parts.sum()), S, acc.kahan_bound(A, grid), "all CTAs (compensated)")
    for c in (0, grid // 2, grid - 1):
        with pytest.raises(AssertionError):
            acc.assert_scalar(float(parts.sum() - parts[c]), S, bnd, "CTA %d missing" % c)


def test_exact_rows_need_no_bound():
    """Rows of 0 or 1 entries and the x = 0 sweep are exact: the checks there are equalities."""
    rng = np.random.default_rng(4)
    d, f = rng.uniform(0.1, 1, 1000), rng.uniform(-1, 1, 1000)
    omega = 0.72
    want = (omega * d) * f
    ld = (acc.LD(omega) * d.astype(acc.LD)).astype(np.float64).astype(acc.LD) * f.astype(acc.LD)
    assert np.array_equal(want, ld.astype(np.float64))
