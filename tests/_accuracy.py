"""Extended-precision references and per-row forward-error bounds for the solve-phase kernels.

Reference
---------
Every reference value is formed in ``np.longdouble`` (64-bit mantissa on x86-64, unit roundoff
u_ld = 2^-64) from the operands AS THE KERNEL READS THEM: FP32 matrices and vectors are rounded
to FP32 first, and a gathered x entry is converted to the row sum's type (``(TS)xv`` in
csr_kernels.cuh, TS = the output type TY), so the check measures the kernel's arithmetic and not
the rounding of its inputs.  All conversions to longdouble are exact.

    S_r = sum_e a_e * x_c        M_r = sum_e |a_e * x_c|        (e over the entries of row r)

Both are formed with ``np.add.reduceat`` over the products; empty rows are 0.

Bounds
------
u is the unit roundoff of the accumulation type TY (2^-53 FP64, 2^-24 FP32) and
gamma(m) = m*u / (1 - m*u) (Higham, "Accuracy and Stability of Numerical Algorithms", 3.1).
A sum evaluated with m roundings along every path from an operand to the result satisfies
|fl(S) - S| <= gamma(m) * M.

* A staged row of k entries reduced by L lanes: every lane accumulates its ceil(k/L) entries
  with one fma each (one rounding per entry, the first is a plain product), then the xor
  butterfly adds log2(L) times:  m = ceil(k/L) + log2 L.
* A row of a long block (compute_long): 256 threads accumulate ceil(k/256) entries each, a
  32-lane butterfly adds 5 times, thread 0 adds the 8 warp partials in order:
  m = ceil(k/256) + 5 + 8.
* Epilogues (store_row / tail_csr), each one more rounding per operation:
    SPMV         alpha*S                    gamma(m+1) * |alpha| * M
    SPMV, beta   alpha*S + beta*y0          gamma(m+2) * (|alpha| * M + |beta * y0|)
    RESID        f - S                      gamma(m+1) * (M + |f|)
    RELAX        fma(fl(omega*d), f - S, x0) gamma(m+3) * (|x0| + |omega*d| * (|f| + M))
* The longdouble reference itself carries at most gamma_ld(k + 4) times the same scale; that
  term is added to every bound (it is below 2^-11 of the FP64 term for the rows used here).

Exact checks.  relax_zero_kernel and the x written by MODE_RESID_SCALED compute
fma(TX(omega*d), TX(f), 0), which is the correctly rounded product (omega*d)*f in TX: numpy
gives the same bits.  A row of at most one entry is exact up to the epilogue: alpha*fl(a*x) and
f - fl(a*x) in FP64.

Scalars.  The reference of an in-kernel inner product is taken over the vectors the GPU
produced (q is downloaded, then <q^, p> is formed), so the row error of the spmv and the error
of the reduction are checked separately.  Let D be the depth of the uncompensated combine tree
of red_finish / dot_kernel: butterfly (5) + 8 warp partials + ceil(G/256) CTA partials per
thread of the finishing CTA + butterfly (5) + 8 warp partials, G the grid.
* Kahan-compensated vector kernels (dot_kernel, fused_vec_kernel): each thread's compensated
  sum S_t is within 2u|S_t| (+ O(n_t u^2) sum|p|) of its exact sum of the ROUNDED products, a
  product is rounded once (u |x y|), and sum_t |S_t| <= sum |x y|, so
  |s^ - s| <= gamma(D + 3) * sum |x_i y_i|.
  (2u|S_t| sums to 2u * sum_t |S_t|, not to 2u * |S|: per-thread sums may cancel.)
* CSR in-kernel scalars are not compensated: the thread that stores a row adds y_r * w_r with
  one fma.  It stores at most R = ceil(nblocks / grid) * max(4, ceil(rows_cap / (256 / L))) rows
  (a long block is one quad, all of whose rows thread 0 stores), grid =
  min(nblocks, SMs * ctas_per_sm), so |s^ - s| <= gamma(R + D) * sum |y_r w_r|.
"""
import math

import numpy as np
import pytest

LD = np.longdouble
U64 = 2.0 ** -53
U32 = 2.0 ** -24
ULD = 2.0 ** -64


def require_longdouble():
    if np.finfo(LD).nmant < 63:
        pytest.skip("np.longdouble has a %d-bit mantissa here; the references need >= 63 (x86-64 "
                    "extended precision)" % np.finfo(LD).nmant)


def unit(dtype):
    """Unit roundoff of the accumulation (= output) type."""
    return U32 if np.dtype(dtype) == np.float32 else U64


def gamma(m, u):
    m = np.asarray(m, dtype=np.float64)
    return m * u / (1.0 - m * u)


def row_sums(ptr, col, val, x):
    """(S, M) in longdouble: S_r = sum a_e x_c, M_r = sum |a_e x_c| over the entries of row r.
    val and x must already be the values the kernel multiplies (rounded as stored)."""
    ptr = np.asarray(ptr, dtype=np.int64)
    nr = ptr.size - 1
    S = np.zeros(nr, dtype=LD)
    M = np.zeros(nr, dtype=LD)
    if ptr[-1] == 0:
        return S, M
    prod = np.asarray(val).astype(LD) * np.asarray(x).astype(LD)[np.asarray(col, dtype=np.int64)]
    nonempty = np.flatnonzero(np.diff(ptr) > 0)
    # consecutive non-empty row starts bound exactly one row's entries (empty rows have none)
    starts = ptr[nonempty]
    S[nonempty] = np.add.reduceat(prod, starts)
    M[nonempty] = np.add.reduceat(np.abs(prod), starts)
    return S, M


def plan(ptr, lanes, nnz_cap):
    """The row-block plan b200_csr_create builds (b200_plan_i64): lanes, rows_cap, block row
    starts, block non-zero starts, and which blocks are long (> nnz_cap non-zeros)."""
    import ctypes
    import amgcl_b200 as ab
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    nr = ptr.size - 1
    L = ab.lib()
    nb, lo, rc, nl = ctypes.c_int64(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int64()
    assert L.b200_plan_i64(nr, ptr.ctypes.data, lanes, nnz_cap, None, 0, ctypes.byref(nb),
                           ctypes.byref(lo), ctypes.byref(rc), ctypes.byref(nl)) == 0, L.b200_last_error()
    blk = np.zeros((nb.value + 1, 2), dtype=np.int32)
    assert L.b200_plan_i64(nr, ptr.ctypes.data, lanes, nnz_cap, blk.ctypes.data, blk.shape[0],
                           ctypes.byref(nb), ctypes.byref(lo), ctypes.byref(rc), ctypes.byref(nl)) == 0
    rows, nzs = blk[:, 0].astype(np.int64), blk[:, 1].astype(np.int64)
    long_blk = np.diff(nzs) > nnz_cap
    assert int(long_blk.sum()) == nl.value
    return {"lanes": lo.value, "rows_cap": rc.value, "starts": rows[:-1], "estarts": nzs[:-1],
            "long": long_blk, "nblocks": nb.value, "nnz_cap": nnz_cap}


def block_of(p, rows):
    """Block index of every row in `rows` under plan p."""
    return np.searchsorted(p["starts"], rows, side="right") - 1


def roundings(ptr, p, lanes=None):
    """m of every row (module docstring): per-lane entries + butterfly, or the long-path tree."""
    k = np.diff(np.asarray(ptr, dtype=np.int64))
    L = lanes or p["lanes"]
    m = np.ceil(k / L) + math.log2(L)
    if p["long"].any():
        lrow = p["long"][block_of(p, np.arange(k.size))]
        m[lrow] = np.ceil(k[lrow] / 256.0) + 5 + 8
    return m, k


def bound(mode, m, k, u, M, alpha=1.0, beta=0.0, y0=None, f=None, x0=None, omega=None, d=None):
    """Per-row forward-error bound of one CSR pass (module docstring)."""
    M = np.asarray(M, dtype=np.float64)
    if mode == "spmv":
        c, scale = 1, abs(alpha) * M
    elif mode == "spmv_acc":
        c, scale = 2, abs(alpha) * M + np.abs(beta * np.asarray(y0, dtype=np.float64))
    elif mode == "resid":
        c, scale = 1, M + np.abs(np.asarray(f, dtype=np.float64))
    elif mode == "relax":
        wd = np.abs(omega * np.asarray(d, dtype=np.float64))
        c, scale = 3, np.abs(np.asarray(x0, dtype=np.float64)) + wd * (np.abs(np.asarray(f, dtype=np.float64)) + M)
    else:
        raise ValueError(mode)
    return (gamma(m + c, u) + gamma(k + 4, ULD)) * scale


def reference(mode, S, alpha=1.0, beta=0.0, y0=None, f=None, x0=None, omega=None, d=None):
    """Exact (longdouble) value of one CSR pass from the row sums S."""
    if mode == "spmv":
        return LD(alpha) * S
    if mode == "spmv_acc":
        return LD(alpha) * S + LD(beta) * np.asarray(y0).astype(LD)
    if mode == "resid":
        return np.asarray(f).astype(LD) - S
    if mode == "relax":
        return np.asarray(x0).astype(LD) + LD(omega) * np.asarray(d).astype(LD) * (np.asarray(f).astype(LD) - S)
    raise ValueError(mode)


def assert_rows(got, want, bnd, what, ptr=None, p=None):
    """Every row within its bound; on failure the message names the worst row (error / bound,
    its length, its block in the plan p)."""
    got = np.asarray(got)
    err = np.abs(got.astype(LD) - np.asarray(want, dtype=LD)).astype(np.float64)
    bnd = np.asarray(bnd, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / bnd)
    ratio[~np.isfinite(got.astype(np.float64))] = np.inf
    ratio[np.isnan(ratio)] = np.inf
    if ratio.size == 0 or ratio.max() <= 1.0:
        return
    r = int(np.argmax(ratio))
    where = ""
    if ptr is not None:
        where += ", row length %d" % int(ptr[r + 1] - ptr[r])
    if p is not None:
        b = int(block_of(p, np.array([r]))[0])
        where += ", block %d of %d (rows %d.., %s)" % (b, p["nblocks"], int(p["starts"][b]),
                                                      "long" if p["long"][b] else "staged")
    raise AssertionError("%s: row %d off by %.3g = %.3g x its bound %.3g (got %r, want %r)%s; %d rows "
                         "over their bound" % (what, r, err[r], ratio[r], bnd[r], float(got[r]),
                                               float(np.asarray(want, dtype=LD)[r]), where,
                                               int((ratio > 1.0).sum())))


def red_depth(grid):
    """D: uncompensated combine tree of red_finish / dot_kernel over `grid` CTAs."""
    return 5 + 8 + int(math.ceil(grid / 256.0)) + 5 + 8


def kahan_bound(prod_abs_sum, grid):
    return float(gamma(red_depth(grid) + 3, U64)) * float(prod_abs_sum)


def csr_scalar_bound(prod_abs_sum, nblocks, rows_cap, lanes, sms, ctas_per_sm):
    grid = max(1, min(nblocks, sms * ctas_per_sm))
    R = int(math.ceil(nblocks / grid)) * max(4, int(math.ceil(rows_cap / (256 // lanes))))
    return float(gamma(R + red_depth(grid), U64)) * float(prod_abs_sum)


def assert_scalar(got, want, bnd, what):
    err = abs(LD(got) - LD(want))
    assert np.isfinite(got) and err <= LD(bnd), \
        "%s: got %r, want %r, off by %.3g = %.3g x its bound %.3g" % (
            what, got, float(want), float(err), float(err) / max(bnd, 1e-300), bnd)


def dot_ref(x, y):
    """(sum x*y, sum |x*y|) in longdouble."""
    p = np.asarray(x).astype(LD) * np.asarray(y).astype(LD)
    return p.sum(), np.abs(p).sum()


# ---------------------------------------------------------------------------------------------
# generators
# ---------------------------------------------------------------------------------------------
def ragged_csr(nr, nc, nnz_cap=2048, seed=0, long_blocks=True):
    """A ragged CSR operator with the edges the row-block kernels have to survive:

    * empty rows first and last, and a run of empty rows longer than any block (rows_cap <= 1024);
    * a row of exactly nnz_cap entries (its quad fills a stage exactly);
    * long_blocks: a quad of nnz_cap + 1 entries (barely long) first and at the end, a row of
      more than 3*256 entries, and a long quad that also holds short rows;
    * random row lengths, so block starts e0 fall on every residue mod 4 (bulk-copy alignment);
    * duplicate columns within a row, columns 0 and nc - 1;
    * values whose magnitudes spread over 2^-20 .. 2^20;
    * rows built to cancel: pairs a*x_c - a*x_c on a duplicated column plus one tiny entry, so
      S ~ 2^-30 while M ~ 1.
    Returns (ptr, col, val, x) with x a matching random vector of length nc."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 24, nr)
    lens[:2] = 0                                    # empty rows first
    lens[-1] = 0                                    # ... and last
    assert nr > 3400, "the edge catalogue needs room"
    run0 = 4 * (nr // 6 // 4)
    lens[run0:run0 + 1100] = 0                      # an all-empty stretch longer than a block
    q = 4 * (nr // 12 // 4)
    lens[q:q + 4] = [nnz_cap, 0, 0, 0]              # exactly one stage
    if long_blocks:
        lens[2:4] = [nnz_cap + 1 - 7, 7]            # first quad: nnz_cap + 1 (barely long)
        tail = nr - 5 if nr % 4 == 1 else nr - (nr % 4 or 4)
        lens[tail:tail + 4] = 0
        lens[tail] = nnz_cap + 1                    # a barely long quad at the end
        q = 4 * (nr // 2 // 4)
        lens[q:q + 4] = [5, max(nnz_cap, 3 * 256) + 9, 3, 0]   # long quad with short rows
        lens[-1] = 0
    else:
        q = 4 * (nr // 2 // 4)
        lens[q:q + 4] = [0, 3 * 256 + 9, 2, 0]      # a row of more than 3*256 entries, staged
        # every aligned quad must fit a stage
        for s in range(0, nr, 4):
            while lens[s:s + 4].sum() > nnz_cap:
                lens[s + int(np.argmax(lens[s:s + 4]))] -= 1
    ptr = np.zeros(nr + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    nnz = int(ptr[-1])
    col = rng.integers(0, nc, nnz)
    mag = np.exp2(rng.uniform(-20, 20, nnz))
    val = rng.choice([-1.0, 1.0], nnz) * rng.uniform(0.5, 1.0, nnz) * mag
    # duplicate columns and the two extreme columns
    multi = np.flatnonzero(lens >= 3)
    for r in multi[::7]:
        col[ptr[r] + 1] = col[ptr[r]]
    for r in multi[1::11]:
        col[ptr[r]] = 0
        col[ptr[r + 1] - 1] = nc - 1
    # cancelling rows: (a, c), (-a, c) pairs + one tiny entry
    for r in multi[3::13]:
        b, e = int(ptr[r]), int(ptr[r + 1])
        k = (e - b - 1) // 2 * 2
        if k < 2:
            continue
        a = rng.uniform(0.5, 1.0, k // 2)
        c = rng.integers(0, nc, k // 2)
        val[b:b + k:2], val[b + 1:b + k:2] = a, -a
        col[b:b + k:2], col[b + 1:b + k:2] = c, c
        val[b + k:e] = 2.0 ** -30
    x = rng.uniform(-1, 1, nc) * np.exp2(rng.uniform(-2, 2, nc))
    return ptr, col, val, x


def band_csr(nr, nc, offsets, seed, keep=0.9):
    """A structured band (few distinct col - row, few row patterns): what the compressed column
    formats store.  Ragged (entries dropped with probability 1 - keep)."""
    from test_offsets import diag_matrix
    ptr, col, val = diag_matrix(nr, nc, offsets, seed, keep=keep)
    rng = np.random.default_rng(seed + 1)
    val = val * np.exp2(rng.uniform(-20, 20, val.size))
    x = rng.uniform(-1, 1, nc)
    return ptr, col, val, x
