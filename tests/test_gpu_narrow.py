"""GPU parity of the narrow column formats (csr_kernels.cuh FMT_COL16 / FMT_COL24, narrow.cuh)
and of the block-relative row pointers every staged format streams: an operator streamed with
16- or 24-bit block-relative columns must give the bits of the same operator with plain int32
columns -- only where the column number comes from changes -- in every mode, on 1..8 lanes,
in every precision mix, in the fused Krylov step and in whole solves; and within the per-row
error bounds of tests/_accuracy.py on the ring-knob cases."""
import numpy as np
import pytest

import amgcl_b200 as ab
from test_gpu_accuracy import KNOBS, Case, options, sized, walks_the_ring
from test_gpu_primitives import _f32csr, _f32vec

pytestmark = pytest.mark.gpu

WIDTHS = [16, 24]


def narrow_csr(nr, nc, lanes, width, seed):
    """Random rows of about 6 * lanes entries; width 16: every row within 2000 columns of the
    diagonal, width 24: each row also reaches about 100 000 columns away (kept < nc)."""
    rng = np.random.default_rng(seed)
    per = 6 * lanes
    lens = rng.integers(0, 2 * per, nr)
    lens[rng.uniform(size=nr) < 0.05] = 0                 # empty rows
    ptr = np.zeros(nr + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    rows = np.repeat(np.arange(nr), lens)
    near = rows * nc // nr + rng.integers(-2000, 2000, rows.size)
    col = near if width == 16 else np.where(rng.uniform(size=rows.size) < 0.3, near + 100000, near)
    col = np.clip(col, 0, nc - 1)[np.lexsort((col, rows))]      # sorted within each row
    val = rng.uniform(-1, 1, col.size)
    return ptr, col.astype(np.int64), val


def both(ctx, fn):
    """fn() with narrow columns, then with plain columns (the same uploaded operator)."""
    ctx.set_option("narrow_columns", 1)
    a = fn()
    ctx.set_option("narrow_columns", 0)
    try:
        b = fn()
    finally:
        ctx.set_option("narrow_columns", 1)
    return a, b


@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_narrow_columns_give_the_bits_of_plain_columns(ctx, lanes, width):
    nr, nc = 30001, 230000
    ptr, col, val = narrow_csr(nr, nc, lanes, width, seed=lanes + width)
    with options(ctx, lanes=lanes, spmv_variant=1):
        A = ctx.csr(nr, nc, ptr, col, val)
        assert A.plan()["lanes"] == lanes and A.narrow() == width
        rng = np.random.default_rng(1)
        x, y, f = rng.uniform(-1, 1, nc), rng.uniform(-1, 1, nr), rng.uniform(-1, 1, nr)
        vx, vf = ctx.vector(x), ctx.vector(f)

        def spmv(beta):
            vy = ctx.vector(y)
            ctx.spmv(1.5, A, vx, beta, vy)
            return vy.numpy()
        for beta in (0.0, -0.25):
            a, b = both(ctx, lambda: spmv(beta))
            np.testing.assert_array_equal(a, b)

        def resid():
            vr = ctx.vector(nr)
            ctx.residual(vf, A, vx, vr)
            return vr.numpy()
        a, b = both(ctx, resid)
        np.testing.assert_array_equal(a, b)


def square(ptr, col, val, n):
    """The operator folded onto n columns (col mod n, re-sorted): a square one for the sweeps."""
    rows = np.repeat(np.arange(ptr.size - 1), np.diff(ptr))
    c = col % n
    o = np.lexsort((c, rows))
    return ptr, c[o], val[o]


@pytest.mark.parametrize("width", WIDTHS)
def test_sweeps_fused_first_sweep_and_cg_step(ctx, width):
    n = 120000
    ptr, col, val = square(*narrow_csr(n, n, 1, width, seed=7 + width), n)
    A = ctx.csr(n, n, ptr, col, val)
    assert A.narrow() == width
    rng = np.random.default_rng(3)
    x, f, d = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.1, 1.0, n)
    vf, vd = ctx.vector(f), ctx.vector(d)

    def sweep(zero):
        vxx, vt = ctx.vector(x), ctx.vector(n)
        if zero:
            ctx.clear(vxx)
        ctx.relax(A, vf, vxx, vt, vd, 0.72)
        vr = ctx.vector(n)
        ctx.residual(vf, A, vxx, vr)
        return np.concatenate([vxx.numpy(), vr.numpy()])
    for zero in (False, True):
        a, b = both(ctx, lambda: sweep(zero))
        np.testing.assert_array_equal(a, b)

    # the streaming pass that also leaves scalars behind (CG: q = A p with <q, p>)
    def step():
        K = ab.Krylov(ctx, n)
        vp, vq, vxx, vr = ctx.vector(x), ctx.vector(n), ctx.vector(d), ctx.vector(f)
        K.cg_direction(vf, vf, vp)
        K.cg_step(A, vp, vq, vxx, vr)
        s = K.scalars()
        K.close()
        return np.concatenate([vq.numpy(), vxx.numpy(), vr.numpy(), [s["qp"], s["alpha"], s["rr"]]])
    a, b = both(ctx, step)
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("width", WIDTHS)
def test_mixed_precision_combinations(ctx, width):
    n = 100000
    ptr, col, val = square(*narrow_csr(n, n, 2, width, seed=11 + width), n)
    A32 = _f32csr(ctx, n, n, ptr, col, val)
    assert A32.narrow() == width
    rng = np.random.default_rng(2)
    x, f, y = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    d = rng.uniform(0.1, 1.0, n).astype(np.float32)

    def run():
        out = []
        vx, vf = ctx.vector(x), ctx.vector(f)
        fx, ff = _f32vec(ctx, x), _f32vec(ctx, f)
        vy = ctx.vector(y); ctx.spmv(1.0, A32, vx, 0.5, vy); out.append(vy.numpy())          # FD
        fy = _f32vec(ctx, y); ctx.spmv(1.0, A32, fx, 0.5, fy); out.append(fy.numpy32())       # FF
        vz = ctx.vector(y); ctx.spmv(1.0, A32, fx, 1.0, vz); out.append(vz.numpy())           # FFD
        vr = ctx.vector(n); ctx.residual(vf, A32, vx, vr); out.append(vr.numpy())             # FD
        fr = _f32vec(ctx, np.zeros(n)); ctx.residual(vf, A32, vx, fr); out.append(fr.numpy32())   # FDF
        fr2 = _f32vec(ctx, np.zeros(n)); ctx.residual(ff, A32, fx, fr2); out.append(fr2.numpy32())  # FF
        fd, ft = _f32vec(ctx, d), _f32vec(ctx, np.zeros(n))
        fxx = _f32vec(ctx, x); ctx.relax(A32, ff, fxx, ft, fd, 0.72); out.append(fxx.numpy32())     # FF sweep
        vxx = ctx.vector(x); ctx.relax(A32, vf, vxx, ft, fd, 0.72); out.append(vxx.numpy())         # FD sweep
        return np.concatenate([np.asarray(v, dtype=np.float64) for v in out])
    a, b = both(ctx, run)
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("precision", ["f64", "mixed"])
def test_solver_is_bit_transparent_to_narrow_columns(ctx, precision):
    """The whole drop-in solve with the coarse operators narrowed against the same solve with
    plain columns; the library profile names the format each pass streamed."""
    ptr, col, val, rhs = ab.poisson3d(48)
    res, fmts = [], []
    for on in (1, 0):
        ctx.set_option("narrow_columns", on)
        S = ab.DropinSolver(ptr, col, val, "damped_jacobi", "cg", ctx=ctx, precision=precision)
        ctx.profile_begin()
        res.append(S.solve(rhs))
        fmts.append({p["format"] for p in ctx.profile_end() if p["nnz"] > 0})
        S.close()
    ctx.set_option("narrow_columns", 1)
    assert res[0][1] == res[1][1] and np.array_equal(res[0][0], res[1][0])
    assert fmts[0] & {"col16", "col24"} and not fmts[1] & {"col16", "col24"}


@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: "S%d-C%d-cap%d" % k)
@pytest.mark.parametrize("width", WIDTHS)
def test_ring_knobs_narrow(ctx, knobs, width):
    """The ring-knob cases of tests/test_gpu_accuracy.py on narrow columns: rings of 1..8
    stages, 1..4 CTAs per SM, 256..6144 entries per block, every row within its error bound."""
    stages, ctas, cap = knobs
    i = KNOBS.index(knobs)
    with options(ctx, stages=stages, ctas_per_sm=ctas, nnz_cap=cap, spmv_variant=1, lanes=0,
                 patterns=0, offsets=0, window=0, narrow_columns=1):
        def make(nr):
            nc = max(nr, 150000)
            ptr, col, val = narrow_csr(nr, nc, 1 + (i % 2), width, seed=nr + cap)
            rng = np.random.default_rng(nr)
            return ptr, col, val * np.exp2(rng.uniform(-20, 20, val.size)), rng.uniform(-1, 1, nc)
        ptr, col, val, x = sized(make, knobs, 0, 1 + i % 3)
        c = Case(ctx, ptr, col, val, x, seed=ptr.size)
        assert c.A.narrow() == width
        walks_the_ring(c, knobs, "plain")
        c.check_all("col%d stages=%d ctas=%d cap=%d" % (width, stages, ctas, cap))
