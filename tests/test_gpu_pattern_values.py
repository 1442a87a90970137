"""GPU parity of value-keyed patterns (option "pattern_values", csr_kernels.cuh FMT_PATVAL): an
operator whose rows take few (offset, value) patterns gives the same bits whether the streaming
passes take its values from the pattern table (FP32 where exact, else FP64) or stream them
(FMT_PATTERN) -- in every mode, on 1, 2 and 4 lanes, for every precision the format is
instantiated for, in the fused Krylov steps and in whole solves -- and stays within the
extended-precision per-row bounds of tests/_accuracy.py."""
import contextlib

import numpy as np
import pytest

import amgcl_b200 as ab
import _accuracy as acc
from test_gpu_accuracy import Case, PRECS
from test_gpu_values import all_modes
from test_offsets import diag_matrix

pytestmark = pytest.mark.gpu

PATTERN = dict(patterns=1, patterns_min_nnz=0, offsets=0, window=0, spmv_variant=1)
CSR_MODES = ("spmv", "spmv_acc", "residual", "relax", "residual_scaled")


@contextlib.contextmanager
def options(ctx, **kw):
    old = {k: ctx.get_option(k) for k in kw}
    try:
        for k, v in kw.items():
            ctx.set_option(k, v)
        yield
    finally:
        for k, v in old.items():
            ctx.set_option(k, v)


def coefficient(off, exact):
    """The value of every entry at col - row == off: exact FP32 numbers, or thirds (not exact)."""
    off = np.asarray(off, dtype=np.float64)
    return 1.0 + 0.25 * off if exact else (1.1 + off) / 3.0


def stencil(n, offsets, exact):
    """Square operator with entries at row + k for every k in offsets inside the matrix, its
    value a function of k: few (offset, value) row patterns."""
    rows = np.repeat(np.arange(n), len(offsets))
    col = rows + np.tile(np.asarray(offsets), n)
    keep = (col >= 0) & (col < n)
    rows, col = rows[keep], col[keep]
    ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=ptr[1:])
    return ptr, col.astype(np.int64), coefficient(col - rows, exact)


# (pattern_values, narrow_values) at launch: the FP32 table (where exact), the FP64 table, the
# streamed FP64 values of the same uploaded operator
CONFIGS = ((1, 1), (1, 0), (0, 1))


def every_config(ctx, fn):
    """fn() under each of CONFIGS, and the (format, value width) each run's CSR passes reported."""
    out, seen = [], []
    for pv, nv in CONFIGS:
        with options(ctx, pattern_values=pv, narrow_values=nv):
            ctx.profile_begin()
            out.append(fn())
            seen.append({(p["format"], p["value_bytes"]) for p in ctx.profile_end()
                         if p["nnz"] > 0 and p["mode"] in CSR_MODES})
    return out, seen


def expected(exact):
    return [{("pattern_values", 4 if exact else 8)}, {("pattern_values", 8)}, {("pattern", 8)}]


@pytest.mark.parametrize("exact", [True, False], ids=["fp32_table", "fp64_table"])
@pytest.mark.parametrize("lanes", [1, 2, 4])
def test_every_mode_gives_the_bits_of_streamed_values(ctx, lanes, exact):
    ptr, col, val = stencil(30000, list(range(-3 * lanes, 3 * lanes + 1)), exact)
    n = ptr.size - 1
    with options(ctx, lanes=lanes, narrow_values=1, narrow_values_min_nnz=0, **PATTERN):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.plan()["lanes"] == lanes and A.patterns()["pattern_indexed"]
        assert A.value_bytes() == (4 if exact else 8)
        run = all_modes(ctx, A, n, lanes)
        ctx.profile_begin()
        run()
        assert "residual_scaled" in {p["mode"] for p in ctx.profile_end()}, "the fused first sweep did not run"
        out, seen = every_config(ctx, run)
        for o in out[1:]:
            np.testing.assert_array_equal(out[0], o)
        assert seen == expected(exact)


@pytest.mark.parametrize("exact", [True, False], ids=["fp32_table", "fp64_table"])
def test_fused_cg_and_bicgstab_steps(ctx, exact):
    """q = A p with <q, p> (CG), and BiCGStab's two A-passes with their dot products."""
    ptr, col, val = stencil(30000, list(range(-3, 4)), exact)
    n = ptr.size - 1
    rng = np.random.default_rng(4)
    x0, f, d = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.1, 1, n)
    with options(ctx, lanes=1, narrow_values=1, narrow_values_min_nnz=0, **PATTERN):
        A = ctx.csr(n, n, ptr, col, val)

        def cg():
            K = ab.Krylov(ctx, n)
            vp, vq, vxx, vr = ctx.vector(x0), ctx.vector(n), ctx.vector(d), ctx.vector(f)
            out = []
            for _ in range(3):
                K.cg_direction(vr, vr, vp)
                rr = K.cg_step(A, vp, vq, vxx, vr)
                s = K.scalars()
                out += [vq.numpy(), vxx.numpy(), vr.numpy(), [rr, s["qp"], s["alpha"], s["rr"]]]
            K.close()
            return np.concatenate(out)

        def bicg():
            K = ab.Krylov(ctx, n)
            rhs, x = ctx.vector(f), ctx.vector(x0)
            r, p, v, s, t, rh, T = (ctx.vector(n) for _ in range(7))
            dv = ctx.vector(d)
            out = [[K.residual(rhs, A, x, r)]]
            K.bicg_start(r, rh)
            for _ in range(3):
                K.bicg_direction(r, v, p)
                ctx.vmul(1.0, dv, p, 0.0, T)
                ss = K.bicg_step_s(A, rh, T, v, r, s, x)
                sc = K.scalars()
                out += [v.numpy(), s.numpy(), [ss, sc["rho"], sc["alpha"]]]
                ctx.vmul(1.0, dv, s, 0.0, T)
                rr = K.bicg_step_r(A, rh, T, t, s, r, x)
                sc = K.scalars()
                out += [t.numpy(), x.numpy(), r.numpy(), [rr, sc["omega"], sc["rho_next"]]]
            K.close()
            return np.concatenate(out)

        for fn in (cg, bicg):
            out, seen = every_config(ctx, fn)
            for o in out[1:]:
                np.testing.assert_array_equal(out[0], o)
            assert seen == expected(exact)


def band(nr, exact, keep):
    """A ragged band of tests/_accuracy.py's offsets whose values depend on the offset only."""
    from test_gpu_accuracy import BAND_OFFS
    ptr, col, _ = diag_matrix(nr, nr, BAND_OFFS, seed=nr, keep=keep)
    rows = np.repeat(np.arange(nr), np.diff(ptr))
    x = np.random.default_rng(nr).uniform(-1, 1, nr)
    return ptr, col, coefficient(col - rows, exact), x


@pytest.mark.parametrize("prec,exact", [("DD", True), ("DD", False)] + [(p, True) for p in PRECS if p != "DD"])
def test_precisions_meet_the_per_row_bounds(ctx, prec, exact):
    """Every precision the format is instantiated for, within the per-row bounds, and the bits
    of the streamed values."""
    acc.require_longdouble()
    ptr, col, val, x = band(9001, exact, keep=1.0)
    with options(ctx, lanes=0, narrow_values=1, narrow_values_min_nnz=0, **PATTERN):
        c = Case(ctx, ptr, col, val, x, prec=prec, seed=3)
        assert c.A.patterns()["pattern_indexed"]
        ctx.profile_begin()
        c.check_all("pattern_values")
        width = 8 if prec == "DD" and not exact else 4
        assert {(p["format"], p["value_bytes"]) for p in ctx.profile_end() if p["nnz"] > 0} == \
            {("pattern_values", width)}
        on = [c.run(m) for m in c.modes]
        with options(ctx, pattern_values=0):
            off = [c.run(m) for m in c.modes]
        for a, b in zip(on, off):
            np.testing.assert_array_equal(a, b)


def solve_both(ctx, n, relax, krylov, precision="f64"):
    """The drop-in solve uploaded with pattern_values 1 and 0: results, and the formats the
    finest operator's passes reported."""
    ptr, col, val, rhs = ab.poisson3d(n)
    res, fmts = [], []
    for on in (1, 0):
        with options(ctx, pattern_values=on):
            S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx, precision=precision)
            ctx.profile_begin()
            res.append(S.solve(rhs))
            fmts.append({p["format"] for p in ctx.profile_end() if p["nnz"] == col.size})
            S.close()
    return res, fmts


@pytest.mark.parametrize("relax,krylov,precision", [("damped_jacobi", "cg", "f64"), ("spai0", "bicgstab", "f64"),
                                                     ("damped_jacobi", "cg", "mixed")])
def test_whole_solves_64(ctx, relax, krylov, precision):
    (a, b), fmts = solve_both(ctx, 64, relax, krylov, precision)
    assert a[1] == b[1] and a[2] == b[2]
    np.testing.assert_array_equal(a[0], b[0])
    assert fmts == [{"pattern_values"}, {"pattern"}]


def test_headline_solve_256(ctx):
    """The benchmarked solve: Poisson 256^3, SA + damped Jacobi + CG."""
    (a, b), fmts = solve_both(ctx, 256, "damped_jacobi", "cg")
    assert a[1] == b[1] and a[2] == b[2]
    np.testing.assert_array_equal(a[0], b[0])
    assert fmts == [{"pattern_values"}, {"pattern"}]
