"""GPU parity of the FP32 copy of an FP64 operator's values (option "narrow_values", csr_kernels.cuh
PrecSD): an operator whose every value is exactly an FP32 must give the same bits whether the
streaming passes read its 4-byte or its 8-byte values -- in every mode, in every column format,
on every lane width the format allows, in the fused Krylov steps and in whole solves.  The paths
that keep reading the FP64 values (the one-block-per-CTA variant, the small-operator kernel, the
coarse tail) must not change, and one inexact value keeps an operator at 8 bytes."""
import contextlib

import numpy as np
import pytest

import amgcl_b200 as ab

pytestmark = pytest.mark.gpu


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


def exact32(rng, n):
    """FP64 values that are all exact FP32 numbers, over a wide range of exponents."""
    return rng.uniform(-1, 1, n).astype(np.float32).astype(np.float64) * np.exp2(rng.integers(-20, 21, n))


def banded(n, per_row, seed, far=0):
    """Square operator, rows of about per_row entries around the diagonal; far > 0: about 30 %
    of the entries `far` columns further right (a column span beyond 16 bits per block)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(max(0, per_row - 3), per_row + 4, n)
    lens[::97] = 0
    ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    rows = np.repeat(np.arange(n), lens)
    col = rows + rng.integers(-2 * per_row, 2 * per_row + 1, rows.size)
    if far:
        col = np.where(rng.uniform(size=rows.size) < 0.3, col + far, col)
    col = np.clip(col, 0, n - 1)
    o = np.lexsort((col, rows))
    return ptr, col[o], exact32(rng, rows.size)


def stencil(n, offsets, seed):
    """Square operator with entries at row + k for every k in offsets that stays inside the
    matrix: few row patterns and few (col - row), so it qualifies for the pattern and the
    offset format."""
    rows = np.repeat(np.arange(n), len(offsets))
    col = rows + np.tile(np.asarray(offsets), n)
    keep = (col >= 0) & (col < n)
    rows, col = rows[keep], col[keep]
    ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=ptr[1:])
    return ptr, col.astype(np.int64), exact32(np.random.default_rng(seed), col.size)


# format -> (context options, lanes it allows, operator for `lanes`, check of the stored format)
FORMATS = {
    "plain": (dict(patterns=0, offsets=0, window=0, narrow_columns=0), [1, 2, 4, 8, 16, 32],
              lambda L: banded(20000 if L < 16 else 8000, 6 * L, L),
              lambda A: A.narrow() == 0 and not A.patterns()["pattern_indexed"]),
    "pattern": (dict(patterns=1, patterns_min_nnz=0, offsets=0, window=0), [1, 2, 4],
                lambda L: stencil(30000, list(range(-3 * L, 3 * L + 1, 1)), L),
                lambda A: A.patterns()["pattern_indexed"]),
    "offset": (dict(patterns=0, offsets=1, offsets_min_nnz=0, window=0), [1, 2, 4],
               lambda L: stencil(30000, list(range(-3 * L, 3 * L + 1, 1)), L),
               lambda A: A.offsets()["offset_indexed"]),
    "col16": (dict(patterns=0, offsets=0, window=0, narrow_columns=1), [1, 2, 4, 8],
              lambda L: banded(30000, 6 * L, 10 + L),
              lambda A: A.narrow() == 16),
    "col24": (dict(patterns=0, offsets=0, window=0, narrow_columns=1), [1, 2, 4, 8],
              lambda L: banded(90000, 6 * L, 20 + L, far=70000),
              lambda A: A.narrow() == 24),
    "window": (dict(patterns=0, offsets=0, window=1, window_min_nnz=0), [1, 2, 4, 8],
               lambda L: banded(30000, 6 * L, 30 + L),
               lambda A: A.window()["windowed"]),
}
CASES = [(f, L) for f, (_, lanes, _, _) in FORMATS.items() for L in lanes]


def both(ctx, fn):
    """fn() streaming the FP32 values, then the FP64 ones (the same uploaded operator); also the
    value widths the library profile reports for each run's CSR passes."""
    out, widths = [], []
    try:
        for on in (1, 0):
            ctx.set_option("narrow_values", on)
            ctx.profile_begin()
            out.append(fn())
            widths.append({p["value_bytes"] for p in ctx.profile_end() if p["nnz"] > 0
                           and p["mode"] in ("spmv", "spmv_acc", "residual", "relax", "residual_scaled")})
    finally:
        ctx.set_option("narrow_values", 1)
    return out, widths


def all_modes(ctx, A, n, seed):
    """MODE 0-4 on A: spmv with beta 0 and beta != 0, residual, the smoother sweep, and the
    fused first sweep from x = 0 through the real relax -> residual sequence."""
    rng = np.random.default_rng(seed)
    x, y, f, d = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.1, 1, n)
    vx, vf, vd = ctx.vector(x), ctx.vector(f), ctx.vector(d)

    def run():
        out = []
        for beta in (0.0, -0.25):
            vy = ctx.vector(y)
            ctx.spmv(1.5, A, vx, beta, vy)
            out.append(vy.numpy())
        vr = ctx.vector(n)
        ctx.residual(vf, A, vx, vr)
        out.append(vr.numpy())
        for zero in (False, True):
            vxx, vt, vr = ctx.vector(x), ctx.vector(n), ctx.vector(n)
            if zero:
                ctx.clear(vxx)
            ctx.relax(A, vf, vxx, vt, vd, 0.72)
            ctx.residual(vf, A, vxx, vr)
            out += [vxx.numpy(), vr.numpy()]
        return np.concatenate(out)
    return run


@pytest.mark.parametrize("fmt,lanes", CASES, ids=["%s-L%d" % c for c in CASES])
def test_fp32_values_give_the_bits_of_fp64_values(ctx, fmt, lanes):
    opts, _, make, stored = FORMATS[fmt]
    ptr, col, val = make(lanes)
    n = ptr.size - 1
    with options(ctx, lanes=lanes, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **opts):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.plan()["lanes"] == lanes and stored(A), fmt
        assert A.value_bytes() == 4
        (a, b), widths = both(ctx, all_modes(ctx, A, n, lanes))
        np.testing.assert_array_equal(a, b)
        assert widths == [{4}, {8}]


@pytest.mark.parametrize("fmt", ["pattern", "col16"])
def test_fused_cg_and_bicgstab_steps(ctx, fmt):
    """The streaming passes that also leave scalars behind: q = A p with <q, p> (CG), and
    BiCGStab's two A-passes with their dot products."""
    opts, _, make, stored = FORMATS[fmt]
    ptr, col, val = make(1)
    n = ptr.size - 1
    rng = np.random.default_rng(4)
    x0, f, d = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.1, 1, n)
    with options(ctx, lanes=1, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **opts):
        A = ctx.csr(n, n, ptr, col, val)
        assert stored(A) and A.value_bytes() == 4

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
            (a, b), widths = both(ctx, fn)
            np.testing.assert_array_equal(a, b)
            assert widths == [{4}, {8}]


def solve_both(ctx, n, relax, krylov):
    """The drop-in solve uploaded with narrow_values 1 and with 0 (the option decides at upload
    whether the FP32 copy is built): results, and the value width of the finest operator's passes."""
    ptr, col, val, rhs = ab.poisson3d(n)
    res, widths = [], []
    try:
        for on in (1, 0):
            ctx.set_option("narrow_values", on)
            S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
            ctx.profile_begin()
            res.append(S.solve(rhs))
            widths.append({p["value_bytes"] for p in ctx.profile_end() if p["nnz"] == col.size})
            S.close()
    finally:
        ctx.set_option("narrow_values", 1)
    return res, widths


@pytest.mark.parametrize("relax,krylov", [("damped_jacobi", "cg"), ("spai0", "bicgstab")])
def test_whole_solves_64(ctx, relax, krylov):
    (a, b), widths = solve_both(ctx, 64, relax, krylov)
    assert a[1] == b[1] and a[2] == b[2]
    np.testing.assert_array_equal(a[0], b[0])
    assert widths == [{4}, {8}]


def test_headline_solve_256(ctx):
    """The benchmarked solve: Poisson 256^3, SA + damped Jacobi + CG."""
    (a, b), widths = solve_both(ctx, 256, "damped_jacobi", "cg")
    assert a[1] == b[1] and a[2] == b[2]
    np.testing.assert_array_equal(a[0], b[0])
    assert widths == [{4}, {8}]


def test_one_inexact_value_keeps_the_operator_at_8_bytes(ctx):
    ptr, col, val = FORMATS["pattern"][2](1)
    n = ptr.size - 1
    with options(ctx, narrow_values=1, narrow_values_min_nnz=0):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.value_bytes() == 4
        v = val.copy()
        v[v.size // 2] = 0.1
        B = ctx.csr(n, n, ptr, col, v)
        assert B.value_bytes() == 8
        assert B.bytes() < A.bytes()
        vx, vy = ctx.vector(np.ones(n)), ctx.vector(n)
        ctx.profile_begin()
        ctx.spmv(1.0, B, vx, 0.0, vy)
        assert {p["value_bytes"] for p in ctx.profile_end() if p["nnz"] > 0} == {8}
    with options(ctx, narrow_values=0, narrow_values_min_nnz=0):
        assert ctx.csr(n, n, ptr, col, val).value_bytes() == 8       # not built
    with options(ctx, narrow_values=1):
        assert ctx.csr(n, n, ptr, col, val).value_bytes() == 8       # below narrow_values_min_nnz


@pytest.mark.parametrize("path", ["spmv_variant_0", "small_kernel", "coarse_tail"])
def test_fp64_value_paths_are_unchanged(ctx, path):
    """The cross-check variant, the small-operator kernel and the coarse tail read the FP64
    values of an operator that also has the FP32 copy, and give the bits they give without it."""
    ptr, col, val = FORMATS["col16"][2](2)
    n = ptr.size - 1
    opts = {"spmv_variant_0": dict(spmv_variant=0),
            "small_kernel": dict(small_kernel_max_nnz=col.size, fuse_first_sweep=0),
            "coarse_tail": dict(coarse_tail=1, tail_max_nnz=col.size, fuse_first_sweep=0)}[path]
    with options(ctx, narrow_values=1, narrow_values_min_nnz=0, **opts):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.value_bytes() == 4
        run = all_modes(ctx, A, n, 9)
        tail0 = ctx.tail_stats()[1]
        (a, b), widths = both(ctx, run)
        np.testing.assert_array_equal(a, b)
        if path == "coarse_tail":
            assert ctx.tail_stats()[1] > tail0 and widths == [set(), set()]
        else:
            assert widths == [{8}, {8}]
