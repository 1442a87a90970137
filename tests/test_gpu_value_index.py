"""GPU parity of indexed values (option "narrow_values", csr_kernels.cuh PrecI8D / PrecI16D): an
FP64 operator with at most 4,096 distinct values must give the same bits whether the streaming
passes read an 8- / 16-bit index into the table of its values or the FP64 values themselves --
in every mode, column format and lane width, in the fused Krylov steps and in whole solves.  The
paths that keep reading the FP64 values must not change, and an operator whose table does not fit
beside the ring keeps reading 8 bytes."""
import numpy as np
import pytest

import _accuracy as acc
import amgcl_b200 as ab
from test_gpu_values import FORMATS as VALUE_FORMATS, all_modes, both, options
from test_gpu_accuracy import Case

pytestmark = pytest.mark.gpu

# the formats that stream an index (the windowed format keeps FP64 values)
FORMATS = {k: v for k, v in VALUE_FORMATS.items() if k != "window"}
CASES = [(f, L, w) for f, (_, lanes, _, _) in FORMATS.items() for L in lanes for w in (1, 2)]


def few_values(size, k, seed):
    """size FP64 values drawn from k distinct ones, none of them exact in FP32 (so the FP32 copy
    does not take the operator first)."""
    rng = np.random.default_rng(seed)
    pool = rng.uniform(-1, 1, k) / 9.0 * np.exp2(rng.integers(-20, 21, k))
    pool[0] = 1.0 / 3.0
    v = pool[rng.integers(0, k, size)]
    v[:k] = pool                                     # every pool value occurs
    assert not ab.values_fit_f32(v)
    return v


def operator(fmt, lanes, width, seed=0, k=None):
    ptr, col, _ = FORMATS[fmt][2](lanes)
    k = k or (100 if width == 1 else 1500)
    return ptr, col, few_values(col.size, k, seed + 31 * lanes + width)


@pytest.mark.parametrize("fmt,lanes,width", CASES, ids=["%s-L%d-%dB" % c for c in CASES])
def test_indexed_values_give_the_bits_of_fp64_values(ctx, fmt, lanes, width):
    opts, _, _, stored = FORMATS[fmt]
    ptr, col, val = operator(fmt, lanes, width)
    n = ptr.size - 1
    with options(ctx, lanes=lanes, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **opts):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.plan()["lanes"] == lanes and stored(A), fmt
        assert A.value_bytes() == width
        (a, b), widths = both(ctx, all_modes(ctx, A, n, lanes))
        np.testing.assert_array_equal(a, b)
        assert widths == [{width}, {8}]


@pytest.mark.parametrize("width", [1, 2])
@pytest.mark.parametrize("fmt", ["pattern", "col24"])
def test_fused_cg_and_bicgstab_steps(ctx, fmt, width):
    """The passes that also leave scalars behind: q = A p with <q, p> (CG), and BiCGStab's two
    A-passes with their dot products."""
    opts, _, _, stored = FORMATS[fmt]
    ptr, col, val = operator(fmt, 1, width, seed=5)
    n = ptr.size - 1
    rng = np.random.default_rng(4)
    x0, f, d = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.1, 1, n)
    with options(ctx, lanes=1, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **opts):
        A = ctx.csr(n, n, ptr, col, val)
        assert stored(A) and A.value_bytes() == width

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
            assert widths == [{width}, {8}]


@pytest.mark.parametrize("width", [1, 2])
@pytest.mark.parametrize("fmt,lanes", [("plain", 1), ("plain", 32), ("pattern", 2), ("col16", 4), ("col24", 8)])
def test_indexed_passes_meet_the_per_row_bounds(ctx, fmt, lanes, width):
    """Every mode on the indexed path within the extended-precision per-row bounds of
    tests/_accuracy.py (the operands as stored: the FP64 values)."""
    acc.require_longdouble()
    opts = FORMATS[fmt][0]
    ptr, col, val = operator(fmt, lanes, width, seed=9)
    x = np.random.default_rng(lanes).uniform(-1, 1, ptr.size - 1)
    with options(ctx, lanes=lanes, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **opts):
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        assert c.A.value_bytes() == width
        ctx.profile_begin()
        c.check_all("indexed %s L=%d" % (fmt, lanes))
        assert {p["value_bytes"] for p in ctx.profile_end() if p["nnz"] > 0} == {width}


@pytest.mark.parametrize("path", ["spmv_variant_0", "small_kernel", "coarse_tail"])
def test_fp64_value_paths_are_unchanged(ctx, path):
    """The cross-check variant, the small-operator kernel and the coarse tail read the FP64
    values of an indexed operator, and give the bits they give without the index."""
    ptr, col, val = operator("col16", 2, 1, seed=3)
    n = ptr.size - 1
    opts = {"spmv_variant_0": dict(spmv_variant=0),
            "small_kernel": dict(small_kernel_max_nnz=col.size, fuse_first_sweep=0),
            "coarse_tail": dict(coarse_tail=1, tail_max_nnz=col.size, fuse_first_sweep=0)}[path]
    with options(ctx, lanes=2, narrow_values=1, narrow_values_min_nnz=0, **FORMATS["col16"][0], **opts):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.value_bytes() == 1
        run = all_modes(ctx, A, n, 9)
        tail0 = ctx.tail_stats()[1]
        (a, b), widths = both(ctx, run)
        np.testing.assert_array_equal(a, b)
        if path == "coarse_tail":
            assert ctx.tail_stats()[1] > tail0 and widths == [set(), set()]
        else:
            assert widths == [{8}, {8}]


def test_table_that_does_not_fit_beside_the_ring_keeps_8_bytes(ctx):
    """4,096 values (32 KB of table): beside two plain-format stages they do not fit the budget of
    four CTAs per SM, so the plain operator keeps its FP64 values; the col16 operator gets the
    index, and streams FP64 values again when the ring is configured deeper after the upload."""
    ptr, col, _ = FORMATS["col16"][2](1)
    val = few_values(col.size, 4096, 77)
    n = ptr.size - 1
    with options(ctx, lanes=1, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **FORMATS["plain"][0]):
        P = ctx.csr(n, n, ptr, col, val)
        assert P.narrow() == 0 and P.value_bytes() == 8
    with options(ctx, lanes=1, spmv_variant=1, narrow_values=1, narrow_values_min_nnz=0, **FORMATS["col16"][0]):
        A = ctx.csr(n, n, ptr, col, val)
        assert A.narrow() == 16 and A.value_bytes() == 2
        assert A.bytes() > P.bytes()
        run = all_modes(ctx, A, n, 2)
        (a, b), widths = both(ctx, run)
        np.testing.assert_array_equal(a, b)
        assert widths == [{2}, {8}]
        with options(ctx, stages=3):
            ctx.profile_begin()
            c = run()
            assert {p["value_bytes"] for p in ctx.profile_end() if p["nnz"] > 0} == {8}
        np.testing.assert_array_equal(a, c)
    with options(ctx, narrow_values=1, narrow_values_min_nnz=0):
        assert ctx.csr(n, n, ptr, col, few_values(col.size, 4097, 78)).value_bytes() == 8


def solve_both(ctx, n):
    """The drop-in solve (SA + damped Jacobi + CG) uploaded with narrow_values 1 and 0: results,
    and per finest-level P0 / R0 and first coarse operator A1 the value widths of their passes."""
    ptr, col, val, rhs = ab.poisson3d(n)
    N = n ** 3
    res, widths = [], []
    try:
        for on in (1, 0):
            ctx.set_option("narrow_values", on)
            S = ab.DropinSolver(ptr, col, val, "damped_jacobi", "cg", ctx=ctx)
            ctx.profile_begin()
            res.append(S.solve(rhs))
            prof = [p for p in ctx.profile_end() if p["value_bytes"]]
            n1 = next(p["ncols"] for p in prof if p["nrows"] == N and p["ncols"] < N)
            w = {"A0": set(), "P0": set(), "R0": set(), "A1": set()}
            for p in prof:
                key = ("A0" if p["nrows"] == p["ncols"] == N else "P0" if p["nrows"] == N
                       else "R0" if p["ncols"] == N else "A1" if p["nrows"] == p["ncols"] == n1 else None)
                if key:
                    w[key].add(p["value_bytes"])
            widths.append(w)
            S.close()
    finally:
        ctx.set_option("narrow_values", 1)
    return res, widths


@pytest.mark.parametrize("n", [128, 256])
def test_whole_solves(ctx, n):
    """Poisson 128^3 and the benchmarked 256^3 solve: identical iterations, residual and x."""
    (a, b), widths = solve_both(ctx, n)
    assert a[1] == b[1] and a[2] == b[2]
    np.testing.assert_array_equal(a[0], b[0])
    assert widths[0] == {"A0": {4}, "P0": {1}, "R0": {1}, "A1": {2}}
    assert widths[1] == {"A0": {8}, "P0": {8}, "R0": {8}, "A1": {8}}
