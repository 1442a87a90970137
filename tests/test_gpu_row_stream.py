"""The ring kernel's stream of rows (csr_kernels.cuh, csr_ring_kernel): a CTA hands the rows of
the blocks it walks to its warps in chunks of 32 / L rows, across block boundaries, without a CTA
barrier between blocks.  Which warp reduces a row must not change the row's bits: every pass must
give the vectors of the one-block-per-CTA kernel (spmv_variant = 0), stay within the per-row
bounds of tests/_accuracy.py, and leave in-kernel scalars that are within csr_scalar_bound and the
same from run to run.  The cases are built so that blocks end in a partial chunk, so that the
stream position of a block's first row is not a multiple of the warp count, and so that long
blocks (reduced by the whole CTA) sit between short ones."""
import numpy as np
import pytest

import amgcl_b200 as ab
import _accuracy as acc
from test_gpu_accuracy import FORMAT_OPTS, OMEGA, Case, options, sized, sms

pytestmark = pytest.mark.gpu

# 2 lanes at ~30 entries per row (the coarse operators of smoothed aggregation at 256^3),
# 4 lanes at ~50
PER_ROW = {2: 30, 4: 50}
FMTS = {"plain": dict(narrow_columns=0), "col16": dict(narrow_columns=1), "col24": dict(narrow_columns=1)}


def long_row_csr(n, per, width, seed, long_rows=0):
    """A square operator with about `per` entries per row (a few empty rows), columns sorted
    within each row; width 16: every row within 2000 columns of the diagonal, width 24: a third
    of the entries 70 000 columns further on, modulo n (so some blocks need 24-bit columns);
    long_rows rows of 2500 entries (each makes a block too long to stage)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(per // 2, 3 * per // 2 + 1, n)
    lens[rng.uniform(size=n) < 0.03] = 0
    lens[rng.choice(n, long_rows, replace=False)] = 2500
    ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    rows = np.repeat(np.arange(n), lens)
    col = rows + rng.integers(-2000, 2000, rows.size)
    if width == 24:
        col = np.where(rng.uniform(size=rows.size) < 0.3, (col + 70000) % n, col)
    col = np.clip(col, 0, n - 1)
    col = col[np.lexsort((col, rows))]
    val = rng.uniform(-1, 1, col.size) * np.exp2(rng.uniform(-20, 20, col.size))
    return ptr, col.astype(np.int64), val, rng.uniform(-1, 1, n)


def partial_chunks(c, lanes):
    """Blocks of the plan whose row count is not a multiple of 32 / lanes."""
    rows = np.diff(np.append(c.p["starts"], c.nr))
    return int((rows % (32 // lanes) != 0).sum())


def decoupled(c, lanes):
    """Whether the ring kernel runs the operator without a CTA barrier between blocks: most
    staged blocks have fewer chunks of 32 / lanes rows than a CTA has warps (csr_create)."""
    rows = np.diff(np.append(c.p["starts"], c.nr))
    few = (-(-rows // (32 // lanes)) < 8) & ~c.p["long"]
    return 2 * int(few.sum()) > c.p["nblocks"]


def on_variant(ctx, variant, fn):
    with options(ctx, spmv_variant=variant):
        return fn()


def scalar_bound(ctx, c, lanes):
    return lambda s: acc.csr_scalar_bound(s, c.A.plan()["blocks"], c.p["rows_cap"], lanes, sms(),
                                          ctx.get_option("ctas_per_sm"))


def modes_match_block_kernel(ctx, c, what):
    """Every mode: within its bound on the ring kernel, and the bits of csr_block_kernel."""
    for mode in c.modes:
        got = on_variant(ctx, 1, lambda: c.run(mode))
        c.check(mode, got, what)
        np.testing.assert_array_equal(got, on_variant(ctx, 0, lambda: c.run(mode)), err_msg="%s %s" % (what, mode))


def fused_first_sweep(ctx, c):
    """clear -> relax -> residual: (x, r) and the number of launches it took."""
    vf, vd = ctx.vector(c.f), ctx.vector(c.d)
    vx, vt, vr = ctx.vector(c.nr), ctx.vector(c.nr), ctx.vector(c.nr)
    ctx.clear(vx)
    l0 = ctx.launches
    ctx.relax(c.A, vf, vx, vt, vd, OMEGA)
    ctx.residual(vf, c.A, vx, vr)
    return vx.numpy(), vr.numpy(), ctx.launches - l0


def cg_step(ctx, c, s):
    """CG's direction p from s, then q = A p with <q, p> left by the same pass: (q, <q,p>, p)."""
    K = ab.Krylov(ctx, c.nr)
    try:
        vs, vp, vq, vx, vr = ctx.vector(s), ctx.vector(c.nr), ctx.vector(c.nr), ctx.vector(c.x), ctx.vector(c.f)
        K.cg_direction(vs, vs, vp)
        K.cg_step(c.A, vp, vq, vx, vr)
        return vq.numpy(), K.scalars()["qp"], vp.numpy()
    finally:
        K.close()


def sweep_dot(ctx, c):
    """A smoother sweep that leaves <rhs, x_new> behind (while a Krylov solver of its size
    lives): (x_new, the in-kernel scalar)."""
    K = ab.Krylov(ctx, c.nr)
    try:
        vf, vxx, vt, vd = ctx.vector(c.f), ctx.vector(c.x), ctx.vector(c.nr), ctx.vector(c.d)
        ctx.relax(c.A, vf, vxx, vt, vd, OMEGA)
        l0 = ctx.launches
        got = ctx.dot(vf, vxx)
        assert ctx.launches == l0, "<rhs, x_new> was not produced by the sweep"
        return vxx.numpy(), got
    finally:
        K.close()


@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("lanes", [2, 4])
def test_partial_chunks_every_mode(ctx, lanes, fmt):
    width = 16 if fmt == "col16" else 24
    with options(ctx, lanes=lanes, spmv_variant=1, coarse_tail=0, **FORMAT_OPTS["plain"], **FMTS[fmt]):
        ptr, col, val, x = long_row_csr(90001, PER_ROW[lanes], width, seed=10 * lanes + width)
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        assert c.A.plan()["lanes"] == lanes and c.A.plan()["long_blocks"] == 0
        if fmt != "plain":
            assert c.A.narrow() == width
        assert partial_chunks(c, lanes) > c.p["nblocks"] // 4 and decoupled(c, lanes)
        ctx.profile_begin()
        c.run("spmv")
        assert {p["format"] for p in ctx.profile_end() if p["nnz"] > 0} == {fmt}
        what = "%s lanes=%d" % (fmt, lanes)
        modes_match_block_kernel(ctx, c, what)

        # CG's q = A p with <q, p>; the sweep with <rhs, x_new>
        csb = scalar_bound(ctx, c, lanes)
        s0 = np.random.default_rng(lanes).uniform(-1, 1, c.nr)
        q, qp, p = cg_step(ctx, c, s0)
        q0, _, p0 = on_variant(ctx, 0, lambda: cg_step(ctx, c, s0))
        np.testing.assert_array_equal(p, p0)
        np.testing.assert_array_equal(q, q0)
        want, bnd = c.want("spmv", p)
        acc.assert_rows(q, want / acc.LD(1.5), bnd / 1.5, what + " cg_step q", ptr, c.p)
        S, A = acc.dot_ref(q, p)
        acc.assert_scalar(qp, S, csb(A), what + " <q,p> of cg_step")
        xn, rx = sweep_dot(ctx, c)
        c.check("relax", xn, what + " sweep with <rhs,x>")
        S, A = acc.dot_ref(c.f, xn)
        acc.assert_scalar(rx, S, csb(A), what + " <rhs, x_new> of the sweep")


@pytest.mark.parametrize("fmt", ["plain", "col16"])
@pytest.mark.parametrize("lanes", [2, 4])
def test_partial_chunks_fused_first_sweep(ctx, lanes, fmt):
    """clear -> relax -> residual as one pass (MODE_RESID_SCALED).  With more than one lane per
    row the library fuses it up to 32768 rows, too few columns for 24-bit blocks."""
    with options(ctx, lanes=lanes, spmv_variant=1, fuse_first_sweep=1, coarse_tail=0,
                 **FORMAT_OPTS["plain"], **FMTS[fmt]):
        ptr, col, val, x = long_row_csr(32001, PER_ROW[lanes], 16, seed=20 * lanes)
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        assert c.A.plan()["lanes"] == lanes and c.A.narrow() == (16 if fmt == "col16" else 0)
        assert partial_chunks(c, lanes) > c.p["nblocks"] // 4 and decoupled(c, lanes)
        xs, r, n = fused_first_sweep(ctx, c)
        assert n == 1, "the first sweep was not fused into the residual"
        assert np.array_equal(xs, (OMEGA * c.d) * c.f)
        S, M = acc.row_sums(ptr, col, c.val, xs)
        acc.assert_rows(r, c.f - S, acc.bound("resid", c.m, c.k, acc.U64, M, f=c.f), "%s lanes=%d fused sweep"
                        % (fmt, lanes), ptr, c.p)
        xs0, r0, _ = on_variant(ctx, 0, lambda: fused_first_sweep(ctx, c))
        np.testing.assert_array_equal(xs, xs0)
        np.testing.assert_array_equal(r, r0)


@pytest.mark.parametrize("lanes,per", [(1, 30), (2, 30), (4, 50), (16, 200), (32, 400)])
def test_long_blocks_between_short_ones(ctx, lanes, per):
    """A plain operator whose long blocks (reduced by the whole CTA) sit between staged ones of
    a few chunks each: the stream drains to each long block and carries on after it."""
    with options(ctx, lanes=lanes, spmv_variant=1, **FORMAT_OPTS["plain"], narrow_columns=1):
        ptr, col, val, x = long_row_csr(12001, per, 16, seed=70 + lanes, long_rows=6)
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        assert c.A.plan()["lanes"] == lanes and c.A.plan()["long_blocks"] >= 2
        assert c.A.narrow() == 0 and decoupled(c, lanes)
        modes_match_block_kernel(ctx, c, "long blocks lanes=%d" % lanes)


@pytest.mark.parametrize("fmt", ["plain", "col24"])
def test_default_ring_is_walked(ctx, fmt):
    """At the default stages and CTAs per SM every CTA walks more than 2 * stages blocks, so every
    stage is refilled and its mbarrier's parity flips while warps are spread over the ring."""
    stages, ctas = ctx.get_option("stages"), ctx.get_option("ctas_per_sm")
    knobs = (stages, ctas, ctx.get_option("nnz_cap"))
    with options(ctx, lanes=2, spmv_variant=1, **FORMAT_OPTS["plain"], **FMTS[fmt]):
        ptr, col, val, x = sized(lambda nr: long_row_csr(nr, 30, 24, seed=nr), knobs, 2, 1)
        c = Case(ctx, ptr, col, val, x, seed=3)
        blocks = c.A.plan()["blocks"]
        grid = min(blocks, sms() * ctas)
        assert -(-blocks // grid) > 2 * stages, (blocks, grid, stages)
        assert decoupled(c, 2)
        if fmt == "col24":
            assert c.A.narrow() == 24
        modes_match_block_kernel(ctx, c, "default ring %s" % fmt)


def test_in_kernel_scalars_are_deterministic(ctx):
    with options(ctx, lanes=2, spmv_variant=1, coarse_tail=0, **FORMAT_OPTS["plain"], narrow_columns=1):
        ptr, col, val, x = long_row_csr(90001, 30, 24, seed=5)
        c = Case(ctx, ptr, col, val, x, seed=5)
        assert c.A.narrow() == 24 and partial_chunks(c, 2) > 0 and decoupled(c, 2)
        p = np.random.default_rng(9).uniform(-1, 1, c.nr)
        runs = [(cg_step(ctx, c, p)[1], sweep_dot(ctx, c)[1]) for _ in range(3)]
        assert all(r == runs[0] for r in runs), runs
