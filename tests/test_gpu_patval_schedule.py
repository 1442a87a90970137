"""GPU parity of the value-keyed pattern kernel's schedule (csr_kernels.cuh csr_patval_kernel): it
reduces the rows the ring kernel gives each thread on FMT_PATTERN, in the same order, several at a
time.  Every output vector and every in-kernel scalar (CG's <q, p>, the residual's <r, r>, the
sweep's <rhs, x_new>, BiCGStab's <v, rh>, <t, s> and <t, t>) must have the bits of pattern_values 0
(FMT_PATTERN on the ring, values streamed) -- over the ring knobs that fix the grid and the block
plan, 1, 2 and 4 lanes, blocks that end mid-chunk, fewer blocks than the grid and CTAs that own
one block more than others."""
import numpy as np
import pytest

import amgcl_b200 as ab
from test_gpu_accuracy import KNOBS, sized, sms
from test_gpu_pattern_values import CSR_MODES, PATTERN, options, stencil
from test_gpu_values import all_modes
import _accuracy as acc

pytestmark = pytest.mark.gpu


def offsets(lanes):
    """6 * lanes + 1 entries per interior row; the rows near either end have fewer (boundary
    patterns of other lengths)."""
    return list(range(-3 * lanes, 3 * lanes + 1))


def every_pass(ctx, A, n, seed):
    """MODE 0-4 without scalars, then every pass that leaves one: CG's q = A p with <q, p> (ndot 1
    with w), the residual with <r, r> (ndot 1, w = r), the smoother sweep with <rhs, x_new> while a
    Krylov solver of this size is alive (ndot 1, w = rhs), BiCGStab's v = A p with <v, rh> and
    t = A s with <t, s> and <t, t> (ndot 2)."""
    modes = all_modes(ctx, A, n, seed)
    rng = np.random.default_rng(seed)
    x0, f, d = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.1, 1, n)

    def run():
        out = [modes()]
        K = ab.Krylov(ctx, n)
        vp, vq, vx, vr, vf = ctx.vector(x0), ctx.vector(n), ctx.vector(d), ctx.vector(f), ctx.vector(f)
        K.cg_direction(vr, vr, vp)
        rr = K.cg_step(A, vp, vq, vx, vr)
        s = K.scalars()
        out += [vq.numpy(), vx.numpy(), vr.numpy(), [rr, s["qp"], s["alpha"], s["rr"]]]
        out += [[K.residual(vf, A, vx, vr)], vr.numpy()]
        vs, vt, vd = ctx.vector(x0), ctx.vector(n), ctx.vector(d)
        ctx.relax(A, vf, vs, vt, vd, 0.72)
        out += [vs.numpy(), [ctx.dot(vf, vs)]]
        rhs, x = ctx.vector(f), ctx.vector(x0)
        r, p, v, sv, t, rh, T = (ctx.vector(n) for _ in range(7))
        out += [[K.residual(rhs, A, x, r)]]
        K.bicg_start(r, rh)
        for _ in range(2):
            K.bicg_direction(r, v, p)
            ctx.vmul(1.0, vd, p, 0.0, T)
            ss = K.bicg_step_s(A, rh, T, v, r, sv, x)
            sc = K.scalars()
            out += [v.numpy(), sv.numpy(), [ss, sc["rho"], sc["alpha"]]]
            ctx.vmul(1.0, vd, sv, 0.0, T)
            rr = K.bicg_step_r(A, rh, T, t, sv, r, x)
            sc = K.scalars()
            out += [t.numpy(), x.numpy(), r.numpy(), [rr, sc["ts"], sc["tt"], sc["omega"], sc["rho_next"]]]
        K.close()
        return np.concatenate([np.asarray(o, dtype=np.float64).ravel() for o in out])
    return run


def check(ctx, ptr, col, val, lanes, seed):
    n = ptr.size - 1
    A = ctx.csr(n, n, ptr, col, val)
    assert A.plan()["lanes"] == lanes and A.patterns()["pattern_indexed"]
    run = every_pass(ctx, A, n, seed)
    out, fmts = [], []
    for pv in (1, 0):
        with options(ctx, pattern_values=pv):
            ctx.profile_begin()
            out.append(run())
            fmts.append({p["format"] for p in ctx.profile_end() if p["nnz"] > 0 and p["mode"] in CSR_MODES})
    assert fmts == [{"pattern_values"}, {"pattern"}]
    np.testing.assert_array_equal(out[0], out[1])
    return A


@pytest.mark.parametrize("lanes", [1, 2, 4])
@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: "S%d-C%d-cap%d" % k)
def test_ring_knobs(ctx, knobs, lanes):
    """CTAs per SM (the grid) and nnz_cap (the block plan) as the ring kernel runs them, each CTA
    walking many blocks; the stage count changes nothing for this format.  nrows = 1, 2 or 3 mod 4."""
    stages, ctas, cap = knobs
    i = KNOBS.index(knobs)
    exact = i % 2 == 0                      # the FP32 table, or the FP64 one
    with options(ctx, stages=stages, ctas_per_sm=ctas, nnz_cap=cap, lanes=lanes, narrow_values=1,
                 narrow_values_min_nnz=0, **PATTERN):
        ptr, col, val = sized(lambda nr: stencil(nr, offsets(lanes), exact), knobs, lanes, 1 + i % 3)
        check(ctx, ptr, col, val, lanes, seed=cap + lanes)


def rows_for_blocks(lanes, cap, nblocks, residue):
    """Rows of a stencil operator whose plan has about nblocks blocks, = residue mod 4."""
    starts = acc.plan(stencil(40001, offsets(lanes), True)[0], lanes, cap)["starts"]
    per = int(np.median(np.diff(starts)))
    return 4 * ((nblocks - 1) * per // 4) + residue


# (blocks in units of the grid, extra blocks): fewer blocks than the grid; one block per CTA;
# some CTAs owning one block more than others, with 1, 2, 3 and 4 blocks per CTA (rows per thread
# divisible by two rows per batch, and not)
SHAPES = [(0, 37), (1, 0), (1, 5), (2, 1), (3, 7), (4, -3)]


@pytest.mark.parametrize("lanes", [1, 2, 4])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "g%d%+d" % s)
def test_walk_edges(ctx, shape, lanes):
    """nnz_cap 256: 36-row blocks of 7-entry rows at one lane, so most blocks end mid-chunk and
    the warp that takes a block's first chunk rotates; the grid is 4 CTAs per SM."""
    grid_units, extra = shape
    cap, ctas = 256, 4
    nblocks = grid_units * sms() * ctas + extra
    with options(ctx, ctas_per_sm=ctas, nnz_cap=cap, lanes=lanes, narrow_values=1, narrow_values_min_nnz=0,
                 **PATTERN):
        ptr, col, val = stencil(rows_for_blocks(lanes, cap, nblocks, 1 + lanes % 3), offsets(lanes), lanes != 2)
        A = check(ctx, ptr, col, val, lanes, seed=nblocks)
        assert abs(A.plan()["blocks"] - nblocks) <= 2
