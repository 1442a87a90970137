"""Coarsest levels above 16384 rows: the banded-LU coarse solver on the device, against an
extended-precision solution, the reference's skyline LU and the live reference solver."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import amgcl_b200 as ab
import oracle
import _accuracy as acc
from _accuracy import LD
from conftest import TOL_RESID_REL, TOL_SOLUTION, rel_err
from test_gpu_accuracy import F32, F64, _coarse_f32, dvec, get
from test_coarse_lu import C_LU, poisson2d, shuffled

pytestmark = pytest.mark.gpu

DENSE_MAX = 16384


def kappa_inf(A, lu):
    """||A||inf * ||A^-1||inf, the second factor by Higham's 1-norm estimator on A^-T (exact for
    most matrices, a lower bound at worst; the bound below has orders of magnitude to spare)."""
    n = A.shape[0]
    inv_t = spla.LinearOperator((n, n), matvec=lambda v: lu.solve(v, trans="T"),
                                rmatvec=lambda v: lu.solve(v))
    return abs(A).sum(axis=1).max() * spla.onenormest(inv_t)


def exact(A, b):
    """Solution of A x = b to well below FP64 rounding: sparse LU plus one refinement step with
    the residual in extended precision."""
    lu = spla.splu(A.tocsc())
    x = lu.solve(b)
    AL = A.tocsr()
    r = b.astype(LD) - sp.csr_matrix((AL.data.astype(LD), AL.indices, AL.indptr), shape=A.shape) @ x.astype(LD)
    return x + lu.solve(np.asarray(r, dtype=F64)), lu


def create(ctx, n, ptr, col, val, dt=F64):
    S = ctx.coarse(n, ptr, col, val) if dt == F64 else _coarse_f32(ctx, n, ptr, col, val)
    info = ab.Coarse.info(S)
    assert info["kind"] == "banded_lu" and info["n"] == n > DENSE_MAX, info
    return S


def check(ctx, A, what, dt=F64, csr=None, seed=0):
    """Solve A x = b with b uniform in [-1, 1] and check ||x^ - x||inf / ||x||inf <= C_LU * n * u *
    kappa_inf(A) (C_LU and its justification: test_coarse_lu.py).  FP32 vectors: the factor is
    formed in FP64 from the FP32-rounded matrix and x is rounded once at the store, so one FP32
    rounding is added."""
    A = A.tocsr()
    n = A.shape[0]
    ptr, col, val = csr if csr is not None else (A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data)
    b = np.random.default_rng(seed).uniform(-1, 1, n)
    S = create(ctx, n, ptr, col, val, dt)
    vb, vx = dvec(ctx, b, dt), dvec(ctx, np.zeros(n), dt)
    ctx.coarse_solve(S, vb, vx)
    got = get(vx, dt).astype(F64)
    A_ = A.astype(dt).astype(F64)
    x, lu = exact(A_, b.astype(dt).astype(F64))
    kappa = kappa_inf(A_, lu)
    err = np.abs(got - x).max() / np.abs(x).max()
    bnd = C_LU * n * acc.U64 * kappa + (acc.U32 if dt == F32 else 0.0)
    assert err <= bnd, "%s: error %.3g > bound %.3g (kappa %.3g)" % (what, err, bnd, kappa)
    return S, b, got, bnd


def poisson3d_sp(m, convection=0.0):
    ptr, col, val, _ = ab.poisson3d(m, convection=convection)
    n = ptr.size - 1
    return sp.csr_matrix((val, col, ptr), shape=(n, n))


def test_poisson2d(ctx):
    check(ctx, poisson2d(130), "2-D Poisson 130^2")


def test_poisson3d(ctx):
    check(ctx, poisson3d_sp(26), "3-D Poisson 26^3")


def test_convection_diffusion(ctx):
    check(ctx, poisson3d_sp(26, convection=1.0), "3-D convection-diffusion 26^3")


def test_duplicates_and_unsorted_rows(ctx):
    A = poisson2d(131)
    ptr, col, val = shuffled(A, 5)
    # every entry as two halves, the halves apart (the upload sums duplicates)
    n = A.shape[0]
    cnt = np.diff(ptr)
    ptr2 = np.concatenate([[0], np.cumsum(2 * cnt)]).astype(np.int64)
    col2 = np.empty(2 * col.size, dtype=np.int64)
    val2 = np.empty(2 * col.size)
    for i in range(n):
        s, e = ptr[i], ptr[i + 1]
        col2[ptr2[i]:ptr2[i + 1]] = np.concatenate([col[s:e], col[s:e][::-1]])
        val2[ptr2[i]:ptr2[i + 1]] = np.concatenate([val[s:e] / 2, (val[s:e] / 2)[::-1]])
    check(ctx, A, "duplicates + unsorted rows", csr=(ptr2, col2, val2))


def test_fp32_vectors(ctx):
    check(ctx, poisson3d_sp(26, convection=0.5), "FP32 convection-diffusion", dt=F32)


def test_sa_level_against_reference_skyline_lu(ctx):
    """The reference's own level-1 operator of 3-D Poisson 52^3 (smoothed aggregation, about
    17,000 rows), with coarse_enough above it so that the reference's skyline LU solves that
    level too."""
    ptr, col, val, _ = ab.poisson3d(52)
    R = oracle.RefSolver(ptr, col, val, "damped_jacobi", "cg", coarse_enough=20000)
    assert R.nlevels == 2
    n, _, (cp, cc, cv) = R.level_matrix(1, "A")
    A = sp.csr_matrix((cv, cc, cp), shape=(n, n))
    S, b, got, bnd = check(ctx, A, "SA level 1", csr=(cp, cc, cv))
    ref = R.coarse_solve(b)
    x, _ = exact(A, b)
    assert np.abs(ref - x).max() / np.abs(x).max() <= bnd
    assert rel_err(got, ref) <= 2 * bnd
    R.close()


def test_singular_and_zero_pivot(ctx):
    A = poisson2d(130).tolil()
    A[77, :] = 0                                  # an empty row: singular
    A = A.tocsr()
    with pytest.raises(ab.B200Error, match="singular"):
        ctx.coarse(A.shape[0], A.indptr, A.indices, A.data)
    # non-singular, but the 2 x 2 block [[0, 1], [1, 0]] (a component of its own) has a zero
    # pivot without pivoting
    B = sp.block_diag([poisson2d(130), sp.csr_matrix([[0.0, 1.0], [1.0, 0.0]])]).tocsr()
    B.eliminate_zeros()
    L = ab.lib()
    h = ctypes.c_void_p()
    ptr, col = B.indptr.astype(np.int64), B.indices.astype(np.int64)
    rc = L.b200_coarse_create_i64(ctx.h, B.shape[0], ptr.ctypes.data, col.ctypes.data,
                                  B.data.ctypes.data, ctypes.byref(h))
    assert rc == -5 and not h.value, rc          # B200_ESINGULAR


def test_too_large_for_the_device(ctx):
    """A random sparse matrix (an expander: no ordering gives it a small bandwidth) whose factor
    needs more memory than the device has: B200_ENOMEM before anything is allocated."""
    import torch
    n = 300000
    rng = np.random.default_rng(0)
    i = np.repeat(np.arange(n), 3)
    j = rng.integers(0, n, 3 * n)
    R = sp.csr_matrix((np.ones(3 * n), (i, j)), shape=(n, n))
    A = (R + R.T + sp.diags(np.full(n, 10.0))).tocsr()
    plan = ab.coarse_lu_plan(n, A.indptr, A.indices)
    free0, total = torch.cuda.mem_get_info()
    assert plan["factor_bytes"] + plan["setup_bytes"] > total
    L = ab.lib()
    h = ctypes.c_void_p()
    ptr, col = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    rc = L.b200_coarse_create_i64(ctx.h, n, ptr.ctypes.data, col.ctypes.data, A.data.ctypes.data,
                                  ctypes.byref(h))
    assert rc == -3 and not h.value, rc          # B200_ENOMEM
    free1, _ = torch.cuda.mem_get_info()
    assert free1 >= free0 - (4 << 20), (free0, free1)
    check(ctx, poisson2d(130), "after the refusal")


def test_graph_replay_and_repeated_solves_are_bit_identical(ctx):
    A = poisson3d_sp(26, convection=1.0)
    n = A.shape[0]
    S = create(ctx, n, A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data)
    b = np.random.default_rng(3).uniform(-1, 1, n)
    vb, vx = ctx.vector(b), ctx.vector(n)
    ctx.coarse_solve(S, vb, vx)
    first = vx.numpy()
    for _ in range(3):                            # every launch is a new epoch of the sweeps
        vx2 = ctx.vector(n)
        ctx.coarse_solve(S, vb, vx2)
        assert np.array_equal(vx2.numpy(), first)
    vy = ctx.vector(np.zeros(n))                  # (no pending lazy clear: replays need the entry state)
    assert ctx.graph_begin()
    ctx.coarse_solve(S, vb, vy)
    g = ctx.graph_end()                           # runs once
    assert np.array_equal(vy.numpy(), first)
    for _ in range(3):
        assert g.launch()
        assert np.array_equal(vy.numpy(), first)
        ctx.coarse_solve(S, vb, vx)               # direct launches between replays
        assert np.array_equal(vx.numpy(), first)
    g.close()


def test_profile_shows_the_lu_sweeps_only(ctx):
    from torch.profiler import ProfilerActivity, profile
    A = poisson2d(130)
    n = A.shape[0]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        S = create(ctx, n, A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data)
        vb, vx = ctx.vector(np.ones(n)), ctx.vector(n)
        ctx.coarse_solve(S, vb, vx)
        ctx.sync()
    names = {e.name for e in prof.events() if e.device_type.name == "CUDA"}
    assert any("coarse_lu_sweep_kernel" in k for k in names), sorted(names)[:20]
    assert any("lu_step_kernel" in k for k in names)
    assert not any(g in k for k in names for g in ("coarse_pivot", "coarse_eliminate", "coarse_gemv"))
    ctx.profile_begin()
    ctx.coarse_solve(S, vb, vx)
    modes = {e["mode"]: e for e in ctx.profile_end()}
    assert "coarse_lu" in modes and "coarse_gemv" not in modes
    assert modes["coarse_lu"]["nrows"] == n


# ---------------------------------------------------------------------------------------------
# end to end: AMGCL's own solvers on the b200 backend with coarse_enough above the coarsest level
# ---------------------------------------------------------------------------------------------
COARSE_ENOUGH = 40000


@pytest.fixture(scope="module")
def poisson400():
    A = poisson2d(400)                          # smoothed aggregation: level 1 has 26,800 rows
    ptr, col = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    return ptr, col, A.data, np.ones(A.shape[0])


@pytest.mark.parametrize("relax,krylov,precision", [("damped_jacobi", "cg", "f64"),
                                                    ("spai0", "bicgstab", "f64"),
                                                    ("damped_jacobi", "cg", "mixed")])
def test_dropin_against_live_reference(ctx, poisson400, relax, krylov, precision):
    ptr, col, val, rhs = poisson400
    R = oracle.RefSolver(ptr, col, val, relax, krylov, coarse_enough=COARSE_ENOUGH, precision=precision)
    if precision == "f64":                      # (the mixed-precision reference keeps its levels to itself)
        assert R.nlevels == 2
        n1, _, _ = R.level_matrix(1, "A")
        assert DENSE_MAX < n1 <= COARSE_ENOUGH
    xr, itr, resr = R.solve(rhs)
    S = ab.DropinSolver(ptr, col, val, relax, krylov, coarse_enough=COARSE_ENOUGH, ctx=ctx,
                        precision=precision)
    x, it, res = S.solve(rhs)
    if precision == "f64":
        assert it == itr, (it, itr)
        assert abs(res - resr) <= TOL_RESID_REL * resr, (res, resr)
        assert rel_err(x, xr) <= TOL_SOLUTION
    else:
        # the reference's FP32 hierarchy factors the coarsest level in FP32, this one in FP64
        # (as the dense inverse does), and FP32 rounding differs elsewhere too: FP32-sized
        # tolerances, as in test_gpu_solver.py's mixed-precision parity test
        assert abs(it - itr) <= 1, (it, itr)
        A = sp.csr_matrix((val, col, ptr), shape=(rhs.size, rhs.size))
        assert np.linalg.norm(rhs - A @ x) / np.linalg.norm(rhs) < 2e-8
        assert abs(np.linalg.norm(x) - np.linalg.norm(xr)) <= 1e-6 * np.linalg.norm(xr)
    R.close()


def test_dropin_cycle_graph_bit_identical(ctx, poisson400):
    ptr, col, val, rhs = poisson400
    S = ab.DropinSolver(ptr, col, val, "damped_jacobi", "cg", coarse_enough=COARSE_ENOUGH, ctx=ctx)
    G = ab.DropinSolver(ptr, col, val, "damped_jacobi", "cg", coarse_enough=COARSE_ENOUGH, ctx=ctx,
                        graph=True)
    x, it, res = S.solve(rhs)
    for _ in range(2):
        xg, itg, resg = G.solve(rhs)
        assert itg == it and resg == res and np.array_equal(xg, x)
