"""GPU end-to-end parity: AMGCL's own make_solver<amg<...>, cg|bicgstab> running on
backend::b200 (the drop-in) against the reference's builtin backend (its answers are stored
under tests/golden/, written by make_golden.py, make_large_answers.py and make_live_answers.py).

Tolerances (DESIGN.md): equal iteration count, final relative residual within 1e-6
relative, ||x - x_ref||_inf / ||x_ref||_inf <= 1e-8."""
import os

import numpy as np
import pytest

import amgcl_b200 as ab
import oracle
from conftest import GOLDEN, rel_err, TOL_RESID_REL, TOL_SOLUTION

pytestmark = pytest.mark.gpu

LIVE = np.load(os.path.join(GOLDEN, "live_answers.npz"))


def live_err(key, v):
    """max |v - v_ref| / max |v_ref| over the stored samples of the reference's vector `key`
    (tests/golden/make_live_answers.py), and the relative difference of the 2-norms."""
    idx = np.sort(np.random.default_rng(0).choice(v.size, min(v.size, int(LIVE["samples"])), replace=False))
    err = float(np.abs(v[idx] - LIVE[key + "_samples"]).max() / LIVE[key + "_max"])
    return max(err, abs(float(np.linalg.norm(v)) - float(LIVE[key + "_norm2"])) / float(LIVE[key + "_norm2"]))

CONFIGS = [("damped_jacobi", "cg"), ("spai0", "bicgstab"), ("spai0", "cg"),
           ("damped_jacobi", "bicgstab")]


def test_dropin_matches_golden_fixture(ctx, golden):
    """Same hierarchy parameters as the fixture (coarse_enough=100 -> 3 levels)."""
    ptr, col, val, rhs = ab.poisson3d(golden.n)
    S = ab.DropinSolver(ptr, col, val, golden.relax, golden.krylov,
                        coarse_enough=golden.coarse_enough, ctx=ctx)
    x, iters, resid = S.solve(rhs)
    assert iters == int(golden["iters"])
    assert abs(resid - float(golden["resid"])) <= TOL_RESID_REL * float(golden["resid"])
    assert rel_err(x, golden["x"]) < TOL_SOLUTION
    # one V-cycle on a seeded vector
    assert rel_err(S.apply_precond(golden["in_a"]), golden["precond_a"]) < 1e-11
    rep = S.report()
    assert "Number of levels:    %d" % golden.nlevels in rep
    S.close()


@pytest.mark.parametrize("n", [16, 32, 64])
@pytest.mark.parametrize("relax,krylov", CONFIGS)
def test_dropin_matches_known_answers(ctx, known_answers, n, relax, krylov):
    """Configs #1 of BASELINE.json (64^3) and smaller: iterations / residual / solution
    samples recorded from the reference (tests/golden/known_answers.json)."""
    case = [c for c in known_answers["cases"]
            if (c["n"], c["relax"], c["krylov"]) == (n, relax, krylov)][0]
    ptr, col, val, rhs = ab.poisson3d(n)
    S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
    x, iters, resid = S.solve(rhs)
    assert iters == case["iters"]
    assert abs(resid - case["resid"]) <= TOL_RESID_REL * case["resid"]
    assert abs(x[0] - case["x_first"]) <= TOL_SOLUTION * abs(case["x_first"])
    assert abs(x[x.size // 2] - case["x_mid"]) <= TOL_SOLUTION * abs(case["x_mid"])
    assert abs(np.linalg.norm(x) - case["x_norm2"]) <= TOL_SOLUTION * case["x_norm2"]
    # true residual of the returned solution (size-independent property)
    r = rhs - oracle.c().spmv(1.0, (ptr, col, val), x, 0.0, np.zeros_like(x))
    assert np.linalg.norm(r) / np.linalg.norm(rhs) < 2e-8
    S.close()


@pytest.mark.parametrize("relax,krylov", CONFIGS[:2])
def test_dropin_vs_live_reference_random_rhs(ctx, relax, krylov):
    n = 40
    ptr, col, val, _ = ab.poisson3d(n)
    rng = np.random.default_rng(7)
    rhs = rng.uniform(-1, 1, ptr.size - 1)
    x0 = rng.uniform(-1, 1, ptr.size - 1)
    key = "random_%s_%s" % (relax, krylov)
    itr, resr = int(LIVE[key + "_iters"]), float(LIVE[key + "_resid"])
    S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
    xg, itg, resg = S.solve(rhs, x0)
    assert itg == itr
    assert abs(resg - resr) <= TOL_RESID_REL * resr
    assert live_err(key + "_x", xg) < TOL_SOLUTION
    # the preconditioner alone
    assert live_err(key + "_precond", S.apply_precond(rhs)) < 1e-10
    S.close()


@pytest.mark.parametrize("anisotropy,convection,relax,krylov", [
    (0.5, 0.0, "damped_jacobi", "cg"), (0.5, 0.0, "spai0", "bicgstab"),
    (1.0, 0.7, "spai0", "bicgstab"), (1.0, 0.7, "damped_jacobi", "gmres"),
    (2.0, 0.3, "spai0", "bicgstab")])
def test_anisotropic_and_nonsymmetric_systems_vs_live_reference(ctx, anisotropy, convection, relax, krylov):
    """tests/sample_problem.hpp's anisotropy parameter (different strength-of-connection
    pattern, hence different aggregates and coarse stencils) and a non-symmetric
    convection-diffusion operator: hierarchy shape, iteration count, residual and solution
    against the reference running on the same host."""
    n = 32
    ptr, col, val, rhs = ab.poisson3d(n, anisotropy=anisotropy, convection=convection)
    key = "aniso_%g_%g_%s_%s" % (anisotropy, convection, relax, krylov)
    itr, resr = int(LIVE[key + "_iters"]), float(LIVE[key + "_resid"])
    S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
    xg, itg, resg = S.solve(rhs)
    assert itg == itr
    tol = 1e-4 if krylov == "bicgstab" else TOL_RESID_REL      # BiCGStab amplifies rounding
    assert abs(resg - resr) <= tol * resr
    assert live_err(key + "_x", xg) < TOL_SOLUTION
    true_res = np.linalg.norm(rhs - oracle.c().spmv(1.0, (ptr, col, val), xg, 0.0, np.zeros_like(rhs)))
    assert true_res <= 2e-8 * np.linalg.norm(rhs)
    rng = np.random.default_rng(3)
    f = rng.uniform(-1, 1, rhs.size)
    assert live_err(key + "_precond", S.apply_precond(f)) < 1e-10
    S.close()


@pytest.mark.parametrize("krylov,graph,iters", [("cg", "", 14), ("bicgstab", "", 8), ("bicgstab", "graph", 8)])
def test_tutorial_program_runs(known_answers, krylov, graph, iters):
    """examples/poisson_b200.cpp (the reference tutorial with the backend typedef switched,
    compiled with plain g++) on 64^3: the iteration counts of the reference."""
    import subprocess
    from amgcl_b200 import build
    exe = build.build_example()
    case = [c for c in known_answers["cases"]
            if (c["n"], c["relax"], c["krylov"]) == (64, "spai0", krylov)]
    if case:
        assert case[0]["iters"] == iters
    out = subprocess.run([exe, "64", krylov] + ([graph] if graph else []), stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:]
    assert "Iterations: %d" % iters in out.stdout, out.stdout[-2000:]
    assert "Number of levels" in out.stdout          # the reference's own hierarchy report


def test_driver_smoke_entry_point():
    """__graft_entry__.smoke(): the call the driver makes on the GPU box before the bench."""
    import __graft_entry__
    __graft_entry__.smoke()


def test_zero_rhs(ctx):
    ptr, col, val, rhs = ab.poisson3d(12)
    S = ab.DropinSolver(ptr, col, val, ctx=ctx)
    x, iters, resid = S.solve(np.zeros_like(rhs), x0=np.ones_like(rhs))
    assert iters == 0 and resid == 0.0 and not x.any()      # cg.hpp:162-169
    S.close()


def test_resident_path_equals_host_path(ctx):
    ptr, col, val, rhs = ab.poisson3d(24)
    S = ab.DropinSolver(ptr, col, val, ctx=ctx)
    x1, it1, r1 = S.solve(rhs)
    S.upload_rhs(rhs)
    it2, r2 = S.solve_resident()
    assert (it1, r1) == (it2, r2)
    assert np.array_equal(S.download_x(), x1)
    S.close()


@pytest.mark.parametrize("fused_krylov", [0, 1])
def test_variants_and_fusion_agree(ctx, fused_krylov):
    """Kernel scheduling variants and the fused / unfused smoother give the same solve.  With
    the reference's Krylov sequence (fused_krylov = 0) every variant reduces its inner products
    with the same kernel, so the agreement is to rounding of the row sums only; with the fused
    Krylov steps the variants that cannot reduce inside the streaming kernel (variant 0) use the
    stand-alone reduction, i.e. another summation order: the stated end-to-end tolerances."""
    ptr, col, val, rhs = ab.poisson3d(32)
    results = []
    try:
        ctx.set_option("fused_krylov", fused_krylov)
        for variant, fuse, shortcut in ((1, 1, 1), (0, 1, 1), (1, 0, 1), (1, 1, 0)):
            ctx.set_option("spmv_variant", variant)
            ctx.set_option("fuse_relax", fuse)
            ctx.set_option("zero_shortcut", shortcut)
            S = ab.DropinSolver(ptr, col, val, ctx=ctx)
            results.append(S.solve(rhs))
            S.close()
    finally:
        ctx.set_option("spmv_variant", 1)
        ctx.set_option("fuse_relax", 1)
        ctx.set_option("zero_shortcut", 1)
        ctx.set_option("fused_krylov", 1)
    x0, it0, r0 = results[0]
    for x, it, r in results[1:]:
        assert it == it0
        if fused_krylov:
            assert abs(r - r0) <= TOL_RESID_REL * r0 and rel_err(x, x0) < TOL_SOLUTION
        else:
            assert abs(r - r0) <= 1e-9 * r0 and rel_err(x, x0) < 1e-12


@pytest.mark.parametrize("n", [12, 32, 64])
@pytest.mark.parametrize("relax,krylov", [("damped_jacobi", "cg"), ("spai0", "bicgstab")])
def test_coarse_tail_is_bit_transparent(ctx, n, relax, krylov):
    """Option "coarse_tail": calls on small operators are deferred and run as ONE cooperative
    kernel (device-wide barriers instead of kernel boundaries).  Same arithmetic in the same
    order: the solve and the V-cycle alone must give the same bits, with fewer launches."""
    ptr, col, val, rhs = ab.poisson3d(n)
    rng = np.random.default_rng(11)
    f = rng.uniform(-1, 1, rhs.size)
    out = {}
    try:
        for tail in (0, 1):
            ctx.set_option("coarse_tail", tail)
            S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
            S.solve(rhs)
            l0, t0 = ctx.launches, ctx.tail_stats()
            x, it, res = S.solve(rhs)
            l1, t1 = ctx.launches, ctx.tail_stats()
            out[tail] = (x, it, res, S.apply_precond(f), l1 - l0, t1[0] - t0[0], t1[1] - t0[1])
            S.close()
    finally:
        ctx.set_option("coarse_tail", 0)
    (x0, it0, r0, m0, l0, f0, c0), (x1, it1, r1, m1, l1, f1, c1) = out[0], out[1]
    assert (it1, r1) == (it0, r0) and np.array_equal(x1, x0) and np.array_equal(m1, m0)
    assert f0 == 0 and c0 == 0 and f1 >= it1 and c1 >= f1
    if n >= 32:
        assert c1 >= 3 * f1 and l1 < l0                               # several calls per tail launch


@pytest.mark.parametrize("relax,krylov", [("damped_jacobi", "cg"), ("spai0", "bicgstab")])
def test_first_sweep_fusion_is_bit_transparent(ctx, relax, krylov):
    """Option "fuse_first_sweep": the smoother's sweep from x = 0 is postponed and done on the
    fly by the residual that follows it (one pass over A instead of an element-wise kernel + a
    pass).  Same arithmetic: same bits, one launch less per level and cycle."""
    ptr, col, val, rhs = ab.poisson3d(32)
    rng = np.random.default_rng(13)
    f = rng.uniform(-1, 1, rhs.size)
    out = {}
    try:
        for fuse in (0, 1):
            ctx.set_option("fuse_first_sweep", fuse)
            S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
            S.solve(rhs)
            l0 = ctx.launches
            x, it, res = S.solve(rhs)
            out[fuse] = (x, it, res, S.apply_precond(f), ctx.launches - l0)
            S.close()
    finally:
        ctx.set_option("fuse_first_sweep", 1)
    (x0, it0, r0, m0, l0), (x1, it1, r1, m1, l1) = out[0], out[1]
    assert (it1, r1) == (it0, r0) and np.array_equal(x1, x0) and np.array_equal(m1, m0)
    cycles = it0 * (2 if krylov == "bicgstab" else 1)
    assert l0 - l1 >= cycles                     # at least the finest level, every cycle


@pytest.mark.parametrize("relax,krylov,n", [("damped_jacobi", "cg", 32), ("spai0", "bicgstab", 48)])
def test_small_operator_kernel_is_bit_transparent(ctx, relax, krylov, n):
    """Option "small_kernel_max_nnz": operators below the threshold are applied by the
    direct-load kernel instead of the TMA ring pipeline -- same lanes per row, same entry
    order, same shuffle tree, same epilogue: the same bits."""
    ptr, col, val, rhs = ab.poisson3d(n)
    rng = np.random.default_rng(15)
    f = rng.uniform(-1, 1, rhs.size)
    out = {}
    try:
        for cap in (0, 1000000):
            ctx.set_option("small_kernel_max_nnz", cap)
            S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
            x, it, res = S.solve(rhs)
            out[cap] = (x, it, res, S.apply_precond(f))
            S.close()
    finally:
        ctx.set_option("small_kernel_max_nnz", 0)
    (x0, it0, r0, m0), (x1, it1, r1, m1) = out[0], out[1000000]
    assert (it1, r1) == (it0, r0) and np.array_equal(x1, x0) and np.array_equal(m1, m0)


def test_pending_first_sweep_is_materialised_by_any_other_reader(ctx):
    ptr, col, val, _ = ab.poisson3d(10)
    n = ptr.size - 1
    import scipy.sparse as sp
    M = sp.csr_matrix((val, col, ptr), shape=(n, n))
    rng = np.random.default_rng(14)
    f, g = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    d = 1.0 / M.diagonal()
    A = ctx.csr(n, n, ptr, col, val)
    vf, vg, vd, x, tmp, r = ctx.vector(f), ctx.vector(g), ctx.vector(d), ctx.vector(n), ctx.vector(n), ctx.vector(n)
    x1 = 0.72 * d * f
    # the matching residual: fused
    ctx.clear(x); ctx.relax(A, vf, x, tmp, vd, 0.72)
    before = ctx.launches
    ctx.residual(vf, A, x, r)
    assert ctx.launches == before + 1
    assert rel_err(r.numpy(), f - M @ x1) < 1e-13 and rel_err(x.numpy(), x1) < 1e-15
    # some other reader first: the sweep is written out by its own kernel
    ctx.clear(x); ctx.relax(A, vf, x, tmp, vd, 0.72)
    assert abs(ctx.dot(x, x) - x1 @ x1) <= 1e-13 * (x1 @ x1)
    # a residual against ANOTHER right-hand side: not the fused pass, still right
    ctx.clear(x); ctx.relax(A, vf, x, tmp, vd, 0.72)
    ctx.residual(vg, A, x, r)
    assert rel_err(r.numpy(), g - M @ x1) < 1e-13
    # cleared again before anybody looked
    ctx.clear(x); ctx.relax(A, vf, x, tmp, vd, 0.72)
    ctx.clear(x)
    assert not x.numpy().any()


def test_deferred_calls_keep_call_order(ctx):
    """Deferred (small-operator) calls interleaved with immediate ones and with host reads."""
    ptr, col, val, _ = ab.poisson3d(10)
    n = ptr.size - 1
    import scipy.sparse as sp
    M = sp.csr_matrix((val, col, ptr), shape=(n, n))
    rng = np.random.default_rng(12)
    a, b = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    A = ctx.csr(n, n, ptr, col, val)
    va, vb, vy, vz = ctx.vector(a), ctx.vector(b), ctx.vector(n), ctx.vector(n)
    ctx.set_option("coarse_tail", 1)
    try:
        before = ctx.tail_stats()
        ctx.spmv(1.0, A, va, 0.0, vy)          # deferred
        ctx.residual(vb, A, vy, vz)            # deferred, reads the deferred result
        ctx.axpby(2.0, vz, 1.0, vy)            # immediate: flushes first
        ctx.spmv(1.0, A, vy, 1.0, vz)          # deferred again (beta != 0)
        got = vz.numpy()                       # host read: flushes
    finally:
        ctx.set_option("coarse_tail", 0)
    y = M @ a
    z = b - M @ y
    y = 2.0 * z + y
    want = M @ y + z
    assert rel_err(got, want) < 1e-12
    after = ctx.tail_stats()
    assert after[0] - before[0] == 2 and after[1] - before[1] == 3


def test_dependent_launch_is_bit_transparent(ctx):
    """Programmatic dependent launch only changes when kernels are scheduled: the solve with
    and without it must be bit-identical (same arithmetic, same order)."""
    ptr, col, val, rhs = ab.poisson3d(48)
    out = []
    try:
        for pdl in (1, 0, 1):
            ctx.set_option("pdl", pdl)
            for relax, krylov in (("damped_jacobi", "cg"), ("spai0", "bicgstab")):
                S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
                for _ in range(3):           # repeated solves: back-to-back kernel chains
                    out.append((pdl, relax, S.solve(rhs)))
                S.close()
    finally:
        ctx.set_option("pdl", 1)
    base = {r: (x, it, res) for p, r, (x, it, res) in out if p == 0}
    for p, r, (x, it, res) in out:
        x0, it0, res0 = base[r]
        assert it == it0 and res == res0 and np.array_equal(x, x0), (p, r)


@pytest.mark.parametrize("relax,krylov,precision", [
    ("damped_jacobi", "cg", "f64"), ("spai0", "bicgstab", "f64"), ("spai0", "cg", "f64"),
    ("damped_jacobi", "bicgstab", "f64"), ("damped_jacobi", "cg", "mixed"),
    ("spai0", "bicgstab", "mixed"), ("damped_jacobi", "gmres", "f64")])
def test_cycle_graph_wrapper_is_bit_transparent(ctx, relax, krylov, precision):
    """amgcl::preconditioner::b200_cycle_graph<amg<...>> (every V-cycle one CUDA graph launch)
    gives the very same iterates as the unwrapped hierarchy: same kernels, same arguments."""
    ptr, col, val, rhs = ab.poisson3d(40)
    rng = np.random.default_rng(5)
    rhs2 = rng.uniform(-1, 1, rhs.size)
    plain = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx, precision=precision)
    graphed = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx, precision=precision, graph=True)
    assert plain.graph_stats() == (0, 0, 0)
    for b in (rhs, rhs2, rhs):
        l0 = ctx.launches
        x0, it0, r0 = plain.solve(b)
        l1 = ctx.launches
        x1, it1, r1 = graphed.solve(b)
        l2 = ctx.launches
        assert (it1, r1) == (it0, r0) and np.array_equal(x1, x0)
        assert l2 - l1 >= l1 - l0                   # replays count the kernels they contain
                                                    # (recorded calls are never deferred/merged)
    ngraphs, kernels, replays = graphed.graph_stats()
    assert 1 <= ngraphs <= 64 and kernels >= 6
    if krylov != "gmres":                           # GMRES permutes its basis storage: few hits
        assert replays >= it0
    # the preconditioner alone, and the wrapper switched off at run time
    f = rng.uniform(-1, 1, rhs.size)
    assert np.array_equal(graphed.apply_precond(f), plain.apply_precond(f))
    ctx.set_option("cycle_graph", 0)
    try:
        x2, it2, r2 = graphed.solve(rhs)
    finally:
        ctx.set_option("cycle_graph", 1)
    assert (it2, r2) == (it0, r0) and np.array_equal(x2, x0)
    plain.close()
    graphed.close()


def test_large_problem_size_independent_properties(ctx):
    """128^3 (2.1M rows): survey iteration count, true residual, linearity of the V-cycle."""
    n = 128
    ptr, col, val, rhs = ab.poisson3d(n)
    S = ab.DropinSolver(ptr, col, val, "damped_jacobi", "cg", ctx=ctx)
    x, iters, resid = S.solve(rhs)
    assert iters == 21                                     # BASELINE.md section 2
    assert abs(resid - 6.07447143094944e-09) <= TOL_RESID_REL * 6.07447143094944e-09
    A = ctx.csr(n ** 3, n ** 3, ptr, col, val)
    vx, vf, vr = ctx.vector(x), ctx.vector(rhs), ctx.vector(n ** 3)
    ctx.residual(vf, A, vx, vr)
    assert np.sqrt(ctx.dot(vr, vr)) / np.sqrt(ctx.dot(vf, vf)) < 2e-8
    rng = np.random.default_rng(5)
    u, v = rng.uniform(-1, 1, n ** 3), rng.uniform(-1, 1, n ** 3)
    Mu, Mv, Muv = S.apply_precond(u), S.apply_precond(v), S.apply_precond(2.0 * u - 3.0 * v)
    assert rel_err(Muv, 2.0 * Mu - 3.0 * Mv) < 1e-12        # the V-cycle is a linear operator
    S.close()


@pytest.mark.parametrize("n", [16, 32, 48])
@pytest.mark.parametrize("relax,krylov", [("chebyshev", "cg"), ("damped_jacobi", "gmres"),
                                          ("spai0", "bicgstabl"), ("ilu0", "bicgstab"), ("ilu0", "cg")])
def test_components_that_only_use_the_primitives(ctx, known_answers, n, relax, krylov):
    """SURVEY 8f rank 4: AMGCL's Chebyshev smoother (relaxation/chebyshev.hpp), GMRES
    (solver/gmres.hpp, via lin_comb -> axpby/axpbypcz), BiCGStab(L) and the ILU(0) smoother
    (relaxation/ilu0.hpp; triangular solves as damped Jacobi sweeps,
    relaxation/detail/ilu_solve.hpp:97-113 -- the goldens come from the same generic code
    path on a non-builtin CPU backend) run unmodified on the backend through spmv / residual /
    vmul / axpby / axpbypcz / inner_product alone."""
    case = [c for c in known_answers["primitive_only"]
            if (c["n"], c["relax"], c["krylov"]) == (n, relax, krylov)][0]
    ptr, col, val, rhs = ab.poisson3d(n)
    S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
    x, iters, resid = S.solve(rhs)
    assert iters == case["iters"]
    assert abs(resid - case["resid"]) <= 1e-5 * case["resid"]
    assert abs(np.linalg.norm(x) - case["x_norm2"]) <= TOL_SOLUTION * case["x_norm2"]
    assert abs(x[0] - case["x_first"]) <= TOL_SOLUTION * abs(case["x_first"])
    S.close()


def test_multi_gpu_parity_when_two_devices_are_present():
    """Row-partitioned solve (NCCL and peer-memory transports) vs the reference's answers;
    needs >= 2 GPUs, otherwise skipped (tools/dist_check.py is the same check for 4 / 8)."""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                          "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
                          "29541", os.path.join(root, "tools", "dist_check.py"), "32"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert "DIST_CHECK PASS" in out.stdout, out.stdout[-2000:]


@pytest.mark.parametrize("n", [16, 32, 64])
@pytest.mark.parametrize("relax,krylov", CONFIGS)
def test_mixed_precision_matches_reference_mixed(ctx, known_answers, n, relax, krylov):
    """SURVEY 8f rank 2: FP32 hierarchy (amg<backend::b200<float>>) under an FP64 Krylov solver,
    against the reference's own mixed composition amg<builtin<float>> + builtin<double>
    (tutorial/1.poisson3Db/poisson3Db.cpp:45-51).  FP32 rounding differs between the two
    (summation order, FMA), so the tolerance is FP32-sized: same iteration count (+-1),
    solution within 1e-6 of the reference's, true FP64 residual below 2e-8."""
    case = [c for c in known_answers["mixed"]
            if (c["n"], c["relax"], c["krylov"]) == (n, relax, krylov)][0]
    ptr, col, val, rhs = ab.poisson3d(n)
    S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx, precision="mixed")
    x, iters, resid = S.solve(rhs)
    assert abs(iters - case["iters"]) <= 1
    assert resid < 1e-8
    assert abs(np.linalg.norm(x) - case["x_norm2"]) <= 1e-6 * case["x_norm2"]
    assert abs(x[0] - case["x_first"]) <= 1e-6 * abs(case["x_first"])
    r = rhs - oracle.c().spmv(1.0, (ptr, col, val), x, 0.0, np.zeros_like(x))
    assert np.linalg.norm(r) / np.linalg.norm(rhs) < 2e-8
    S.close()


@pytest.mark.parametrize("relax,krylov", CONFIGS[:2])
def test_unstructured_matrix_vs_live_reference(ctx, relax, krylov):
    """BASELINE.json config #4 class of input (poisson3Db.mtx itself is not available offline):
    an unstructured SPD matrix with ~28 non-zeros per row in random row order.  Irregular rows
    exercise the multi-lane reduction and scattered gathers on every level."""
    ptr, col, val, rhs = ab.unstructured3d(20000, order="random" if krylov == "cg" else "morton")
    key = "unstructured_%s_%s" % (relax, krylov)
    itr, resr = int(LIVE[key + "_iters"]), float(LIVE[key + "_resid"])
    S = ab.DropinSolver(ptr, col, val, relax, krylov, ctx=ctx)
    xg, itg, resg = S.solve(rhs)
    assert int(LIVE[key + "_nlevels"]) >= 3
    assert "Number of levels:    %d" % int(LIVE[key + "_nlevels"]) in S.report()
    assert itg == itr
    # CG's residual norm is a smooth function of the rounding; BiCGStab's final value is not
    # (the reference itself moves in the 2nd-3rd digit with the OpenMP thread count on these
    # irregular matrices), so for it the solution and the true residual carry the check
    assert abs(resg - resr) <= (1e-5 if krylov == "cg" else 5e-2) * resr
    assert live_err(key + "_x", xg) < TOL_SOLUTION
    r = rhs - oracle.c().spmv(1.0, (ptr, col, val), xg, 0.0, np.zeros_like(xg))
    assert np.linalg.norm(r) / np.linalg.norm(rhs) < 2e-8
    S.close()
