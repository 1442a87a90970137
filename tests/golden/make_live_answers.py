"""Write tests/golden/live_answers.npz: the reference's answers for the systems
tests/test_gpu_solver.py solves beside it (random right-hand side and initial guess,
anisotropic / convection-diffusion operators, unstructured graph Laplacians) and the systems
its sample_problem generator makes, so the tests compare with the reference without needing
its build.

Solutions and preconditioner outputs are stored at 256 indices drawn with a fixed seed, with
their max-norm and 2-norm (the full vectors would exceed 1 MB).

    python tests/golden/make_live_answers.py      # needs oracle/_ref (AMGCL's headers)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import oracle                      # noqa: E402
import amgcl_b200 as ab            # noqa: E402

SAMPLES = 256


def sample_index(n):
    return np.sort(np.random.default_rng(0).choice(n, min(n, SAMPLES), replace=False))


def put(out, key, v):
    idx = sample_index(v.size)
    out[key + "_samples"] = v[idx]
    out[key + "_max"] = np.abs(v).max()
    out[key + "_norm2"] = np.linalg.norm(v)


def random_rhs_cases(out):
    for relax, krylov in (("damped_jacobi", "cg"), ("spai0", "bicgstab")):
        ptr, col, val, _ = ab.poisson3d(40)
        rng = np.random.default_rng(7)
        rhs = rng.uniform(-1, 1, ptr.size - 1)
        x0 = rng.uniform(-1, 1, ptr.size - 1)
        R = oracle.RefSolver(ptr, col, val, relax, krylov)
        x, it, res = R.solve(rhs, x0)
        key = "random_%s_%s" % (relax, krylov)
        out[key + "_iters"], out[key + "_resid"] = it, res
        put(out, key + "_x", x)
        put(out, key + "_precond", R.apply_precond(rhs))
        R.close()


def anisotropic_cases(out):
    for a, c, relax, krylov in ANISOTROPIC:
        ptr, col, val, rhs = ab.poisson3d(32, anisotropy=a, convection=c)
        R = oracle.RefSolver(ptr, col, val, relax, krylov)
        x, it, res = R.solve(rhs)
        key = "aniso_%g_%g_%s_%s" % (a, c, relax, krylov)
        out[key + "_iters"], out[key + "_resid"] = it, res
        put(out, key + "_x", x)
        f = np.random.default_rng(3).uniform(-1, 1, rhs.size)
        put(out, key + "_precond", R.apply_precond(f))
        R.close()


def unstructured_cases(out):
    for relax, krylov in (("damped_jacobi", "cg"), ("spai0", "bicgstab")):
        ptr, col, val, rhs = ab.unstructured3d(20000, order="random" if krylov == "cg" else "morton")
        R = oracle.RefSolver(ptr, col, val, relax, krylov)
        x, it, res = R.solve(rhs)
        key = "unstructured_%s_%s" % (relax, krylov)
        out[key + "_nlevels"] = R.nlevels
        out[key + "_iters"], out[key + "_resid"] = it, res
        put(out, key + "_x", x)
        R.close()


def generator_cases(out):
    r = oracle.ref()
    for n, a in GENERATOR:
        for name, v in zip(("ptr", "col", "val", "rhs"), r.sample_problem(n, a)):
            out["sample_problem_%d_%g_%s" % (n, a, name)] = v


GENERATOR = [(1, 1.0), (4, 1.0), (7, 0.5), (6, 2.0), (9, 0.1)]
ANISOTROPIC = [(0.5, 0.0, "damped_jacobi", "cg"), (0.5, 0.0, "spai0", "bicgstab"),
               (1.0, 0.7, "spai0", "bicgstab"), (1.0, 0.7, "damped_jacobi", "gmres"),
               (2.0, 0.3, "spai0", "bicgstab")]


if __name__ == "__main__":
    assert oracle.have_ref(), "needs oracle/_ref/libamgcl_ref.so (built where AMGCL's headers are)"
    out = {"samples": SAMPLES}
    random_rhs_cases(out)
    anisotropic_cases(out)
    unstructured_cases(out)
    generator_cases(out)
    np.savez_compressed(os.path.join(HERE, "live_answers.npz"), **out)
    print("wrote", os.path.join(HERE, "live_answers.npz"), len(out), "arrays")
