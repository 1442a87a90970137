import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")

# Stated FP64 tolerances (DESIGN.md "Parity"): the GPU path and the oracle differ
# only in summation order / FMA contraction.
TOL_PRIMITIVE = 1e-13      # relative, per primitive, vs oracle on identical inputs
TOL_RESID_REL = 1e-6       # relative agreement of the final relative residual
TOL_SOLUTION = 1e-8        # ||x - x_ref||_inf / ||x_ref||_inf after a converged solve


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _have_gpu():
    try:
        import amgcl_b200
        return amgcl_b200.lib().b200_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Fixture:
    """A golden hierarchy written by tests/golden/make_golden.py (real reference)."""

    def __init__(self, path):
        z = np.load(path)
        self.z = z
        self.n = int(z["n"])
        self.relax = str(z["relax"])
        self.krylov = str(z["krylov"])
        self.omega = float(z["omega"])
        self.nlevels = int(z["nlevels"])
        self.coarse_enough = int(z["coarse_enough"])
        self.levels = []
        for l in range(self.nlevels - 1):
            lv = {}
            for key in ("A", "P", "R"):
                lv[key] = tuple(z["L%d_%s_%s" % (l, key, nm)] for nm in ("ptr", "col", "val"))
            lv["diag"] = z["L%d_diag" % l]
            self.levels.append(lv)
        self.coarse = tuple(z["C_%s" % nm] for nm in ("ptr", "col", "val"))

    def __getitem__(self, k):
        return self.z[k]


@pytest.fixture(scope="session", params=["poisson12_damped_jacobi_cg", "poisson12_spai0_bicgstab"])
def golden(request):
    return Fixture(os.path.join(GOLDEN, request.param + ".npz"))


@pytest.fixture(scope="session")
def known_answers():
    with open(os.path.join(GOLDEN, "known_answers.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def ctx():
    import amgcl_b200
    c = amgcl_b200.Context(0)
    yield c


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    denom = max(np.abs(b).max(), 1e-300)
    return float(np.abs(a - b).max() / denom)
