"""CPU: the C-ABI library loads, exports every declared symbol, refuses to run
without a device (no CPU fallback), and its pure-host logic (row-block plan) is right."""
import ctypes
import os
import re

import numpy as np
import pytest

import amgcl_b200 as ab
import oracle
from amgcl_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "amgcl_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol():
    path = build.build_cuda()
    assert os.path.isfile(path)
    L = ctypes.CDLL(path)
    names = declared_symbols()
    assert len(names) >= 40
    for name in names:
        assert hasattr(L, name), "missing export: " + name


def test_version_and_error_strings():
    L = ab.lib()
    assert b"sm_90a" in L.b200_version()
    assert isinstance(L.b200_last_error(), bytes)


def test_dropin_library_exports():
    D = ab.dropin_lib()
    for name in ("dropin_create", "dropin_solve", "dropin_solve_resident", "dropin_upload_rhs",
                 "dropin_download_x", "dropin_apply_precond", "dropin_report", "dropin_destroy"):
        assert hasattr(D, name)


def test_no_cpu_fallback_without_device():
    L = ab.lib()
    if L.b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(ab.B200Error):
        ab.Context(0)
    h = ctypes.c_void_p()
    rc = L.b200_ctx_create(0, ctypes.byref(h))
    assert rc != 0 and not h.value
    assert L.b200_last_error()
    # the drop-in solver must fail loudly as well, not compute on the CPU
    ptr, col, val, rhs = ab.poisson3d(4)
    with pytest.raises(ab.B200Error):
        ab.DropinSolver(ptr, col, val)


def test_null_arguments_are_rejected():
    L = ab.lib()
    assert L.b200_spmv(None, 1.0, None, None, 0.0, None) == -1
    assert L.b200_vec_size(None, None) == -1
    assert b"null" in L.b200_last_error()


def plan(ptr, lanes=0, nnz_cap=2048):
    L = ab.lib()
    L.b200_plan_i64.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64),
                                ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int),
                                ctypes.POINTER(ctypes.c_int64)]
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    n = ptr.size - 1
    cap = n // 4 + 3
    blk = np.zeros((cap, 2), dtype=np.int32)
    nb, nl = ctypes.c_int64(), ctypes.c_int64()
    ln, rc_ = ctypes.c_int(), ctypes.c_int()
    rc = L.b200_plan_i64(n, ptr.ctypes.data, lanes, nnz_cap, blk.ctypes.data, cap,
                         ctypes.byref(nb), ctypes.byref(ln), ctypes.byref(rc_), ctypes.byref(nl))
    assert rc == 0, L.b200_last_error()
    return blk[:nb.value + 1], ln.value, rc_.value, nl.value


def check_plan(ptr, blk, rows_cap, nnz_cap):
    n = ptr.size - 1
    assert blk[0, 0] == 0 and blk[-1, 0] == n and blk[-1, 1] == ptr[-1]
    rows = blk[:, 0].astype(np.int64)
    assert np.all(np.diff(rows) > 0) or n == 0
    assert np.all(rows[:-1] % 4 == 0), "blocks must start on a 16-byte boundary of ptr"
    assert np.all(blk[:, 1] == ptr[rows]), "first non-zero must equal ptr[first row]"
    assert np.all(np.diff(rows) <= rows_cap)
    nnz = np.diff(blk[:, 1].astype(np.int64))
    too_long = nnz > nnz_cap
    # only a single quad may overflow the stage
    assert np.all(np.diff(rows)[too_long] <= 4)
    return int(too_long.sum())


def test_plan_poisson():
    ptr, col, val, rhs = ab.poisson3d(20)
    blk, lanes, rows_cap, nlong = plan(ptr)
    assert lanes == 1 and rows_cap == 256 and nlong == 0
    assert check_plan(ptr, blk, rows_cap, 2048) == 0
    # 7-pt rows: a block is rows-bound (256 rows ~ 1.8k non-zeros)
    assert np.diff(blk[:, 0]).max() == 256


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_plan_ragged(seed):
    rng = np.random.default_rng(seed)
    n = 4099
    lens = rng.integers(0, 90, n)
    lens[5] = 0
    lens[1000] = 9000            # longer than any stage
    lens[n - 1] = 1
    ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    for lanes in (0, 1, 8, 32):
        for cap in (512, 2048, 6144):
            blk, ln, rows_cap, nlong = plan(ptr, lanes, cap)
            assert nlong == check_plan(ptr, blk, rows_cap, cap) >= 1
            assert rows_cap % 4 == 0 and rows_cap <= 1024


def test_plan_lane_heuristic():
    for avg, want in ((3, 1), (7, 1), (20, 2), (30, 2), (50, 4), (70, 8), (200, 16), (500, 32)):
        ptr = np.arange(0, 1001, dtype=np.int64) * avg
        _, lanes, _, _ = plan(ptr)
        assert lanes == want


def test_plan_empty_and_tiny():
    blk, lanes, rows_cap, nlong = plan(np.zeros(1, dtype=np.int64))
    assert blk.shape[0] == 1 and nlong == 0
    blk, *_ = plan(np.array([0, 2, 2, 5], dtype=np.int64))
    assert blk.tolist() == [[0, 0], [3, 5]]


def test_poisson_generator_matches_reference_counts():
    """tests/sample_problem.hpp: rows n^3, nnz 7n^3 - 6n^2, diag 6, rhs 1."""
    for n in (1, 2, 5, 9):
        ptr, col, val, rhs = ab.poisson3d(n)
        assert ptr.size - 1 == n ** 3 and ptr[-1] == 7 * n ** 3 - 6 * n ** 2
        assert np.all(rhs == 1.0)
        for i in range(n ** 3):
            c = col[ptr[i]:ptr[i + 1]]
            v = val[ptr[i]:ptr[i + 1]]
            assert np.all(np.diff(c) > 0)
            assert v[c == i] == 6.0 and np.all(v[c != i] == -1.0)
    # symmetric
    import scipy.sparse as sp
    ptr, col, val, _ = ab.poisson3d(6)
    A = sp.csr_matrix((val, col, ptr))
    assert abs(A - A.T).max() == 0


def test_poisson_generator_equals_the_reference_generator():
    """bit-for-bit against tests/sample_problem.hpp compiled from the reference, including
    its anisotropy parameter (its output stored by tests/golden/make_live_answers.py)."""
    live = np.load(os.path.join(ROOT, "tests", "golden", "live_answers.npz"))
    for n, a in ((1, 1.0), (4, 1.0), (7, 0.5), (6, 2.0), (9, 0.1)):
        want = [live["sample_problem_%d_%g_%s" % (n, a, name)] for name in ("ptr", "col", "val", "rhs")]
        got = ab.poisson3d(n, anisotropy=a)
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), (n, a)
    # the transport term (not in the reference's generator) keeps the sparsity pattern and
    # an M-matrix, and breaks symmetry
    ptr, col, val, _ = ab.poisson3d(5, convection=0.7)
    p0, c0, v0, _ = ab.poisson3d(5)
    assert np.array_equal(ptr, p0) and np.array_equal(col, c0)
    import scipy.sparse as sp
    A = sp.csr_matrix((val, col, ptr))
    assert abs(A - A.T).max() > 0 and np.all(A.diagonal() > 0) and (A - sp.diags(A.diagonal())).max() <= 0
    assert np.all(np.asarray(A.sum(axis=1)).ravel() >= -1e-12)


@pytest.mark.skipif(build.amgcl_root() is None, reason="AMGCL headers not available")
def test_tutorial_program_compiles_without_nvcc():
    """INTEGRATION.md section 1: user code is plain C++ against the AMGCL headers and
    include/amgcl/backend/b200.hpp, linked with libamgcl_b200.so only."""
    exe = build.build_example(force=True)
    assert os.path.isfile(exe) and os.access(exe, os.X_OK)
    import subprocess
    needed = subprocess.run(["readelf", "-d", exe], stdout=subprocess.PIPE, text=True).stdout
    assert "libamgcl_b200.so" in needed and "libcudart" not in needed and "libcusparse" not in needed


def test_product_code_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing that ships (package, headers, native sources)
    may import, include, link or execute it, and there is no CPU fallback to route through."""
    offenders = []
    for base in ("amgcl_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if not f.endswith((".py", ".cpp", ".cu", ".cuh", ".h", ".hpp")):
                    continue
                text = open(os.path.join(dirpath, f), errors="replace").read()
                for lineno, line in enumerate(text.splitlines(), 1):
                    code = line.split("//")[0].split("#")[0] if not f.endswith(".py") else line.split("#")[0]
                    if re.search(r"\boracle\b|liboracle|libamgcl_ref|_ref/", code):
                        offenders.append("%s:%d: %s" % (os.path.join(dirpath, f), lineno, line.strip()))
    assert not offenders, "\n".join(offenders)


def test_every_header_entry_point_cites_the_reference():
    """include/amgcl_b200.h: the primitives name the reference interface they replace."""
    text = open(os.path.join(ROOT, "include", "amgcl_b200.h")).read()
    for needle in ("interface.hpp:312-323", "interface.hpp:329-335", "interface.hpp:356-371",
                   "interface.hpp:377-382", "interface.hpp:388-393", "interface.hpp:399-405",
                   "damped_jacobi.hpp:103-132", "spai0.hpp:86-109", "cuda.hpp:61-84",
                   "mpi/distributed_matrix.hpp:51-557"):
        assert needle in text, needle
