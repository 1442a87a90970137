"""GPU: the random programs of tests/_state.py on the real library, under every option set that
changes which path a call takes, each on its own Context; and the call sequences the programs
found wrong, as directed regression tests."""
import collections
import ctypes
import os

import numpy as np
import pytest

import _accuracy as acc
import _state as st
import amgcl_b200 as ab

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ("poisson12_damped_jacobi_cg", "poisson12_spai0_bicgstab")
_c = ctypes


@pytest.fixture(autouse=True)
def _extended():
    acc.require_longdouble()


class _Handle:
    def __init__(self, n, f32=False, tensor=None):
        self.h, self.n, self.f32, self.tensor = _c.c_void_p(), n, f32, tensor


class GpuApi:
    """The adapter tests/_state.Runner drives: one Context with the given options, the fixture's
    operators uploaded, vectors as raw handles (FP32 ones and wrapped torch memory included)."""
    Error = ab.B200Error

    def __init__(self, world, **options):
        self.L = ab.lib()
        self.ctx = ab.Context(0)
        for k, v in options.items():
            self.ctx.set_option(k, v)
        self.w = world
        self.ops = {}
        for nm, op in world.ops.items():
            if op.f32:
                A = ab.Csr.__new__(ab.Csr)
                A.ctx, A.h = self.ctx, _c.c_void_p()
                ab._check(self.L.b200_csr_create_i64_f32(self.ctx.h, op.nrows, op.ncols, ab._ptr(op.ptr),
                                                         ab._ptr(op.col), ab._ptr(op.val.astype(np.float32)),
                                                         _c.byref(A.h)), "b200_csr_create_i64_f32")
            else:
                A = self.ctx.csr(op.nrows, op.ncols, op.ptr, op.col, op.val)
            self.ops[nm] = A
        self.coarse = self.ctx.coarse(world.nc, *world.coarse)
        self.index = self.ctx.index(world.index, world.n0)
        self.vecs, self.krylovs, self.graphs = [], [], []

    @property
    def launches(self):
        return self.ctx.launches

    def tail_stats(self):
        return self.ctx.tail_stats()

    def vec(self, n, f32=False):
        v = _Handle(n, f32)
        fn = self.L.b200_vec_create_f32 if f32 else self.L.b200_vec_create
        ab._check(fn(self.ctx.h, n, _c.byref(v.h)), "b200_vec_create")
        self.vecs.append(v)
        return v

    def wrap(self, n):
        import torch
        t = torch.zeros(n, dtype=torch.float64, device="cuda:0")
        torch.cuda.synchronize()
        v = _Handle(n, tensor=t)
        ab._check(self.L.b200_vec_wrap(self.ctx.h, _c.c_void_p(t.data_ptr()), n, _c.byref(v.h)), "b200_vec_wrap")
        self.vecs.append(v)
        return v

    def caller_view(self, v):
        import torch
        torch.cuda.synchronize()
        return v.tensor.cpu().numpy()

    def destroy(self, v):
        ab._check(self.L.b200_vec_destroy(v.h), "b200_vec_destroy")
        self.vecs.remove(v)
        v.h = _c.c_void_p()

    def upload(self, v, a):
        if v.f32:
            a = np.ascontiguousarray(a, dtype=np.float32)
            ab._check(self.L.b200_vec_upload_f32(v.h, ab._ptr(a), v.n), "b200_vec_upload_f32")
        else:
            a = np.ascontiguousarray(a, dtype=np.float64)
            ab._check(self.L.b200_vec_upload(v.h, ab._ptr(a), v.n), "b200_vec_upload")

    def download(self, v):
        if v.f32:
            out = np.empty(v.n, dtype=np.float32)
            ab._check(self.L.b200_vec_download_f32(v.h, ab._ptr(out), v.n), "b200_vec_download_f32")
            return out.astype(np.float64)
        out = np.empty(v.n)
        ab._check(self.L.b200_vec_download(v.h, ab._ptr(out), v.n), "b200_vec_download")
        return out

    def flush(self):
        self.ctx.flush()

    def sync(self):
        self.ctx.sync()

    def clear(self, x):
        self.ctx.clear(x)

    def copy(self, x, y):
        self.ctx.copy(x, y)

    def axpby(self, a, x, b, y):
        self.ctx.axpby(a, x, b, y)

    def axpbypcz(self, a, x, b, y, c, z):
        self.ctx.axpbypcz(a, x, b, y, c, z)

    def vmul(self, a, x, y, b, z):
        self.ctx.vmul(a, x, y, b, z)

    def dot(self, x, y):
        return self.ctx.dot(x, y)

    def spmv(self, a, name, x, b, y):
        self.ctx.spmv(a, self.ops[name], x, b, y)

    def residual(self, f, name, x, r):
        self.ctx.residual(f, self.ops[name], x, r)

    def relax(self, name, f, x, t, d, om):
        self.ctx.relax(self.ops[name], f, x, t, d, om)

    def coarse_solve(self, f, x):
        self.ctx.coarse_solve(self.coarse, f, x)

    def gather(self, s, d):
        self.ctx.gather(self.index, s, d)

    def scatter(self, s, d):
        self.ctx.scatter(self.index, s, d)

    def graph_begin(self):
        return self.ctx.graph_begin()

    def graph_end(self):
        g = self.ctx.graph_end()
        self.graphs.append(g)
        return g

    def graph_abort(self):
        self.ctx.graph_abort()

    def graph_launch(self, g):
        return g.launch()

    def graph_destroy(self, g):
        g.close()
        self.graphs.remove(g)

    def krylov(self, n):
        K = ab.Krylov(self.ctx, n)
        self.krylovs.append(K)
        return K

    def krylov_destroy(self, K):
        K.close()
        self.krylovs.remove(K)

    def k_residual(self, K, f, name, x, r):
        return K.residual(f, self.ops[name], x, r)

    def k_scalars(self, K):
        return K.scalars()

    def cg_direction(self, K, r, s, p):
        K.cg_direction(r, s, p)

    def cg_step(self, K, name, p, q, x, r):
        return K.cg_step(self.ops[name], p, q, x, r)

    def bicg_start(self, K, r, rh):
        K.bicg_start(r, rh)

    def bicg_direction(self, K, r, v, p):
        K.bicg_direction(r, v, p)

    def bicg_step_s(self, K, name, rh, T, v, r, s, x):
        return K.bicg_step_s(self.ops[name], rh, T, v, r, s, x)

    def bicg_step_r(self, K, name, rh, T, t, s, r, x):
        return K.bicg_step_r(self.ops[name], rh, T, t, s, r, x)

    def close(self):
        self.ctx.graph_abort()                 # (a failed program may stop mid-recording)
        for g in self.graphs:
            g.close()
        for K in self.krylovs:
            K.close()
        for v in self.vecs:
            self.L.b200_vec_destroy(v.h)
            v.h = _c.c_void_p()
        for A in self.ops.values():
            self.L.b200_csr_destroy(A.h)
            A.h = _c.c_void_p()
        for o, fn in ((self.coarse, self.L.b200_coarse_destroy), (self.index, self.L.b200_index_destroy)):
            fn(o.h)
            o.h = _c.c_void_p()
        self.ctx.close()


_worlds = {}


def world(i):
    if i not in _worlds:
        _worlds[i] = st.World(os.path.join(GOLDEN, FIXTURES[i] + ".npz"))
    return _worlds[i]


def run_programs(seeds, **options):
    cov = collections.Counter()
    for seed in seeds:
        w = world(seed % 2)
        api = GpuApi(w, **options)
        try:
            cov.update(st.Runner(api, w, seed, tail=bool(options.get("coarse_tail"))).run())
        except ab.B200Error as e:
            raise AssertionError("seed %d: %s" % (seed, e))
        finally:
            api.close()
    return cov


def test_random_programs_default_options_reach_every_event():
    cov = run_programs(range(24))
    missing = [e for e in st.EVENTS if cov[e] == 0]
    assert not missing, "coverage events never reached: %s\n%s" % (missing, dict(cov))


OPTION_SETS = {
    "no_first_sweep_fusion": dict(fuse_first_sweep=0),
    "no_zero_shortcut": dict(zero_shortcut=0),
    "unfused_relax": dict(fuse_relax=0),
    "spmv_variant_0": dict(spmv_variant=0),
    "no_scalar_polling": dict(poll_scalars=0),
    # A1 (4,947 non-zeros), the coarse solve and the n1 sweeps from zero go to the coarse tail
    "coarse_tail": dict(coarse_tail=1, tail_max_nnz=5000, tail_max_vec=1000),
}


@pytest.mark.parametrize("name", sorted(OPTION_SETS))
def test_random_programs_under_other_options(name):
    cov = run_programs(range(100, 104), **OPTION_SETS[name])
    if name == "coarse_tail":
        assert all(cov[e] for e in st.TAIL_EVENTS), dict(cov)


# ---------------------------------------------------------------------------------------------
# directed regression tests: call sequences that gave wrong answers
# ---------------------------------------------------------------------------------------------
class Level0:
    """A context with A0 for one directed test.  Every handle that names the context is made
    here and destroyed before the context, even when a failing test's frame outlives it."""

    def __init__(self):
        self.w = world(0)
        self.ctx = ab.Context(0)
        op = self.w.ops["A0"]
        self.A = self.ctx.csr(op.nrows, op.ncols, op.ptr, op.col, op.val)
        self.rng = np.random.default_rng(5)
        self.vecs, self.krylovs = [], []

    def vec(self, data_or_n):
        v = self.ctx.vector(data_or_n)
        self.vecs.append(v)
        return v

    def wrap(self, t):
        v = ab.Vector.__new__(ab.Vector)
        v.ctx, v.h, v.n = self.ctx, _c.c_void_p(), t.numel()
        self.vecs.append(v)
        ab._check(ab.lib().b200_vec_wrap(self.ctx.h, _c.c_void_p(t.data_ptr()), v.n, _c.byref(v.h)), "b200_vec_wrap")
        return v

    def krylov(self, n):
        K = ab.Krylov(self.ctx, n)
        self.krylovs.append(K)
        return K

    def close(self):
        L = ab.lib()
        for K in self.krylovs:
            K.close()
        for v in self.vecs:
            if v.h:
                L.b200_vec_destroy(v.h)
            v.h = _c.c_void_p()
        L.b200_csr_destroy(self.A.h)
        self.A.h = _c.c_void_p()
        self.ctx.close()


@pytest.fixture
def lv0():
    L0 = Level0()
    yield L0
    L0.close()


def test_copy_of_a_zero_vector_drops_a_pending_first_sweep(lv0):
    ctx, A, w, rng, V = lv0.ctx, lv0.A, lv0.w, lv0.rng, lv0.vec
    n = w.n0
    f, t, d = V(rng.uniform(-1, 1, n)), V(n), V(w.diag["A0"])
    x, zero = V(n), V(n)                       # (creating a vector would flush the sweep)
    before = ctx.launches
    ctx.relax(A, f, x, t, d, w.omega)
    assert ctx.launches == before              # the sweep is pending
    ctx.copy(zero, x)
    got = x.numpy()
    assert not got.any(), "x holds the dropped sweep: max |x| = %g" % np.abs(got).max()


def test_copy_of_a_zero_vector_invalidates_products(lv0):
    ctx, A, w, rng, V = lv0.ctx, lv0.A, lv0.w, lv0.rng, lv0.vec
    n = w.n0
    K = lv0.krylov(n)
    r, s = V(rng.uniform(-1, 1, n)), V(rng.uniform(-1, 1, n))
    t, d, p, zero = V(n), V(w.diag["A0"]), V(n), V(n)
    ctx.relax(A, r, s, t, d, w.omega)          # full sweep: leaves <r, s>
    ctx.copy(zero, s)
    K.cg_direction(r, s, p)
    rho = K.scalars()["rho"]
    assert rho == 0.0, "rho = <r, 0> came out as %r" % rho
    assert not p.numpy().any()


def test_graph_abort_forgets_products_recorded_during_the_capture(lv0):
    ctx, A, w, rng, V = lv0.ctx, lv0.A, lv0.w, lv0.rng, lv0.vec
    n = w.n0
    lv0.krylov(n)
    rh, xh = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    r, x = V(rh), V(xh)
    t, d = V(n), V(w.diag["A0"])
    assert ctx.graph_begin()
    ctx.relax(A, r, x, t, d, w.omega)          # would leave <r, x>, but never runs
    ctx.graph_abort()
    assert np.array_equal(x.numpy(), xh)
    got = ctx.dot(r, x)
    want, scale = acc.dot_ref(rh, xh)
    acc.assert_scalar(got, want, acc.kahan_bound(scale, 2048), "dot(r, x) after an aborted recording")


def test_clear_of_wrapped_memory_reaches_the_callers_memory(lv0):
    import torch
    ctx, rng, V = lv0.ctx, lv0.rng, lv0.vec
    n = 1000
    t = torch.tensor(rng.uniform(1, 2, n), device="cuda:0")
    torch.cuda.synchronize()
    v = lv0.wrap(t)
    ctx.clear(v)
    ctx.sync()
    torch.cuda.synchronize()
    got = t.cpu().numpy()
    assert not got.any(), "the caller's memory still holds %d non-zeros" % int((got != 0).sum())
    src, zero = V(rng.uniform(1, 2, n)), V(n)
    ctx.copy(src, v)
    ctx.copy(zero, v)                          # a copy from a zero vector, too
    ctx.sync()
    torch.cuda.synchronize()
    assert not t.cpu().numpy().any()


def test_upload_invalidates_products(lv0):
    ctx, A, w, rng, V = lv0.ctx, lv0.A, lv0.w, lv0.rng, lv0.vec
    n = w.n0
    lv0.krylov(n)
    rh = rng.uniform(-1, 1, n)
    r, x = V(rh), V(rng.uniform(-1, 1, n))
    t, d = V(n), V(w.diag["A0"])
    ctx.relax(A, r, x, t, d, w.omega)          # leaves <r, x>
    xh = rng.uniform(-1, 1, n)
    x.upload(xh)
    got = ctx.dot(r, x)
    want, scale = acc.dot_ref(rh, xh)
    acc.assert_scalar(got, want, acc.kahan_bound(scale, 2048), "dot(r, x) after an upload of x")
