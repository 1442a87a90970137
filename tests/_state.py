"""Random call sequences against an extended-precision shadow model of the library's vectors.

Most of what can go wrong in the library between two calls is host-side state: the lazy clear
(``zero_pending``), the postponed first smoother sweep (``scale_pending`` / ``ctx->lazy_vec``),
the storage swaps of ``b200_relax``, the generation counters behind the product cache, the
Krylov workspace's rho parity, the deferred coarse-tail commands and graph recording.  This
module drives the library with seeded random programs of about 200 valid calls and checks every
value the program can observe against a model that knows nothing about any of that state.

Model
-----
Every library vector v is shadowed by its exact value ``val`` in ``np.longdouble`` and an
element-wise bound ``e`` on |GPU copy - val|.  A vector may also be *undefined* (``val is
None``): the ``tmp`` of a ``b200_relax`` (its contents are unspecified) and a vector that was
filled with NaNs, which the program only ever overwrites in full (outputs with a zero coefficient
are not read).  Operand magnitudes are taken as  x~ = |x| + e_x.  Each call updates ``val`` from
the model's own values in longdouble and propagates the bound to first order; u is the unit
roundoff of the output type (2^-53, FP32 outputs 2^-24) and gamma(m) = m u / (1 - m u):

* element-wise  y = a x + b y (+ c z), z = a x y + b z:  with c roundings (2 for axpby, 3 for
  axpbypcz and vmul; one more for FP32, whose coefficients are rounded to float first)
      e_y' = gamma(c) * sum |coef| * operands~  +  sum |coef| * (e of each operand)
  (for a product x y the operand term is x~ y~ and the error term e_x y~ + x~ e_y);
* CSR passes (spmv, residual, relax) reuse ``_accuracy``: the pass's own rounding is
  ``bound(mode, m, k, u, M~)`` with m, k from ``roundings(ptr, plan(ptr, 0, 2048))`` and
  M~ = |A| x~, and the propagated part is |alpha| |A| e_x (+ |beta| e_y), resp. e_f + |A| e_x
  for a residual and e_x + |omega d| (e_f + |A| e_x) for a sweep.  The sweep is bounded as a
  full sweep even from x = 0 (that dominates the exact scaling of the shortcut), with m + 1
  roundings for the unfused residual + vmul; an FP32 operator's sweep adds
  gamma32(m + 2) |omega d| (f~ + M~) for the FP32 residual (summed in FP32) of its unfused form;
* the dense coarse solve x = A_c^-1 rhs:  (4 n u kappa + gamma(n + 2)) |A_c^-1| rhs~ + |A_c^-1| e_rhs;
* copies, gather and scatter are exact (an FP64 -> FP32 copy adds u32 x~);
* inner products (``dot``, the in-kernel scalars of the Krylov steps):
      |s^ - s| <= G * sum x~ y~ + sum (e_x y~ + x~ e_y)
  with G the larger of ``kahan_bound``'s and ``csr_scalar_bound``'s coefficient (the model does
  not know whether a producer kernel left the value);
* Krylov quotients carry relative bounds: rel(a / b) = rel(a) + rel(b) + u, and an update
  x += alpha p adds |alpha| rel(alpha) p~ to the propagated terms.

Observation
-----------
Downloading a vector is one of the program's actions (it flushes a pending sweep but bumps no
generation and touches no product, so it barely perturbs the state) and every vector is
observed at the end.  Every element must lie within its bound; a failure names the vector, the
element, error / bound and the numbered calls that touched the vector since it was last
observed.  A passing observation adopts the GPU's values as exact (e = 0), so bounds never grow
over a long program.  Wrapped caller memory is also observed through the caller's own view after
a ``sync``.  Dots, Krylov scalars and ``Krylov.scalars()`` are checked in the same way.

The model decides nothing about which path the library takes: a graph replay is modelled as
re-applying the recorded calls when ``launch`` returns True and as nothing when it returns False;
a refused call (a host-side ``B200_REQUIRE``) must raise and changes nothing.

The runner talks to an adapter object (the real library in test_gpu_state.py, a numpy fake in
test_state_model.py) and classifies the calls by launch-count deltas into the coverage events
listed in ``EVENTS``.
"""
import collections
import math

import numpy as np
import scipy.sparse as sp

import _accuracy as acc

LD = acc.LD
U = acc.U64
U32 = acc.U32


def gam(m, u=U):
    return m * u / (1.0 - m * u)


# coverage events every default-option run set must reach (test_state_model / test_gpu_state)
EVENTS = (
    "lazy->fused_residual", "lazy->residual_other_rhs", "lazy->elementwise", "lazy->dot", "lazy->download",
    "lazy->clear", "lazy->copy_onto", "lazy->copy_from", "lazy->relax", "lazy->graph_begin",
    "product_hit:dot", "product_hit:cg_direction",
    "invalidated:relax", "invalidated:elementwise", "invalidated:copy", "invalidated:clear",
    "invalidated:upload", "invalidated:graph_abort", "invalidated:replay",
    "swap->read", "replay:launched", "replay:refused", "graph:abort", "parity:cg", "parity:bicg",
)
TAIL_EVENTS = ("tail:deferred", "tail:interleaved")


# ---------------------------------------------------------------------------------------------
# the problem: the two-level hierarchy of a poisson12 golden fixture
# ---------------------------------------------------------------------------------------------
class Op:
    """A CSR operator as the kernels read it (FP32 operators: values rounded to FP32)."""

    def __init__(self, name, ptr, col, val, ncols, f32=False):
        self.name, self.f32 = name, f32
        self.ptr = np.asarray(ptr, dtype=np.int64)
        self.col = np.asarray(col, dtype=np.int64)
        v = np.asarray(val, dtype=np.float64)
        self.val = v.astype(np.float32).astype(np.float64) if f32 else v
        self.nrows, self.ncols = self.ptr.size - 1, int(ncols)
        self.abs = sp.csr_matrix((np.abs(self.val), self.col, self.ptr), shape=(self.nrows, self.ncols))
        self.plan = acc.plan(self.ptr, 0, 2048)
        self.m, self.k = acc.roundings(self.ptr, self.plan)

    def S(self, x):
        return acc.row_sums(self.ptr, self.col, self.val, x)[0]

    def absdot(self, v):
        return self.abs.dot(np.asarray(v, dtype=np.float64)) * (1 + 1e-12)


class World:
    def __init__(self, fixture):
        z = np.load(fixture) if isinstance(fixture, str) else fixture
        self.omega = float(z["omega"])
        n0 = int(z["L0_A_ptr"].size - 1)
        n1 = int(z["L1_A_ptr"].size - 1)
        nc = int(z["C_ptr"].size - 1)
        self.n0, self.n1, self.nc = n0, n1, nc
        self.raw = {k: np.asarray(z[k]) for k in z.files if k[:3] in ("L0_", "L1_", "C_p", "C_c", "C_v")}
        g = lambda l, k: (z["L%d_%s_ptr" % (l, k)], z["L%d_%s_col" % (l, k)], z["L%d_%s_val" % (l, k)])
        self.ops = {
            "A0": Op("A0", *g(0, "A"), n0), "P0": Op("P0", *g(0, "P"), n1), "R0": Op("R0", *g(0, "R"), n0),
            "A1": Op("A1", *g(1, "A"), n1), "A0f": Op("A0f", *g(0, "A"), n0, f32=True),
        }
        self.diag = {"A0": np.asarray(z["L0_diag"], dtype=np.float64), "A1": np.asarray(z["L1_diag"], dtype=np.float64)}
        self.d32 = self.diag["A0"].astype(np.float32)
        C = sp.csr_matrix((z["C_val"], z["C_col"], z["C_ptr"]), shape=(nc, nc)).toarray()
        self.coarse = (np.asarray(z["C_ptr"]), np.asarray(z["C_col"]), np.asarray(z["C_val"]))
        inv = np.linalg.inv(C)
        # one step of refinement in longdouble: the model's inverse is far closer than the GPU's
        R = np.eye(nc, dtype=LD) - C.astype(LD) @ inv.astype(LD)
        self.Cinv = inv.astype(LD) + inv.astype(LD) @ R
        self.Cinv_abs = np.abs(inv) * (1 + 1e-6)
        kappa = np.abs(C).sum(axis=1).max() * np.abs(inv).sum(axis=1).max()
        self.coarse_rel = 4 * nc * U * kappa + gam(nc + 2)
        rng = np.random.default_rng(1)
        self.index = np.sort(rng.permutation(n0)[:n1])           # gather n0 -> n1, scatter back
        # one coefficient for every inner product (module docstring)
        sms = 132
        G = acc.kahan_bound(1.0, 2048)
        for nm in ("A0", "A1", "P0", "R0"):
            p = self.ops[nm].plan
            G = max(G, acc.csr_scalar_bound(1.0, p["nblocks"], p["rows_cap"], p["lanes"], sms, 8))
        self.G = G


# ---------------------------------------------------------------------------------------------
# shadows
# ---------------------------------------------------------------------------------------------
class Shadow:
    _ids = 0

    def __init__(self, h, n, name, f32=False, wrapped=False):
        self.h, self.n, self.name, self.f32, self.wrapped = h, n, name, f32, wrapped
        self.val = np.zeros(n, dtype=LD)
        self.e = np.zeros(n)
        self.touched = []        # call numbers since the last observation
        self.last_write = None   # call number of the last call that changed the model's value
        self.alive = True

    @property
    def defined(self):
        return self.val is not None

    def mag(self):
        return np.abs(self.val).astype(np.float64) * (1 + 1e-15) + self.e

    def set(self, val, e):
        self.val, self.e = val, np.asarray(e, dtype=np.float64)

    def undefine(self):
        self.val, self.e = None, np.zeros(self.n)

    def zero(self):
        return self.defined and not self.val.any()

    def __repr__(self):
        return self.name


class KModel:
    """A Krylov workspace and the model of its device scalars (value, absolute bound)."""

    def __init__(self, h, n, op):
        self.h, self.n, self.op = h, n, op
        self.kind = None          # "cg" | "bicg" once a residual started a solve
        self.stage = None         # next legal step
        self.roles = {}
        self.sc = {}              # scalar name -> (value LD, bound)
        self.last_step = None     # call number of the workspace's last step

    def __repr__(self):
        return "K%d" % self.n


class Fail(AssertionError):
    pass


# ---------------------------------------------------------------------------------------------
# the runner: generator + model + checks
# ---------------------------------------------------------------------------------------------
class Runner:
    def __init__(self, api, world, seed, ncalls=200, tail=False):
        self.api, self.w, self.seed, self.ncalls = api, world, seed, ncalls
        self.rng = np.random.default_rng(seed)
        self.log = []
        self.cov = collections.Counter()
        self.tail = tail
        self.recording = None         # list of recorded calls while a graph is being recorded
        self.snapshot = None
        self.graphs = []              # [(handle, calls)]
        self.K = {}                   # size -> KModel
        self.lazy = None              # (x, rhs) of a sweep that launched nothing
        self.swapped = set()          # vectors whose last write was a full sweep
        self.pairs = {}               # (rhs, x) -> writer kinds since a sweep left <rhs, x>
        self.pending_tail = False
        self.abort_touched = set()
        w = world
        mk = lambda n, nm: Shadow(api.vec(n), n, nm)
        self.pool = {w.n0: [mk(w.n0, "a%d" % i) for i in range(8)],
                     w.n1: [mk(w.n1, "b%d" % i) for i in range(8)],
                     w.nc: [mk(w.nc, "c%d" % i) for i in range(4)]}
        self.wrapv = Shadow(api.wrap(w.n0), w.n0, "w0", wrapped=True)
        self.pool[w.n0].append(self.wrapv)
        self.d = {"A0": Shadow(api.vec(w.n0), w.n0, "d0"), "A1": Shadow(api.vec(w.n1), w.n1, "d1")}
        for nm, s in self.d.items():
            api.upload(s.h, w.diag[nm])
            s.set(w.diag[nm].astype(LD), np.zeros(s.n))
        self.d32 = Shadow(api.vec(w.n0, f32=True), w.n0, "d32", f32=True)
        api.upload(self.d32.h, w.d32)
        self.d32.set(w.d32.astype(LD), np.zeros(w.n0))
        self.t32 = Shadow(api.vec(w.n0, f32=True), w.n0, "t32", f32=True)
        for n, vs in self.pool.items():
            for v in vs[:3]:
                self._upload(v, self._random(n))

    # ---- helpers ---------------------------------------------------------------------------
    def _random(self, n):
        r = self.rng
        return r.uniform(-1, 1, n) * np.exp2(r.integers(-4, 5))

    def _coef(self):
        u = self.rng.random()
        if u < 0.15:
            return 0.0
        if u < 0.3:
            return 1.0
        return float(self.rng.uniform(-2, 2))

    def vecs(self, n=None, defined=None, f64=True):
        out = []
        for m, vs in self.pool.items():
            if n is None or m == n:
                out += [v for v in vs if defined is None or v.defined == defined]
        if not f64:
            out += [v for v in (self.t32,) if defined is None or v.defined == defined]
        return out

    def pick(self, cands, k=1, distinct=True):
        cands = list(cands)
        if len(cands) < k:
            return None
        idx = self.rng.choice(len(cands), size=k, replace=not distinct)
        return [cands[i] for i in idx]

    def all_shadows(self):
        return [v for vs in self.pool.values() for v in vs] + list(self.d.values()) + [self.d32, self.t32]

    # ---- error messages ---------------------------------------------------------------------
    def _history(self, vs):
        idx = set(i for v in vs for i in v.touched)
        idx |= set(v.last_write for v in vs if v.last_write is not None)
        idx = sorted(idx)
        return "\n".join("    %s" % self.log[i] for i in idx) or "    (none)"

    def check_vector(self, v, got, how):
        if not v.defined:
            return
        got = np.asarray(got)
        err = np.abs(got.astype(LD) - v.val).astype(np.float64)
        bnd = v.e * (1 + 1e-9) + 1e-300
        bad = ~(err <= bnd)
        if bad.any():
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = np.where(bad, err / bnd, 0.0)
            ratio[~np.isfinite(ratio)] = np.inf
            i = int(np.argmax(ratio))
            raise Fail("seed %d, call #%d %s: vector %s element %d off by %.3g = %.3g x its bound %.3g "
                       "(got %r, want %r); %d elements over their bound.  Calls on %s since it was last "
                       "observed:\n%s" % (self.seed, len(self.log) - 1, how, v.name, i, err[i], ratio[i], bnd[i],
                                          float(got[i]), float(v.val[i]), int(bad.sum()), v.name,
                                          self._history([v])))

    def check_scalar(self, what, got, want, bnd, vs):
        err = abs(LD(got) - LD(want))
        if not (np.isfinite(got) and err <= LD(bnd) * (1 + 1e-9) + LD(1e-300)):
            raise Fail("seed %d, call #%d: %s got %r, want %r, off by %.3g = %.3g x its bound %.3g.  Calls on "
                       "its operands (%s) since they were last observed:\n%s" % (
                           self.seed, len(self.log) - 1, what, got, float(want), float(err),
                           float(err) / max(bnd, 1e-300), bnd, ", ".join(v.name for v in vs), self._history(vs)))

    def adopt(self, v, got):
        v.set(np.asarray(got).astype(LD), np.zeros(v.n))
        v.touched = []

    # ---- issuing calls -----------------------------------------------------------------------
    def issue(self, name, args, kind=None):
        """Log, call the adapter, apply the model; returns the adapter's result."""
        i = len(self.log)
        self.log.append("#%d %s(%s)" % (i, name, ", ".join(self._fmt(a) for a in args)))
        for a in args:
            if isinstance(a, Shadow):
                a.touched.append(i)
        self.api.call_index = i
        l0, t0 = self.api.launches, self.api.tail_stats()
        before = {v: (id(v.val), id(v.e)) for v in self.all_shadows()}
        res = getattr(self, "do_" + name)(*args)
        if args and isinstance(args[0], KModel):
            args[0].last_step = i
        for v, ids in before.items():
            if (id(v.val), id(v.e)) != ids and name not in ("download", "k_scalars"):
                v.last_write = i
        dl = self.api.launches - l0
        t1 = self.api.tail_stats()
        self.classify(name, args, dl, (t1[0] - t0[0], t1[1] - t0[1]), res)
        return res

    @staticmethod
    def _fmt(a):
        if isinstance(a, float):
            return "%.6g" % a
        if isinstance(a, np.ndarray):
            return "<NaN>" if np.isnan(a).any() else "<new values>"
        return str(a.name if isinstance(a, (Shadow, Op)) else a)

    def refuse(self, name, fn, vs):
        i = len(self.log)
        self.log.append("#%d %s (refused)" % (i, name))
        for v in vs:
            v.touched.append(i)
        try:
            fn()
        except self.api.Error:
            return
        raise Fail("seed %d, call #%d %s was not refused" % (self.seed, i, name))

    # ---- the model of each call --------------------------------------------------------------
    def rec(self, name, args):
        if self.recording is not None:
            self.recording.append((name, args))

    def m_clear(self, x):
        x.set(np.zeros(x.n, dtype=LD), np.zeros(x.n))

    def m_copy(self, x, y):
        if x is y:
            return
        if not x.defined:
            return y.undefine()
        e = x.e.copy()
        if y.f32 and not x.f32:
            e += U32 * x.mag()
        y.set(x.val.copy(), e)

    def _ew(self, out, terms, c):
        """out = sum coef * prod(operands); terms: [(coef, [shadows])]"""
        u = U32 if out.f32 else U
        if out.f32:
            c += 1
        if any(not s.defined for _, ss in terms for s in ss):
            return out.undefine()
        val = np.zeros(out.n, dtype=LD)
        scale = np.zeros(out.n)
        prop = np.zeros(out.n)
        for coef, ss in terms:
            p = np.full(out.n, LD(coef))
            m = np.full(out.n, abs(coef))
            for s in ss:
                p = p * s.val
            for j, s in enumerate(ss):
                others = np.full(out.n, abs(coef))
                for k2, t in enumerate(ss):
                    if k2 != j:
                        others = others * t.mag()
                prop += others * s.e
                m = m * s.mag()
            val += p
            scale += m
        out.set(val, gam(c, u) * scale + prop)

    def do_clear(self, x):
        self.api.clear(x.h); self.m_clear(x); self.rec("clear", (x,))

    def do_copy(self, x, y):
        self.api.copy(x.h, y.h); self.m_copy(x, y); self.rec("copy", (x, y))

    def do_axpby(self, a, x, b, y):
        self.api.axpby(a, x.h, b, y.h)
        self.m_axpby(a, x, b, y)
        self.rec("axpby", (a, x, b, y))

    def m_axpby(self, a, x, b, y):
        self._ew(y, [(a, [x])] + ([(b, [y])] if b != 0.0 else []), 2)

    def do_axpbypcz(self, a, x, b, y, c, z):
        self.api.axpbypcz(a, x.h, b, y.h, c, z.h)
        self.m_axpbypcz(a, x, b, y, c, z)
        self.rec("axpbypcz", (a, x, b, y, c, z))

    def m_axpbypcz(self, a, x, b, y, c, z):
        self._ew(z, [(a, [x]), (b, [y])] + ([(c, [z])] if c != 0.0 else []), 3)

    def do_vmul(self, a, x, y, b, z):
        self.api.vmul(a, x.h, y.h, b, z.h)
        self.m_vmul(a, x, y, b, z)
        self.rec("vmul", (a, x, y, b, z))

    def m_vmul(self, a, x, y, b, z):
        self._ew(z, [(a, [x, y])] + ([(b, [z])] if b != 0.0 else []), 3)

    def m_spmv(self, a, A, x, b, y):
        if not x.defined or (b != 0.0 and not y.defined):
            return y.undefine()
        xt = x.mag()
        M = A.absdot(xt)
        val = LD(a) * A.S(x.val)
        if b != 0.0:
            val = val + LD(b) * y.val
            bnd = acc.bound("spmv_acc", A.m, A.k, U, M, a, b, y0=y.mag()) + abs(b) * y.e
        else:
            bnd = acc.bound("spmv", A.m, A.k, U, M, a)
        y.set(val, bnd + abs(a) * A.absdot(x.e))

    def do_spmv(self, a, A, x, b, y):
        self.api.spmv(a, A.name, x.h, b, y.h); self.m_spmv(a, A, x, b, y); self.rec("spmv", (a, A, x, b, y))

    def m_residual(self, f, A, x, r):
        if not (f.defined and x.defined):
            return r.undefine()
        xt = x.mag()
        M = A.absdot(xt)
        val = f.val - A.S(x.val)
        r.set(val, acc.bound("resid", A.m, A.k, U, M, f=f.mag()) + f.e + A.absdot(x.e))

    def do_residual(self, f, A, x, r):
        self.api.residual(f.h, A.name, x.h, r.h); self.m_residual(f, A, x, r); self.rec("residual", (f, A, x, r))

    def m_relax(self, A, f, x, t, d, om):
        if not (f.defined and x.defined and d.defined):
            x.undefine()
        else:
            xt = x.mag()
            M = A.absdot(xt)
            wd = np.abs(om * d.val.astype(np.float64))
            val = x.val + LD(om) * d.val * (f.val - A.S(x.val))
            bnd = acc.bound("relax", A.m + 1, A.k, U, M, x0=xt, omega=om, d=d.val.astype(np.float64), f=f.mag())
            bnd = bnd + x.e + wd * (f.e + A.absdot(x.e))
            if A.f32:
                bnd = bnd + gam(A.m + 2, U32) * wd * (f.mag() + M + f.e + A.absdot(x.e))
            x.set(val, bnd)
        t.undefine()

    def do_relax(self, A, f, x, t, d, om):
        self.api.relax(A.name, f.h, x.h, t.h, d.h, om); self.m_relax(A, f, x, t, d, om)
        self.rec("relax", (A, f, x, t, d, om))

    def m_coarse(self, f, x):
        if not f.defined:
            return x.undefine()
        w = self.w
        x.set(w.Cinv @ f.val, w.coarse_rel * (w.Cinv_abs @ f.mag()) + w.Cinv_abs @ f.e)

    def do_coarse_solve(self, f, x):
        self.api.coarse_solve(f.h, x.h); self.m_coarse(f, x); self.rec("coarse_solve", (f, x))

    def m_gather(self, s, d):
        if not s.defined:
            return d.undefine()
        d.set(s.val[self.w.index].copy(), s.e[self.w.index].copy())

    def do_gather(self, s, d):
        self.api.gather(s.h, d.h); self.m_gather(s, d); self.rec("gather", (s, d))

    def m_scatter(self, s, d):
        if not (s.defined and d.defined):
            return d.undefine()
        v, e = d.val.copy(), d.e.copy()
        v[self.w.index], e[self.w.index] = s.val, s.e
        d.set(v, e)

    def do_scatter(self, s, d):
        self.api.scatter(s.h, d.h); self.m_scatter(s, d); self.rec("scatter", (s, d))

    def do_upload(self, v, a):
        self.api.upload(v.h, a)
        if np.isnan(a).any():
            v.undefine()
        else:
            v.set(np.asarray(a).astype(LD), np.zeros(v.n))

    def _upload(self, v, a):
        self.api.upload(v.h, a)
        v.set(np.asarray(a, dtype=np.float32 if v.f32 else np.float64).astype(LD), np.zeros(v.n))

    def do_download(self, v):
        got = self.api.download(v.h)
        self.check_vector(v, got, "download")
        if v.defined:
            self.adopt(v, got)

    def do_view(self, v):
        self.api.sync()
        got = self.api.caller_view(v.h)
        self.check_vector(v, got, "caller's view after sync")

    def dot_bound(self, x, y):
        xt, yt = x.mag(), y.mag()
        return self.w.G * float(np.sum(xt * yt)) * (1 + 1e-12) + float(np.sum(x.e * yt + xt * y.e))

    def do_dot(self, x, y):
        got = self.api.dot(x.h, y.h)
        if x.defined and y.defined:
            self.check_scalar("dot(%s, %s)" % (x.name, y.name), got, np.sum(x.val * y.val), self.dot_bound(x, y), [x, y])
        return got

    def do_flush(self):
        self.api.flush()

    def do_sync(self):
        self.api.sync()

    def do_destroy(self, v):
        n, nm = v.n, v.name
        self.api.destroy(v.h)
        v.alive = False
        new = Shadow(self.api.vec(n), n, nm)
        new.touched = list(v.touched)
        vs = self.pool[n]
        vs[vs.index(v)] = new
        for K in self.K.values():
            if v in K.roles.values():
                K.kind = None

    # ---- graphs -------------------------------------------------------------------------------
    def do_graph_begin(self):
        if not self.api.graph_begin():
            return False
        self.recording = []
        self.snapshot = {v: (v.val, v.e) for v in self.all_shadows()}
        return True

    def do_graph_end(self):
        g = self.api.graph_end()
        self.graphs.append((g, self.recording))
        self.recording, self.snapshot = None, None

    def do_graph_abort(self):
        self.api.graph_abort()
        for v, (val, e) in self.snapshot.items():
            v.val, v.e = val, e
        self.recording, self.snapshot = None, None

    def do_graph_launch(self, gi):
        g, calls = self.graphs[gi]
        ok = self.api.graph_launch(g)
        if ok:
            for name, args in calls:
                if any(isinstance(a, Shadow) and not a.alive for a in args):
                    raise Fail("seed %d, call #%d: a graph that names a destroyed vector replayed"
                               % (self.seed, len(self.log) - 1))
                for a in args:
                    if isinstance(a, Shadow):
                        a.touched.append(len(self.log) - 1)
                getattr(self, "m_" + {"clear": "clear", "copy": "copy", "axpby": "axpby", "axpbypcz": "axpbypcz",
                                      "vmul": "vmul", "spmv": "spmv", "residual": "residual", "relax": "relax",
                                      "coarse_solve": "coarse", "gather": "gather", "scatter": "scatter"}[name])(*args)
        return ok

    def do_graph_destroy(self, gi):
        g, _ = self.graphs.pop(gi)
        self.api.graph_destroy(g)

    # ---- Krylov --------------------------------------------------------------------------------
    def sc_check(self, K, name, got, want, bnd, vs):
        self.check_scalar("%s of the n = %d workspace" % (name, K.n), got, want, bnd, vs)

    def do_k_create(self, n):
        op = self.w.ops["A0" if n == self.w.n0 else "A1"]
        self.K[n] = KModel(self.api.krylov(n), n, op)

    def do_k_destroy(self, n):
        self.api.krylov_destroy(self.K.pop(n).h)

    def do_k_residual(self, K, f, A, x, r):
        got = self.api.k_residual(K.h, f.h, A.name, x.h, r.h)
        self.m_residual(f, A, x, r)
        self.sc_check(K, "Krylov.residual <r,r>", got, np.sum(r.val * r.val), self.dot_bound(r, r), [f, x, r])
        K.sc = {"rr": (np.sum(r.val * r.val), self.dot_bound(r, r))}

    def do_k_scalars(self, K):
        got = self.api.k_scalars(K.h)
        for nm, (want, bnd) in K.sc.items():
            if nm in got:
                self.sc_check(K, "Krylov.scalars()[%r]" % nm, got[nm], want, bnd, list(K.roles.values()))
                K.sc[nm] = (LD(got[nm]), 0.0)

    def _rel(self, K, nm):
        v, b = K.sc[nm]
        return float(b) / abs(float(v)) if v != 0 else math.inf

    def _update(self, out, coef, crel, p, scale_terms=None):
        """out += coef * p with a coefficient of relative error crel (2 roundings)."""
        pt = p.mag()
        val = out.val + LD(coef) * p.val
        e = out.e + abs(float(coef)) * (p.e + crel * pt) + gam(2) * (abs(float(coef)) * pt + out.mag())
        out.set(val, e)

    def parity_event(self, K, kind):
        """A direction step that reads rho_prev (not the first of its solve), with other calls
        between it and the workspace's previous step."""
        i = len(self.log) - 1
        if K.stage == "direction" and K.last_step is not None and K.last_step < i - 1:
            self.cov["parity:" + kind] += 1

    def do_cg_direction(self, K, r, s, p):
        self.parity_event(K, "cg")
        self.api.cg_direction(K.h, r.h, s.h, p.h)
        rho, brho = np.sum(r.val * s.val), self.dot_bound(r, s)
        if K.stage == "first":
            p.set(s.val.copy(), s.e.copy())
        else:
            rp, brp = K.sc["rho"]
            beta = rho / rp
            rb = (brho / abs(float(rho)) if rho != 0 else 0.0) + float(brp) / abs(float(rp)) + U
            pt = p.mag()
            val = s.val + beta * p.val
            e = s.e + abs(float(beta)) * (p.e + rb * pt) + gam(2) * (s.mag() + abs(float(beta)) * pt)
            if rho == 0:
                e = s.e + abs(float(brho / rp)) * pt + gam(2) * s.mag()
            p.set(val, e)
        K.sc["rho"] = (rho, brho)
        K.stage = "step"

    def do_cg_step(self, K, A, p, q, x, r):
        got = self.api.cg_step(K.h, A.name, p.h, q.h, x.h, r.h)
        self.m_spmv(1.0, A, p, 0.0, q)
        qp, bqp = np.sum(q.val * p.val), self.dot_bound(q, p)
        rho, brho = K.sc["rho"]
        alpha = rho / qp
        ra = float(brho) / abs(float(rho)) if rho != 0 else 0.0
        ra += float(bqp) / abs(float(qp)) + U
        if rho == 0:      # alpha == 0 up to |brho / qp|: the updates move by at most that much
            ab_ = float(brho) / abs(float(qp)) * (1 + 1e-6)
            x.set(x.val.copy(), x.e + ab_ * p.mag())
            r.set(r.val.copy(), r.e + ab_ * q.mag())
        else:
            self._update(x, alpha, ra, p)
            self._update(r, -alpha, ra, q)
        rr = np.sum(r.val * r.val)
        self.sc_check(K, "cg_step <r,r>", got, rr, self.dot_bound(r, r), [p, q, x, r])
        K.sc.update(qp=(qp, bqp), alpha=(alpha, abs(float(alpha)) * ra if rho != 0 else float(brho) / abs(float(qp))),
                    rr=(rr, self.dot_bound(r, r)))
        K.stage = "direction"

    def do_bicg_start(self, K, r, rh):
        self.api.bicg_start(K.h, r.h, rh.h)
        rh.set(r.val.copy(), r.e.copy())
        K.sc["rho_next"] = (np.sum(r.val * r.val), self.dot_bound(r, r))
        K.stage = "first"

    def do_bicg_direction(self, K, r, v, p):
        self.parity_event(K, "bicg")
        self.api.bicg_direction(K.h, r.h, v.h, p.h)
        rho, brho = K.sc["rho_next"]
        if K.stage == "first":
            p.set(r.val.copy(), r.e.copy())
        else:
            rp, brp = K.sc["rho"]
            al, bal = K.sc["alpha"]
            om, bom = K.sc["omega"]
            beta = (rho * al) / (rp * om)
            rbeta = sum(float(b) / abs(float(a)) for a, b in ((rho, brho), (al, bal), (rp, brp), (om, bom))) + 3 * U
            b, c = -beta * om, beta
            rb, rc = rbeta + float(bom) / abs(float(om)) + U, rbeta
            vt, pt = v.mag(), p.mag()
            val = r.val + b * v.val + c * p.val
            e = (r.e + abs(float(b)) * (v.e + rb * vt) + abs(float(c)) * (p.e + rc * pt)
                 + gam(3) * (r.mag() + abs(float(b)) * vt + abs(float(c)) * pt))
            p.set(val, e)
        K.sc["rho"] = (rho, brho)
        K.stage = "step_s"

    def do_bicg_step_s(self, K, A, rh, T, v, r, s, x):
        got = self.api.bicg_step_s(K.h, A.name, rh.h, T.h, v.h, r.h, s.h, x.h)
        self.m_spmv(1.0, A, T, 0.0, v)
        rhv, brhv = np.sum(rh.val * v.val), self.dot_bound(rh, v)
        rho, brho = K.sc["rho"]
        alpha = rho / rhv
        ra = float(brho) / abs(float(rho)) + float(brhv) / abs(float(rhv)) + U
        s.set(r.val.copy(), r.e.copy())
        self._update(x, alpha, ra, T)
        self._update(s, -alpha, ra, v)
        ss = np.sum(s.val * s.val)
        self.sc_check(K, "bicg_step_s <s,s>", got, ss, self.dot_bound(s, s), [rh, T, v, r, s, x])
        K.sc.update(qp=(rhv, brhv), alpha=(alpha, abs(float(alpha)) * ra), ss=(ss, self.dot_bound(s, s)))
        K.stage = "step_r"

    def do_bicg_step_r(self, K, A, rh, T, t, s, r, x):
        got = self.api.bicg_step_r(K.h, A.name, rh.h, T.h, t.h, s.h, r.h, x.h)
        self.m_spmv(1.0, A, T, 0.0, t)
        ts, bts = np.sum(t.val * s.val), self.dot_bound(t, s)
        tt, btt = np.sum(t.val * t.val), self.dot_bound(t, t)
        om = ts / tt
        ro = float(bts) / abs(float(ts)) + float(btt) / abs(float(tt)) + U
        r.set(s.val.copy(), s.e.copy())
        self._update(x, om, ro, T)
        self._update(r, -om, ro, t)
        rr = np.sum(r.val * r.val)
        self.sc_check(K, "bicg_step_r <r,r>", got, rr, self.dot_bound(r, r), [rh, T, t, s, r, x])
        K.sc.update(ts=(ts, bts), tt=(tt, btt), omega=(om, abs(float(om)) * ro), rr=(rr, self.dot_bound(r, r)),
                    rho_next=(np.sum(r.val * rh.val), self.dot_bound(r, rh)))
        K.stage = "direction"

    # ---- coverage --------------------------------------------------------------------------
    def classify(self, name, args, dl, dtail, res):
        vs = [a for a in args if isinstance(a, Shadow)]
        if self.lazy is not None:
            x, rhs = self.lazy
            self.lazy = None
            kind = None
            if name == "residual":
                kind = "fused_residual" if (args[0] is rhs and args[2] is x and dl == 1) else \
                    ("residual_other_rhs" if args[2] is x and args[0] is not rhs else None)
            elif name in ("axpby", "axpbypcz", "vmul") and x in vs[:-1]:
                kind = "elementwise"
            elif name == "dot" and x in vs:
                kind = "dot"
            elif name == "download" and x in vs:
                kind = "download"
            elif name == "clear" and x in vs:
                kind = "clear"
            elif name == "copy":
                kind = "copy_onto" if args[1] is x else ("copy_from" if args[0] is x else None)
            elif name == "relax":
                kind = "relax"
            elif name == "graph_begin":
                kind = "graph_begin"
            if kind:
                self.cov["lazy->" + kind] += 1
        if name == "relax" and not self.tail:
            A, f, x = args[0], args[1], args[2]
            if dl == 0 and self.recording is None:
                self.lazy = (x, f)
            else:
                if self.recording is None:
                    self.swapped.add(x)
                if x.n in self.K:
                    self.pairs[(f, x)] = set()
        elif self.swapped and vs:
            reads = vs if name not in ("clear", "copy", "download") else vs[:1]
            if name in ("clear",):
                reads = []
            if any(v in self.swapped for v in reads):
                self.cov["swap->read"] += 1
            self.swapped -= set(vs)
        if name in ("dot", "cg_direction") and self.recording is None:
            pair = (args[0], args[1]) if name == "dot" else (args[1], args[2])
            if name == "cg_direction":
                pair = (args[1], args[2])
            for key in (pair, pair[::-1]):
                if key in self.pairs:
                    for k in self.pairs.pop(key):
                        self.cov["invalidated:" + k] += 1
            hit = (name == "dot" and dl == 0 and not pair[0].zero() and not pair[1].zero()) or \
                  (name == "cg_direction" and dl == 1)
            if hit:
                self.cov["product_hit:" + name] += 1
        writer = {"graph_launch": "replay" if res else None, "relax": "relax", "axpby": "elementwise",
                  "axpbypcz": "elementwise", "vmul": "elementwise", "copy": "copy", "clear": "clear",
                  "upload": "upload", "graph_abort": "graph_abort"}.get(name)
        if writer and self.pairs:
            outs = {"relax": vs[1:3], "copy": vs[1:2], "clear": vs[:1], "upload": vs[:1]}.get(name, vs[-1:])
            if name == "graph_abort":
                outs = list(self.abort_touched)
            if name == "graph_launch":
                outs = [a for _, cargs in self.graphs[args[0]][1] for a in cargs if isinstance(a, Shadow)]
            for key, ks in self.pairs.items():
                if (key[0] in outs or key[1] in outs) and not (name == "relax" and key == (args[1], args[2])):
                    ks.add(writer)
        if name == "graph_launch":
            self.cov["replay:launched" if res else "replay:refused"] += 1
        if name == "graph_abort":
            self.cov["graph:abort"] += 1
        if self.tail:
            if name in ("spmv", "residual", "relax", "coarse_solve") and dl == 0 and self.recording is None:
                self.pending_tail = True
                self.cov["tail:deferred"] += 1
            elif getattr(self, "pending_tail", False) and dl > 0:
                if dtail[0] > 0 and dl > dtail[0]:
                    self.cov["tail:interleaved"] += 1
                self.pending_tail = False

    # ---- the generator --------------------------------------------------------------------------
    def run(self):
        steps = 0
        while len(self.log) < self.ncalls and steps < 20 * self.ncalls:
            steps += 1
            self.step()
        if self.recording is not None:
            self.issue("graph_end", ())
        self.issue("sync", ())
        for v in self.all_shadows():
            if v.defined:
                self.issue("download", (v,))
        self.issue("view", (self.wrapv,))
        for K in list(self.K.values()):
            if K.kind is not None:
                self.issue("k_scalars", (K,))
        return self.cov

    def _defined(self, n):
        return [v for v in self.pool[n] if v.defined]

    def step(self):
        r = self.rng
        w = self.w
        acts = ["ew", "ew", "ew", "copy", "clear", "dot", "spmv", "residual", "relax", "relax", "relax", "coarse",
                "gather", "download", "krylov", "krylov", "krylov", "krylov", "graph", "misc", "refuse", "rescale", "f32"]
        act = acts[r.integers(len(acts))]
        getattr(self, "g_" + act)()

    def g_rescale(self):
        for v in self.vecs():
            if v.defined:
                m = float(np.abs(v.val).max())
                if m > 1e30 or 0 < m < 1e-30:
                    k = -int(math.floor(math.log2(m)))
                    return self.issue("axpby", (2.0 ** k, v, 0.0, v))

    def g_ew(self):
        r = self.rng
        n = [self.w.n0, self.w.n1, self.w.nc][r.integers(3)]
        src = self._defined(n)
        if not src:
            return
        kind = r.integers(3)
        out = self.pick(self.pool[n])[0]
        if kind == 0:
            x = self.pick(src)[0]
            b = self._coef() if out.defined else 0.0
            self.issue("axpby", (self._coef() or 0.5, x, b, out))
        elif kind == 1 and len(src) >= 1:
            x, y = self.pick(src, 2, distinct=False)
            c = self._coef() if out.defined else 0.0
            self.issue("axpbypcz", (self._coef(), x, self._coef(), y, c, out))
        else:
            x, y = self.pick(src, 2, distinct=False)
            b = self._coef() if out.defined else 0.0
            self.issue("vmul", (self._coef(), x, y, b, out))

    def g_copy(self):
        r = self.rng
        n = [self.w.n0, self.w.n1][r.integers(2)]
        u = r.random()
        if u < 0.3:
            z = [v for v in self.pool[n] if v.zero()]
            if not z:
                return
            self.issue("copy", (self.pick(z)[0], self.pick(self.pool[n])[0]))
        elif u < 0.4:
            v = self.pick(self.pool[n])[0]
            self.issue("copy", (v, v))
        else:
            src = self._defined(n)
            if src:
                self.issue("copy", (self.pick(src)[0], self.pick(self.pool[n])[0]))

    def g_clear(self):
        n = [self.w.n0, self.w.n1, self.w.nc][self.rng.integers(3)]
        v = self.pick(self.pool[n])[0]
        if self.rng.random() < 0.2:
            v = self.wrapv
        self.issue("clear", (v,))
        if v is self.wrapv and self.recording is None and self.rng.random() < 0.6:
            self.issue("view", (v,))

    def g_dot(self):
        if self.recording is not None:
            return self.refuse("dot while recording", lambda: self.api.dot(self.d["A0"].h, self.d["A0"].h), [])
        n = [self.w.n0, self.w.n1][self.rng.integers(2)]
        src = self._defined(n)
        if src:
            x = self.pick(src)[0]
            y = x if self.rng.random() < 0.2 else self.pick(src)[0]
            self.issue("dot", (x, y))

    def g_spmv(self):
        w, r = self.w, self.rng
        A = w.ops[["A0", "A1", "P0", "R0", "A0f"][r.integers(5)]]
        xs = self._defined(A.ncols)
        if not xs:
            return
        x = self.pick(xs)[0]
        ys = [v for v in self.pool[A.nrows] if v is not x]
        y = self.pick(ys)[0]
        b = self._coef() if y.defined else 0.0
        self.issue("spmv", (self._coef() or 1.0, A, x, b, y))

    def g_residual(self):
        w, r = self.w, self.rng
        A = w.ops[["A0", "A1", "A0f"][r.integers(3)]]
        src = self._defined(A.nrows)
        if len(src) < 1:
            return
        if self.lazy is not None and self.lazy[0].n == A.nrows and r.random() < 0.7:
            x, f = self.lazy
            if r.random() < 0.3:
                f = self.pick(src)[0]
        else:
            x = self.pick(src)[0]
            f = self.pick(src)[0]
        if r.random() < 0.15 and f is not x:
            rr = f
        else:
            rr = self.pick([v for v in self.pool[A.nrows] if v is not x and v is not f])[0]
        self.issue("residual", (f, A, x, rr))

    def g_relax(self):
        w, r = self.w, self.rng
        nm = ["A0", "A0", "A1", "A0f"][r.integers(4)]
        A = w.ops[nm]
        n = A.nrows
        src = self._defined(n)
        if not src:
            return
        f = self.pick(src)[0]
        rest = [v for v in self.pool[n] if v is not f]
        if nm == "A0f":
            x = self.pick([v for v in rest if v.defined] or [None])[0]
            if x is None:
                return
            t, d = self.t32, self.d32
        else:
            x, t = self.pick(rest, 2)
            d = self.d[nm]
            if not x.defined:
                return
        if r.random() < 0.5 and x is not self.wrapv:
            self.issue("clear", (x,))
        self.issue("relax", (A, f, x, t, d, w.omega))
        if self.lazy is not None and r.random() < 0.85:
            self.resolve_lazy()

    def resolve_lazy(self):
        x, f = self.lazy
        r = self.rng
        u = r.integers(10)
        n = x.n
        others = [v for v in self._defined(n) if v is not x]
        out = self.pick([v for v in self.pool[n] if v is not x and v is not f] or [None])[0]
        if u == 0 and out is not None:
            self.issue("residual", (f, self.w.ops["A0" if n == self.w.n0 else "A1"], x, out))
        elif u == 1 and out is not None and others:
            self.issue("residual", (self.pick(others)[0], self.w.ops["A0" if n == self.w.n0 else "A1"], x, out))
        elif u == 2 and out is not None:
            self.issue("axpby", (1.5, x, 0.0, out))
        elif u == 3:
            self.issue("dot", (x, self.pick(others)[0] if others else x))
        elif u == 4:
            self.issue("download", (x,))
        elif u == 5:
            self.issue("clear", (x,))
        elif u == 6:
            z = self.pick([v for v in self.pool[n] if v.zero() and v is not x] or [None])[0]
            if z is None and out is not None and out is not self.wrapv:
                z = out
                self.issue("clear", (z,))
            if z is not None:
                self.issue("copy", (z, x))
            elif others:
                self.issue("copy", (self.pick(others)[0], x))
        elif u == 7 and out is not None:
            self.issue("copy", (x, out))
        elif u == 8:
            self.g_relax()
        elif self.recording is None:
            self.g_graph(begin_only=True)

    def g_coarse(self):
        r = self.rng
        src = self._defined(self.w.nc)
        if src:
            f = self.pick(src)[0]
            self.issue("coarse_solve", (f, self.pick([v for v in self.pool[self.w.nc] if v is not f])[0]))

    def g_gather(self):
        w = self.w
        if self.rng.random() < 0.5:
            src = self._defined(w.n0)
            if src:
                self.issue("gather", (self.pick(src)[0], self.pick(self.pool[w.n1])[0]))
        else:
            src = self._defined(w.n1)
            dst = self._defined(w.n0)
            if src and dst:
                self.issue("scatter", (self.pick(src)[0], self.pick(dst)[0]))

    def g_download(self):
        if self.recording is not None:
            return
        v = self.pick([v for v in self.vecs() if v.defined] or [None])[0]
        if v is None:
            return
        if v is self.wrapv and self.rng.random() < 0.5:
            self.issue("view", (v,))
        self.issue("download", (v,))

    def g_f32(self):
        r = self.rng
        u = r.integers(4)
        src = self._defined(self.w.n0)
        if u == 0 and src:
            self.issue("copy", (self.pick(src)[0], self.t32))
        elif u == 1 and self.t32.defined:
            self.issue("copy", (self.t32, self.pick(self.pool[self.w.n0])[0]))
        elif u == 2 and self.t32.defined:
            self.issue("axpby", (0.75, self.d32, self._coef(), self.t32))
        elif u == 3 and self.t32.defined:
            out = self.pick(self.pool[self.w.n0])[0]
            self.issue("vmul", (self._coef(), self.d32, self.t32, self._coef() if out.defined else 0.0, out))

    def g_misc(self):
        r = self.rng
        u = r.integers(6)
        if u == 0:
            self.issue("flush", ())
        elif self.recording is not None:
            return
        elif u == 1:
            self.issue("sync", ())
        elif u == 2:
            n = [self.w.n0, self.w.n1][r.integers(2)]
            v = self.pick([v for v in self.pool[n] if v is not self.wrapv])[0]
            self.issue("destroy", (v,))
        elif u == 3:
            # NaNs into a vector whose next use overwrites it in full
            n = [self.w.n0, self.w.n1][r.integers(2)]
            src = self._defined(n)
            v = self.pick(self.pool[n])[0]
            if not src or v in src[:1]:
                return
            self.issue("upload", (v, np.full(n, np.nan)))
            x = self.pick([s for s in src if s is not v] or [None])[0]
            if x is None:
                return self.issue("clear", (v,))
            k = r.integers(4)
            if k == 0:
                self.issue("axpby", (self._coef() or 2.0, x, 0.0, v))
            elif k == 1:
                self.issue("axpbypcz", (1.0, x, -0.5, x, 0.0, v))
            elif k == 2:
                self.issue("vmul", (0.5, x, x, 0.0, v))
            else:
                A = self.w.ops["A0" if n == self.w.n0 else "A1"]
                self.issue("spmv", (1.0, A, x, 0.0, v))
        elif u == 4:
            n = [self.w.n0, self.w.n1][r.integers(2)]
            self.issue("upload", (self.pick(self.pool[n])[0], self._random(n)))
        else:
            v = self.pick([v for v in self.vecs() if v.defined] or [None])[0]
            if v is not None:
                self.issue("download", (v,))

    def g_refuse(self):
        w, api = self.w, self.api
        a, b = self.pool[w.n0][0], self.pool[w.n0][1]
        c = self.pool[w.n1][0]
        u = self.rng.integers(4)
        if u == 0:
            self.refuse("spmv(A0, %s, %s) aliased" % (a, a), lambda: api.spmv(1.0, "A0", a.h, 0.0, a.h), [a])
        elif u == 1:
            self.refuse("axpby(%s, %s) size mismatch" % (a, c), lambda: api.axpby(1.0, a.h, 1.0, c.h), [a, c])
        elif u == 2:
            self.refuse("relax(A0, %s, %s, %s) x == tmp" % (a, b, b),
                        lambda: api.relax("A0", a.h, b.h, b.h, self.d["A0"].h, 0.5), [a, b])
        else:
            self.refuse("residual(%s, A1, %s, %s) size mismatch" % (c, a, c), lambda: api.residual(c.h, "A1", a.h, c.h),
                        [a, c])

    def g_graph(self, begin_only=False):
        r = self.rng
        if self.recording is None:
            u = r.random()
            if begin_only or u < 0.4:
                if self.issue("graph_begin", ()):
                    self.abort_touched = set()
                    if not begin_only and r.random() < 0.5:
                        self.g_replayable()
            elif self.graphs and u < 0.9:
                self.issue("graph_launch", (int(r.integers(len(self.graphs))),))
            elif self.graphs:
                self.issue("graph_destroy", (int(r.integers(len(self.graphs))),))
        else:
            if len(self.recording) < 2 and r.random() < 0.7:
                return
            if r.random() < 0.3:
                self.abort_touched = set(a for _, args in self.recording for a in args if isinstance(a, Shadow))
                self.issue("graph_abort", ())
            else:
                self.issue("graph_end", ())
                if r.random() < 0.6:
                    self.issue("graph_launch", (len(self.graphs) - 1,))

    def g_replayable(self):
        """Record calls that leave every pointer and lazy-clear flag as they found it, end the
        recording and replay it at once."""
        n = [self.w.n0, self.w.n1][self.rng.integers(2)]
        live = [v for v in self._defined(n) if not v.zero()]
        if len(live) < 3:
            return
        x, y, z = self.pick(live, 3)
        self.issue("axpby", (self._coef() or 0.5, x, self._coef(), y))
        A = self.w.ops["A0" if n == self.w.n0 else "A1"]
        self.issue("spmv", (1.0, A, y, 0.5, z))
        self.issue("graph_end", ())
        for _ in range(self.rng.integers(1, 3)):
            self.issue("graph_launch", (len(self.graphs) - 1,))

    def g_krylov(self):
        r = self.rng
        if self.recording is not None:
            if self.K:
                K = next(iter(self.K.values()))
                v = self.pool[K.n][0]
                self.refuse("Krylov.residual while recording",
                            lambda: self.api.k_residual(K.h, v.h, K.op.name, v.h, self.pool[K.n][1].h), [])
            return
        # a solve in progress is continued more often than a new one is started, so that
        # direction steps that read rho_prev come up in every run
        active = [m for m, K in self.K.items() if K.kind is not None]
        n = active[r.integers(len(active))] if active and r.random() < 0.8 else [self.w.n0, self.w.n1][r.integers(2)]
        if n not in self.K:
            return self.issue("k_create", (n,))
        K = self.K[n]
        if r.random() < 0.02:
            return self.issue("k_destroy", (n,))
        if r.random() < 0.06:
            return self.issue("k_scalars", (K,))
        roles = K.roles
        if K.kind is None or any(not v.alive for v in roles.values()) or r.random() < 0.015:
            return self.k_start(K)
        if K.kind == "cg":
            self.k_cg(K)
        else:
            self.k_bicg(K)

    def k_start(self, K):
        r = self.rng
        vs = [v for v in self.pool[K.n] if v is not self.wrapv or r.random() < 0.3]
        src = [v for v in vs if v.defined]
        if len(vs) < 8 or not src:
            return
        kind = "cg" if r.random() < 0.6 else "bicg"
        f = self.pick(src)[0]
        rest = [v for v in vs if v is not f]
        names = ("x", "r", "s", "p", "q", "t") if kind == "cg" else ("x", "r", "rh", "p", "v", "s", "t")
        K.roles = dict(zip(names, self.pick(rest, len(names))))
        K.roles["f"] = f
        K.kind = kind
        x, rr = K.roles["x"], K.roles["r"]
        if not x.defined or r.random() < 0.5:
            self.issue("clear", (x,))
        self.issue("k_residual", (K, f, K.op, x, rr))
        if kind == "cg":
            K.stage = "first"
        else:
            self.issue("bicg_start", (K, rr, K.roles["rh"]))

    def _observe(self, vs):
        for v in vs:
            if v.defined and v.e.max() > 1e-9 * float(np.abs(v.val).max()):
                self.issue("download", (v,))

    def _den_ok(self, K, names, vs):
        """Before a step whose denominator's relative bound exceeds 1e-6, observe its operands
        (and adopt the scalars); give the solve up on a denominator that is (nearly) zero."""
        if any(nm in K.sc and self._rel(K, nm) > 1e-6 for nm in names):
            self._observe(vs)
            self.issue("k_scalars", (K,))
        for nm in names:
            v, b = K.sc[nm]
            if v == 0 or float(b) > 1e-6 * abs(float(v)):
                self.issue("k_scalars", (K,))       # the solve is given up: look at its scalars first
                K.kind = None
                return False
        return True

    @staticmethod
    def _den_pred(A, T, w):
        """<A T, w> of the step about to run is well away from zero."""
        y = A.S(T.val)
        d = abs(float(np.sum(y * w.val)))
        return d > 1e-8 * float(np.sum(np.abs(y * w.val))) and d > 0

    def g_invalidate(self, K, r, s, t):
        """A writer of each kind between the sweep that left <r, s> and its lookup."""
        u = min(self.rng.integers(8), 6)
        u = 2 if u == 6 and self.rng.random() < 0.3 else u
        d = self.d[K.op.name]
        others = [v for v in self._defined(K.n) if v not in (r, s, t)]
        if u == 0 and others:
            self.issue("relax", (K.op, self.pick(others)[0], s, t, d, self.w.omega))
        elif u == 1:
            self.issue("axpby", (1.0, r, 0.5, s))
        elif u == 2:
            z = [v for v in self.pool[K.n] if v.zero() and v not in (r, s)]
            spare = [v for v in self.pool[K.n] if v not in K.roles.values() and v is not t]
            if not z and spare:
                z = spare[:1]
                self.issue("clear", (z[0],))
            self.issue("copy", ((z or [r])[0], s))
        elif u == 3:
            self.issue("clear", (s,))
        elif u == 4:
            self.issue("upload", (s, self._random(K.n)))
        elif u == 6:
            # a replay that writes s: record the write, then two sweeps (their swaps cancel, so
            # the replay's state check passes) leave <r, s> again, then the replay
            if self.issue("graph_begin", ()):
                self.issue("axpby", (0.5, r, 0.5, s))
                self.issue("graph_end", ())
                for _ in range(2):
                    self.issue("relax", (K.op, r, s, t, d, self.w.omega))
                self.issue("graph_launch", (len(self.graphs) - 1,))
        elif u == 5:
            if self.issue("graph_begin", ()):
                self.issue("relax", (K.op, r, s, t, d, self.w.omega))
                self.abort_touched = {r, s, t, d}
                self.issue("graph_abort", ())

    def k_cg(self, K):
        R = K.roles
        r, s, p, q, x, t = R["r"], R["s"], R["p"], R["q"], R["x"], R["t"]
        rnd = self.rng.random
        if K.stage in ("first", "direction"):
            if not r.defined:
                K.kind = None
                return
            # the preconditioner: sweeps from zero (the second leaves <r, s> behind)
            u = rnd()
            if u < 0.7:
                self.issue("clear", (s,))
                self.issue("relax", (K.op, r, s, t, self.d[K.op.name], self.w.omega))
                if u < 0.55:
                    self.issue("relax", (K.op, r, s, t, self.d[K.op.name], self.w.omega))
                    if rnd() < 0.3:
                        self.issue("dot", (r, s) if rnd() < 0.5 else (s, r))
                    if rnd() < 0.6:
                        self.g_invalidate(K, r, s, t)
            elif u < 0.85 or not s.defined:
                self.issue("copy", (r, s))
            if not s.defined or (K.stage == "direction" and (not p.defined or not self._den_ok(K, ["rho"], [r, s]))):
                K.kind = None
                return
            self.issue("cg_direction", (K, r, s, p))
            if rnd() < 0.4:
                self.issue("k_scalars", (K,))
        elif K.stage == "step":
            if not (p.defined and x.defined and r.defined):
                K.kind = None
                return
            self._observe([p])
            if not self._den_pred(K.op, p, p):
                self.issue("k_scalars", (K,))       # the solve is given up: look at its scalars first
                K.kind = None
                return
            self.issue("cg_step", (K, K.op, p, q, x, r))

    def k_bicg(self, K):
        R = K.roles
        r, rh, p, v, s, t, x = R["r"], R["rh"], R["p"], R["v"], R["s"], R["t"], R["x"]
        if K.stage in ("first", "direction"):
            if not (r.defined and (K.stage == "first" or (v.defined and p.defined))):
                K.kind = None
                return
            if K.stage == "direction" and not self._den_ok(K, ["rho", "omega", "alpha", "rho_next"], [r, v, p, rh]):
                return
            self.issue("bicg_direction", (K, r, v, p))
        elif K.stage == "step_s":
            if not (p.defined and rh.defined and x.defined and r.defined):
                K.kind = None
                return
            self._observe([p, rh])
            if not self._den_ok(K, ["rho"], [r, rh]):      # (rho = 0: alpha would be 0)
                return
            if not self._den_pred(K.op, p, rh):
                K.kind = None
                return
            self.issue("bicg_step_s", (K, K.op, rh, p, v, r, s, x))
            if not self._den_ok(K, ["qp"], []):
                return
        elif K.stage == "step_r":
            if not (s.defined and rh.defined and x.defined):
                K.kind = None
                return
            self._observe([s])
            if not (self._den_pred(K.op, s, s) and s.val.any()):
                K.kind = None
                return
            self.issue("bicg_step_r", (K, K.op, rh, s, t, s, r, x))
            self._den_ok(K, ["ts", "tt"], [])

