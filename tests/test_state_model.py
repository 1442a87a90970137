"""CPU: the random programs of tests/_state.py are able to find wrong host-side state.

A numpy fake of the context API follows the library's host-side logic (api_*.cu): lazy clears,
the postponed first sweep, storage swaps, generation counters and the four-entry product cache,
the Krylov workspace's rho parity, the coarse-tail list and graph recording with baked-in
storage.  Its device work runs in numpy.  The faithful fake must run every seed clean and reach
every coverage event; each mutant -- the fake wrong in one small way -- must be rejected by a
fixed seed, and the failure must name a call at which the mutant went its own way."""
import collections
import os

import numpy as np
import pytest

import _accuracy as acc
import _state as st

LD = acc.LD
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ("poisson12_damped_jacobi_cg", "poisson12_spai0_bicgstab")

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


@pytest.fixture(autouse=True)
def _extended():
    acc.require_longdouble()


class FakeError(RuntimeError):
    pass


def require(cond, msg):
    if not cond:
        raise FakeError(msg)


class FVec:
    def __init__(self, n, f32=False, buf=None):
        self.n, self.f32 = n, f32
        self.owned = buf is None
        self.escaped = not self.owned
        self.ptr = np.zeros(n, dtype=np.float32 if f32 else np.float64) if buf is None else buf
        self.caller = buf
        self.zero_pending = self.owned
        self.scale_pending = False
        self.sc = None
        self.gen = 0
        self.in_graph = False


class Holder:
    """An operator's FP64 scratch (trades places with x in the mixed-precision sweep)."""
    zero_pending = None
    gen = None

    def __init__(self, n):
        self.ptr = np.zeros(n)


class FGraph:
    def __init__(self, fake):
        self.ops, self.slots, self.products = [], [], []
        self.destroy_epoch, self.option_epoch = fake.destroy_epoch, fake.option_epoch
        self.launches0, self.launches = fake.launches, 0


class FKrylov:
    def __init__(self, n, base):
        self.n, self.base, self.first, self.parity = n, base, True, 0


# slots of the scalar table (api_krylov.cu)
SLOT_DOT, SLOT_PRODUCT0, SLOT_FIRST_FREE = 0, 2, 6
K_RHO, K_RHOP0, K_RHOP1, K_QP, K_RR, K_SS, K_TS, K_TT, K_ALPHA, K_OMEGA, K_RHO_NEXT = range(11)
K_NSLOTS = 16


def rnd(v, f32=False):
    return np.asarray(v).astype(np.float32 if f32 else np.float64)


class Fake:
    """Numpy stand-in for amgcl_b200's context, vectors, operators and Krylov workspaces."""
    Error = FakeError

    def __init__(self, world, **options):
        self.w = world
        self.opt = dict(fuse_first_sweep=1, zero_shortcut=1, fuse_relax=1, spmv_variant=1, coarse_tail=0,
                        tail_max_nnz=1500000, tail_max_vec=262144)
        self.opt.update(options)
        self.launches = 0
        self.tail, self.tail_flushes, self.tail_commands, self.tail_hold = [], 0, 0, 0
        self.lazy_vec = None
        self.products = [None] * 4
        self.product_next = 0
        self.krylov_sizes = []
        self.scal = np.zeros(256)
        self.scal_used = [i < SLOT_FIRST_FREE for i in range(256)]
        self.recording = None
        self.destroy_epoch = self.option_epoch = 0
        self.scratch = {nm: Holder(op.nrows) for nm, op in world.ops.items()}
        c = world.coarse
        import scipy.sparse as sp
        self.Cinv = np.linalg.inv(sp.csr_matrix((c[2], c[1], c[0]), shape=(world.nc, world.nc)).toarray())
        self.deviations = []
        self.call_index = 0

    def deviate(self):
        self.deviations.append(self.call_index)

    # ---- plumbing --------------------------------------------------------------------------
    def tail_stats(self):
        return self.tail_flushes, self.tail_commands

    def tail_enabled(self):
        return bool(self.opt["coarse_tail"]) and self.recording is None and not self.tail_hold

    def _dev(self, fn):
        """Device work that is not a kernel launch (memset, memcpy)."""
        if self.recording is not None:
            self.recording.ops.append(fn)
        else:
            fn()

    def _launch(self, fn, defer=False):
        if defer:
            self.tail.append(fn)
            return
        self.tail_flush()
        self._dev(fn)
        self.launches += 1

    def tail_flush(self):
        if not self.tail:
            return
        ops, self.tail = self.tail, []
        for fn in ops:
            fn()
        self.launches += 1
        self.tail_flushes += 1
        self.tail_commands += len(ops)

    def guard_defer(self):
        self.lazy_flush()

    def guard(self):
        self.lazy_flush()
        self.tail_flush()

    def touch(self, *vs):
        g = self.recording
        if g is None:
            return
        for v in vs:
            self.touch_slot(v)
            v.in_graph = True

    def touch_slot(self, obj):
        g = self.recording
        if any(s[0] is obj for s in g.slots):
            return
        g.slots.append([obj, obj.ptr, obj.zero_pending, None, None])

    def hold(self, *vs):
        return any(not v.owned or v.escaped for v in vs)

    def materialize(self, v):
        if v.scale_pending:
            self.lazy_flush()
        if v.zero_pending:
            self.tail_flush()
            buf = v.ptr
            self._dev(lambda: buf.fill(0))
            v.zero_pending = False

    def rd(self, v):
        self.materialize(v)
        return v.ptr

    def wr(self, v):
        v.zero_pending = False
        v.gen += 1
        return v.ptr

    def mut(self, v):
        v.gen += 1
        return v.ptr

    # ---- products --------------------------------------------------------------------------
    def product_wanted(self, n):
        return n in self.krylov_sizes

    def product_take_slot(self):
        k = self.product_next
        self.product_next = (k + 1) & 3
        self.products[k] = None
        return SLOT_PRODUCT0 + k

    def product_record(self, a, b, slot):
        if a.escaped or b.escaped:
            return
        self.products[slot - SLOT_PRODUCT0] = (a, b, a.gen, b.gen, slot)
        if self.recording is not None:
            self.recording.products.append((a, b, slot))

    def product_lookup(self, a, b):
        for p in self.products:
            if p is None:
                continue
            if (p[0] is a and p[1] is b and p[2] == a.gen and p[3] == b.gen) or \
               (p[0] is b and p[1] is a and p[2] == b.gen and p[3] == a.gen):
                return p[4]
        return -1

    # ---- vectors ---------------------------------------------------------------------------
    def vec(self, n, f32=False):
        require(self.recording is None, "vector creation while recording")
        self.guard()
        return FVec(n, f32)

    def wrap(self, n):
        return FVec(n, buf=np.zeros(n))

    def caller_view(self, v):
        return v.caller.copy()

    def destroy(self, v):
        if self.lazy_vec is v:
            self.lazy_vec = None
            v.scale_pending = False
        self.products = [None if p is not None and (p[0] is v or p[1] is v) else p for p in self.products]
        if v.in_graph:
            self.destroy_epoch += 1
        self.guard()

    def upload(self, v, a):
        require(self.recording is None, "host transfer: not allowed while a graph is being recorded")
        self.guard()
        v.ptr[:] = rnd(a, v.f32)
        v.zero_pending = False
        v.gen += 1

    def download(self, v):
        require(self.recording is None, "host transfer: not allowed while a graph is being recorded")
        self.guard()
        if v.zero_pending:
            return np.zeros(v.n)
        self.materialize(v)
        return v.ptr.astype(np.float64)

    def flush(self):
        self.guard()

    def sync(self):
        require(self.recording is None, "sync while recording")
        self.guard()

    def clear(self, x):
        self.touch(x)
        if x.scale_pending:
            x.scale_pending = False
            x.sc = None
            if self.lazy_vec is x:
                self.lazy_vec = None
        x.gen += 1
        if self.opt["zero_shortcut"] and x.owned and not x.escaped:
            x.zero_pending = True
            return
        self.guard()
        x.zero_pending = True
        self.materialize(x)

    def copy(self, x, y):
        self.touch(x, y)
        require(x.n == y.n, "copy: size mismatch")
        if x is y or x.ptr is y.ptr:
            return
        if x.zero_pending:
            return self.clear(y)
        self.guard()
        px, py = x.ptr, self.wr(y)
        self._launch(lambda: py.__setitem__(slice(None), px.astype(py.dtype)))

    def _ew(self, out, f, ins, reads_out):
        """out = f(*inputs[, out]) in the output's precision (one kernel)."""
        ps = [self.rd(v) for v in ins]
        po = self.rd(out) if reads_out else None
        po = self.mut(out) if reads_out else self.wr(out)
        ty = np.float32 if out.f32 else np.float64
        srcs = ps + ([po] if reads_out else [])
        self._launch(lambda: po.__setitem__(slice(None), rnd(f(*[s.astype(ty) for s in srcs]), out.f32)))

    def axpby(self, a, x, b, y):
        self.touch(x, y)
        require(x.n == y.n, "axpby: size mismatch")
        require(x.f32 == y.f32, "axpby: unsupported precision combination")
        self.guard()
        T = np.float32 if y.f32 else np.float64
        if b == 0.0 or y.zero_pending:
            return self._ew(y, lambda xv: T(a) * xv, [x], False)
        self._ew(y, lambda xv, yv: T(a) * xv + T(b) * yv, [x], True)

    def axpbypcz(self, a, x, b, y, c, z):
        self.touch(x, y, z)
        require(x.n == y.n == z.n, "axpbypcz: size mismatch")
        self.guard()
        if c == 0.0 or z.zero_pending:
            return self._ew(z, lambda xv, yv: a * xv + b * yv, [x, y], False)
        self._ew(z, lambda xv, yv, zv: a * xv + b * yv + c * zv, [x, y], True)

    def vmul(self, a, x, y, b, z):
        self.touch(x, y, z)
        require(x.n == y.n == z.n, "vmul: size mismatch")
        self.guard()
        if b == 0.0 or z.zero_pending:
            return self._ew(z, lambda xv, yv: a * xv * yv, [x, y], False)
        self._ew(z, lambda xv, yv, zv: a * xv * yv + b * zv, [x, y], True)

    def _sum(self, a, b):
        return float(np.sum(a.astype(LD) * b.astype(LD)))

    def launch_dot(self, x, y, slot):
        px, py = self.rd(x), self.rd(y)
        self._launch(lambda: self.scal.__setitem__(slot, self._sum(px, py)))

    def dot(self, x, y):
        require(self.recording is None, "dot (host-synchronous): not allowed while a graph is being recorded")
        require(x.n == y.n, "dot: size mismatch")
        require(x.f32 == y.f32, "dot: unsupported precision combination")
        self.guard()
        if x.zero_pending or y.zero_pending:
            return 0.0
        if x.f32:
            px, py = self.rd(x), self.rd(y)
            self._launch(lambda: None)
            return self._sum(px, py)
        have = self.product_lookup(x, y)
        if have >= 0:
            return float(self.scal[have])
        self.launch_dot(x, y, SLOT_DOT)
        return float(self.scal[SLOT_DOT])

    # ---- CSR passes ------------------------------------------------------------------------
    def op(self, name):
        return self.w.ops[name]

    def tail_accepts(self, A):
        return self.tail_enabled() and not A.f32 and A.k.sum() <= self.opt["tail_max_nnz"]

    def fusable(self, A):
        o = self.opt
        return (o["fuse_first_sweep"] and o["zero_shortcut"] and o["spmv_variant"] == 1 and not A.f32
                and not self.tail_enabled())

    def spmv(self, a, name, x, b, y, dot_w=None, dot_slots=()):
        A = self.op(name)
        self.touch(x, y)
        require(x.n == A.ncols and y.n == A.nrows, "spmv: size mismatch")
        require(x is not y and x.ptr is not y.ptr, "spmv: x and y must not alias")
        self.guard_defer()
        self.tail_hold += self.hold(x, y)
        try:
            px = self.rd(x)
            acc_ = not (b == 0.0 or y.zero_pending)
            py = self.mut(y) if acc_ else self.wr(y)
            pw = dot_w

            def k():
                S = A.S(px)
                v = LD(a) * S + (LD(b) * py.astype(LD) if acc_ else 0)
                py[:] = rnd(v)
                for j, s in enumerate(dot_slots):
                    self.scal[s] = self._sum(py, pw if j == 0 else py)
            self._launch(k, defer=not dot_slots and self.tail_accepts(A))
        finally:
            self.tail_hold -= self.hold(x, y)

    def residual(self, f, name, x, r, dot_slot=None):
        A = self.op(name)
        self.touch(f, x, r)
        require(x.n == A.ncols and f.n == A.nrows and r.n == A.nrows, "residual: size mismatch")
        require(x is not r and x.ptr is not r.ptr, "residual: x and r must not alias")
        self.tail_hold += self.hold(f, x, r)
        try:
            lv = self.lazy_vec
            if lv is not None:
                if (lv is x and x.sc[2] is f and f is not r and x is not r and r.ptr is not x.ptr
                        and r.ptr is not f.ptr and self.fusable(A) and dot_slot is None and r.owned
                        and not r.escaped and f.ptr is x.sc[1] and not f.zero_pending):
                    self.lazy_vec = None
                    x.scale_pending = False
                    pd, pf, _, om = x.sc
                    x.sc = None
                    px, py = x.ptr, self.wr(r)

                    def k():
                        px[:] = rnd((om * pd) * pf)
                        py[:] = rnd(pf.astype(LD) - A.S(px))
                    return self._launch(k)
                self.lazy_flush()
            px, pf = self.rd(x), self.rd(f)
            py = self.mut(r) if f is r else self.wr(r)

            def k():
                py[:] = rnd(pf.astype(LD) - A.S(px))
                if dot_slot is not None:
                    self.scal[dot_slot] = self._sum(py, py)
            self._launch(k, defer=dot_slot is None and self.tail_accepts(A))
        finally:
            self.tail_hold -= self.hold(f, x, r)

    def lazy_flush(self):
        v = self.lazy_vec
        if v is None:
            return
        self.lazy_vec = None
        v.scale_pending = False
        pd, pf, _, om = v.sc
        v.sc = None
        self.relax_zero(v, pd, pf, om)

    def relax_zero(self, x, pd, pf, om):
        px = self.wr(x)
        x.zero_pending = False
        defer = not x.f32 and self.tail_enabled() and x.n <= self.opt["tail_max_vec"]
        self._launch(lambda: px.__setitem__(slice(None), rnd(rnd(om * pd.astype(np.float64)) * pf)), defer=defer)

    def relax(self, name, rhs, x, tmp, d, om):
        A = self.op(name)
        self.touch(rhs, x, tmp, d)
        require(x.n == A.nrows == rhs.n == d.n == tmp.n, "relax: vector size != matrix rows")
        require(x is not tmp and x is not rhs and tmp is not rhs, "relax: x, tmp and rhs must be distinct vectors")
        require(x.ptr is not tmp.ptr, "relax: x and tmp must not alias")
        self.guard_defer()
        self.tail_hold += self.hold(rhs, x, tmp, d)
        try:
            return self._relax(A, name, rhs, x, tmp, d, om)
        finally:
            self.tail_hold -= self.hold(rhs, x, tmp, d)

    def _relax(self, A, name, rhs, x, tmp, d, om):
        mix = 2 if A.f32 else 0
        pf, pd = self.rd(rhs), self.rd(d)
        if x.zero_pending and self.opt["zero_shortcut"]:
            if mix == 0 and self.fusable(A) and x.owned and not x.escaped:
                x.zero_pending = False
                x.scale_pending = True
                x.sc = (pd, pf, rhs, om)
                x.gen += 1
                self.lazy_vec = x
                return
            return self.relax_zero(x, pd, pf, om)
        if not self.opt["fuse_relax"]:
            self.residual(rhs, name, x, tmp)
            return self.vmul(om, d, tmp, 1.0, x)
        px = self.rd(x)
        if mix == 2:
            h = self.scratch[name]
            if self.recording is not None:
                self.touch_slot(h)
            py = h.ptr
        else:
            py = self.wr(tmp)
        pslot = self.product_take_slot() if self.product_wanted(A.nrows) else None

        def k():
            v = px.astype(LD) + LD(om) * pd.astype(LD) * (pf.astype(LD) - A.S(px))
            py[:] = rnd(v)
            if pslot is not None:
                self.scal[pslot] = self._sum(pf, py)
        self._launch(k, defer=pslot is None and mix == 0 and self.tail_accepts(A))
        x.gen += 1
        self.sweep_swap(x, tmp, h if mix == 2 else None)
        if pslot is not None:
            self.product_record(rhs, x, pslot)

    def sweep_swap(self, x, tmp, h):
        if h is not None:
            if x.owned:
                x.ptr, h.ptr = h.ptr, x.ptr
            else:
                self.tail_flush()
                src, dst = h.ptr, x.ptr
                self._dev(lambda: dst.__setitem__(slice(None), src))
        elif x.owned and tmp.owned:
            x.ptr, tmp.ptr = tmp.ptr, x.ptr
        else:
            self.tail_flush()
            src, dst = tmp.ptr, x.ptr
            self._dev(lambda: dst.__setitem__(slice(None), src))

    def coarse_solve(self, f, x):
        self.touch(f, x)
        require(f.n == x.n == self.w.nc, "coarse solve: size mismatch")
        require(f is not x and f.ptr is not x.ptr, "coarse solve: rhs and x must not alias")
        self.guard_defer()
        self.tail_hold += self.hold(f, x)
        try:
            pr = self.rd(f)
            defer = self.tail_enabled() and self.w.nc ** 2 <= 4 * self.opt["tail_max_nnz"]
            px = self.wr(x)
            C = self.Cinv
            self._launch(lambda: px.__setitem__(slice(None), rnd(C.astype(LD) @ pr.astype(LD))), defer=defer)
        finally:
            self.tail_hold -= self.hold(f, x)

    def gather(self, src, dst):
        self.touch(src, dst)
        self.guard()
        ps, idx = self.rd(src), self.w.index
        pd = self.wr(dst)
        self._launch(lambda: pd.__setitem__(slice(None), ps[idx]))

    def scatter(self, src, dst):
        self.touch(src, dst)
        self.guard()
        ps, idx = self.rd(src), self.w.index
        self.rd(dst)
        pd = self.mut(dst)
        self._launch(lambda: pd.__setitem__(idx, ps))

    # ---- graphs ------------------------------------------------------------------------------
    def graph_begin(self):
        require(self.recording is None, "graph_begin: already recording")
        self.guard()
        self.recording = FGraph(self)
        return True

    def graph_rollback(self, g):
        for s in g.slots:
            s[0].ptr = s[1]
            if s[0].zero_pending is not None:
                s[0].zero_pending = s[2]
                s[0].gen += 1

    def graph_abort(self):
        g = self.recording
        if g is None:
            return
        self.guard()
        self.graph_rollback(g)
        self.launches = g.launches0
        self.recording = None

    def graph_end(self):
        g = self.recording
        require(g is not None, "graph_end: not recording")
        self.guard()
        self.recording = None
        for fn in g.ops:
            fn()
        for s in g.slots:
            s[3], s[4] = s[0].ptr, s[0].zero_pending
        g.launches = self.launches - g.launches0
        return g

    def graph_matches(self, g):
        return all(s[0].ptr is s[1] and (s[0].zero_pending is None or s[0].zero_pending == s[2]) for s in g.slots)

    def graph_launch(self, g):
        require(self.recording is None, "graph_launch: a graph is being recorded")
        if g.destroy_epoch != self.destroy_epoch or g.option_epoch != self.option_epoch:
            return False
        if not self.graph_matches(g):
            return False
        self.guard()
        for fn in g.ops:
            fn()
        for s in g.slots:
            s[0].ptr = s[3]
            if s[0].zero_pending is not None:
                s[0].zero_pending = s[4]
                s[0].gen += 1
        for a, b, slot in g.products:
            self.product_record(a, b, slot)
        self.launches += g.launches
        return True

    def graph_destroy(self, g):
        self.guard()

    # ---- Krylov ------------------------------------------------------------------------------
    def krylov(self, n):
        require(self.recording is None, "Krylov workspace creation while recording")
        for first in range(SLOT_FIRST_FREE, 256 - K_NSLOTS):
            if not any(self.scal_used[first:first + K_NSLOTS]):
                self.scal_used[first:first + K_NSLOTS] = [True] * K_NSLOTS
                self.krylov_sizes.append(n)
                return FKrylov(n, first)
        raise FakeError("scalar table exhausted")

    def krylov_destroy(self, K):
        self.scal_used[K.base:K.base + K_NSLOTS] = [False] * K_NSLOTS
        self.krylov_sizes.remove(K.n)

    def _kcheck(self, K, *vs):
        require(self.recording is None, "Krylov step: not allowed while a graph is being recorded")
        require(all(not v.f32 and v.n == K.n for v in vs), "Krylov step: FP64 vectors of the workspace's size expected")

    def k_residual(self, K, f, name, x, r):
        self._kcheck(K, f, x, r)
        self.guard()
        K.first, K.parity = True, 0
        slot = K.base + K_RR
        if x.zero_pending and self.opt["zero_shortcut"] and r is not f:
            pf = self.rd(f)
            pr = self.wr(r)

            def k():
                pr[:] = pf
                self.scal[slot] = self._sum(pf, pf)
            self._launch(k)
        else:
            self.residual(f, name, x, r, dot_slot=slot)
        return float(self.scal[slot])

    def k_scalars(self, K):
        self._kcheck(K)
        self.guard()
        rel = [K_RHOP0 + K.parity, K_QP, K_ALPHA, K_TS, K_TT, K_OMEGA, K_RR, K_SS, K_RHO_NEXT]
        return dict(zip(("rho", "qp", "alpha", "ts", "tt", "omega", "rr", "ss", "rho_next"),
                        [float(self.scal[K.base + i]) for i in rel]))

    def rho_prev_slot(self, K):
        return K.base + K_RHOP0 + K.parity

    def cg_direction(self, K, r, s, p):
        self._kcheck(K, r, s, p)
        require(s is not p and s.ptr is not p.ptr, "cg_direction: s and p must be distinct")
        self.guard()
        rho = self.product_lookup(r, s)
        if rho < 0:
            rho = K.base + K_RHO
            self.launch_dot(r, s, rho)
        ps = self.rd(s)
        first = K.first
        pp = None if first else self.rd(p)
        prev, save = self.rho_prev_slot(K), K.base + K_RHOP0 + (K.parity ^ 1)
        out = self.wr(p) if first else self.mut(p)

        def k():
            r1 = self.scal[rho]
            self.scal[save] = r1
            if first:
                out[:] = ps
            else:
                out[:] = ps + (r1 / self.scal[prev]) * pp
        self._launch(k)
        K.parity ^= 1
        K.first = False

    def cg_step(self, K, name, p, q, x, r):
        self._kcheck(K, p, q, x, r)
        require(not K.first, "cg_step: call b200_cg_direction first")
        self.guard()
        qp = K.base + K_QP
        self.rd(p)
        self.spmv(1.0, name, p, 0.0, q, dot_w=p.ptr, dot_slots=(qp,))
        pp, pq, px, pr = self.rd(p), self.rd(q), self.rd(x), self.rd(r)
        self.mut(x), self.mut(r)
        rho, al, rr = K.base + K_RHOP0 + K.parity, K.base + K_ALPHA, K.base + K_RR

        def k():
            a = self.scal[rho] / self.scal[qp]
            self.scal[al] = a
            px[:] = a * pp + px
            pr[:] = -a * pq + pr
            self.scal[rr] = self._sum(pr, pr)
        self._launch(k)
        return float(self.scal[rr])

    def bicg_start(self, K, r, rh):
        self._kcheck(K, r, rh)
        require(r is not rh and r.ptr is not rh.ptr, "bicg_start: r and rh must be distinct")
        self.guard()
        pr, prh, slot = self.rd(r), self.wr(rh), K.base + K_RHO_NEXT

        def k():
            prh[:] = pr
            self.scal[slot] = self._sum(pr, pr)
        self._launch(k)
        K.first, K.parity = True, 0

    def bicg_direction(self, K, r, v, p):
        self._kcheck(K, r, v, p)
        require(r is not p and r.ptr is not p.ptr, "bicg_direction: r and p must be distinct")
        self.guard()
        first = K.first
        pr = self.rd(r)
        pv, pp = (None, None) if first else (self.rd(v), self.rd(p))
        b0 = K.base
        prev, save = self.rho_prev_slot(K), b0 + K_RHOP0 + (K.parity ^ 1)
        out = self.wr(p) if first else self.mut(p)

        def k():
            r1 = self.scal[b0 + K_RHO_NEXT]
            self.scal[save] = r1
            if first:
                out[:] = pr
            else:
                om = self.scal[b0 + K_OMEGA]
                beta = (r1 * self.scal[b0 + K_ALPHA]) / (self.scal[prev] * om)
                out[:] = pr + (-beta * om) * pv + beta * pp
        self._launch(k)
        K.parity ^= 1
        K.first = False

    def bicg_step_s(self, K, name, rh, T, v, r, s, x):
        self._kcheck(K, rh, T, v, r, s, x)
        require(not K.first, "bicg_step_s: call b200_bicg_direction first")
        self.guard()
        b0 = K.base
        self.spmv(1.0, name, T, 0.0, v, dot_w=self.rd(rh), dot_slots=(b0 + K_QP,))
        pT, px, pr, pv = self.rd(T), self.rd(x), self.rd(r), self.rd(v)
        self.mut(x)
        ps = self.wr(s)
        rho = b0 + K_RHOP0 + K.parity

        def k():
            a = self.scal[rho] / self.scal[b0 + K_QP]
            self.scal[b0 + K_ALPHA] = a
            px[:] = a * pT + px
            ps[:] = pr - a * pv
            self.scal[b0 + K_SS] = self._sum(ps, ps)
        self._launch(k)
        return float(self.scal[b0 + K_SS])

    def bicg_step_r(self, K, name, rh, T, t, s, r, x):
        self._kcheck(K, rh, T, t, s, r, x)
        self.guard()
        b0 = K.base
        ps0 = self.rd(s)
        self.spmv(1.0, name, T, 0.0, t, dot_w=ps0, dot_slots=(b0 + K_TS, b0 + K_TT))
        pT, px, ps, pt, prh = self.rd(T), self.rd(x), self.rd(s), self.rd(t), self.rd(rh)
        self.mut(x)
        pr = self.wr(r)

        def k():
            om = self.scal[b0 + K_TS] / self.scal[b0 + K_TT]
            self.scal[b0 + K_OMEGA] = om
            px[:] = om * pT + px
            pr[:] = ps - om * pt
            self.scal[b0 + K_RR] = self._sum(pr, pr)
            self.scal[b0 + K_RHO_NEXT] = self._sum(pr, prh)
        self._launch(k)
        return float(self.scal[b0 + K_RR])


# ---- mutants: the fake wrong in one small way ---------------------------------------------------
class CopyFromZeroKeepsSweep(Fake):
    def copy(self, x, y):
        if x.zero_pending and x is not y and x.ptr is not y.ptr and y.scale_pending:
            self.deviate()
            self.touch(x, y)
            y.gen += 1
            y.zero_pending = True
            return
        Fake.copy(self, x, y)


class CopyFromZeroKeepsProducts(Fake):
    def copy(self, x, y):
        if x.zero_pending and x is not y and x.ptr is not y.ptr:
            if any(p is not None and (p[0] is y or p[1] is y) for p in self.products):
                self.deviate()
            g = y.gen
            Fake.copy(self, x, y)
            y.gen = g
            return
        Fake.copy(self, x, y)


class AbortKeepsProducts(Fake):
    def graph_abort(self):
        g = self.recording
        if g is not None and any(p is not None and (p[0], p[1], p[4]) in g.products for p in self.products):
            self.deviate()
        if g is not None:
            gens = {id(s[0]): s[0].gen for s in g.slots if s[0].zero_pending is not None}
            Fake.graph_abort(self)
            for s in g.slots:
                if id(s[0]) in gens:
                    s[0].gen = gens[id(s[0])]
            return
        Fake.graph_abort(self)


class LazyClearOfWrappedMemory(Fake):
    def clear(self, x):
        if not x.owned and self.opt["zero_shortcut"]:
            self.deviate()
            self.touch(x)
            x.gen += 1
            x.zero_pending = True
            return
        Fake.clear(self, x)


class ReplayFromAnyState(Fake):
    def graph_matches(self, g):
        ok = Fake.graph_matches(self, g)
        if not ok:
            self.deviate()
        return True


class ReplayKeepsGenerations(Fake):
    def graph_launch(self, g):
        gens = {id(s[0]): s[0].gen for s in g.slots if s[0].zero_pending is not None}
        ok = Fake.graph_launch(self, g)
        if ok:
            live = [p for p in self.products if p is not None and p not in [(a, b) for a, b, _ in g.products]]
            if any(id(p[0]) in gens or id(p[1]) in gens for p in live):
                self.deviate()
            for s in g.slots:
                if id(s[0]) in gens:
                    s[0].gen = gens[id(s[0])]
        return ok


class SweepForgetsSwap(Fake):
    def sweep_swap(self, x, tmp, h):
        if h is None and x.owned and tmp.owned:
            self.deviate()
            return
        Fake.sweep_swap(self, x, tmp, h)


class RhoPrevWrongParity(Fake):
    def rho_prev_slot(self, K):
        if not K.first:
            self.deviate()
        return K.base + K_RHOP0 + (K.parity ^ 1)


MUTANTS = [CopyFromZeroKeepsSweep, CopyFromZeroKeepsProducts, AbortKeepsProducts, LazyClearOfWrappedMemory,
           ReplayFromAnyState, ReplayKeepsGenerations, SweepForgetsSwap, RhoPrevWrongParity]


_worlds = {}


def world(i):
    if i not in _worlds:
        _worlds[i] = st.World(os.path.join(GOLDEN, FIXTURES[i] + ".npz"))
    return _worlds[i]


SEEDS = range(40)


def runner(cls, seed, **opt):
    w = world(seed % 2)
    fake = cls(w, **opt)
    return st.Runner(fake, w, seed, tail=bool(opt.get("coarse_tail"))), fake


def run(cls, seed, **opt):
    r, fake = runner(cls, seed, **opt)
    return r, fake, r.run()


def test_faithful_fake_runs_every_seed_clean_and_reaches_every_event():
    cov = collections.Counter()
    for seed in SEEDS:
        cov.update(run(Fake, seed)[2])
    missing = [e for e in st.EVENTS if cov[e] == 0]
    assert not missing, "coverage events never reached: %s\n%s" % (missing, dict(cov))


def test_faithful_fake_under_other_options():
    cov = collections.Counter()
    for opt in (dict(fuse_first_sweep=0), dict(zero_shortcut=0), dict(fuse_relax=0), dict(spmv_variant=0),
                dict(coarse_tail=1, tail_max_nnz=5000, tail_max_vec=1000)):
        for seed in range(3):
            cov.update(run(Fake, 100 + seed, **opt)[2])
    assert all(cov[e] for e in st.TAIL_EVENTS), dict(cov)


@pytest.mark.parametrize("cls", MUTANTS, ids=lambda c: c.__name__)
def test_mutant_is_rejected_at_the_call_that_broke(cls):
    """Some fixed seed rejects the mutant, and its failure names a call at which the mutant went
    its own way (an error can also surface later, through values computed from a wrong one)."""
    seen = []
    for seed in range(40):
        r, fake = runner(cls, seed)
        try:
            r.run()
        except st.Fail as e:
            msg = str(e)
            if any(("#%d " % i) in msg for i in fake.deviations):
                return
            seen.append("seed %d deviated at %s:\n%s" % (seed, fake.deviations[:10], msg))
    pytest.fail("no seed rejected %s naming a call at which it deviated\n%s" % (cls.__name__, "\n".join(seen)))
