"""Every solve-phase kernel against an extended-precision reference with per-row error bounds
(tests/_accuracy.py states the reference, the bound model and its derivation).

CSR passes run on a ragged generator with an explicit edge catalogue and on structured bands
(the compressed column formats), across modes, lane widths, both schedulers, the ring's knobs
(stages, CTAs per SM, nnz_cap), the storage formats and every precision combination the
translation units instantiate -- a covering design, not the full product.  The other
schedulers of the same arithmetic (small-operator kernel, coarse tail) must give the ring
kernel's bits.  Element-wise kernels, reductions and the coarse solver have bounds of their own.
Every test that selects a path proves that it ran (storage accessors, launch counters,
tail_stats, kernel names recorded by torch.profiler)."""
import contextlib
import ctypes
import math

import numpy as np
import pytest

import amgcl_b200 as ab
import _accuracy as acc
from _accuracy import LD
from test_gpu_primitives import _f32csr, _f32vec

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
ALPHA, BETA, OMEGA = 1.5, -0.25, 0.72
MODES = ("spmv", "spmv_acc", "resid", "relax")

# (TV, TX, TF, TY, TD) and the modes each mix is launched with (csr_launch.cuh, B200_CSR_PASSES)
PRECS = {
    "DD": ((F64, F64, F64, F64, F64), MODES),
    "FD": ((F32, F64, F64, F64, F32), MODES),
    "FF": ((F32, F32, F32, F32, F32), MODES),
    "FFD": ((F32, F32, None, F64, None), ("spmv", "spmv_acc")),
    "FDF": ((F32, F64, F64, F32, None), ("resid",)),
}
# (stages, CTAs per SM, nnz_cap).  Every ring here fits its shared-memory budget, so the stage count
# is the one requested (asserted through ring_stages): at one CTA per SM and 6144 entries per
# stage three stages fit, eight do not (ring_smem would quietly run three), so the 8-stage ring
# runs with 1024-entry stages.
KNOBS = [(1, 1, 256), (1, 4, 2048), (2, 4, 2048), (3, 2, 512), (8, 1, 1024), (3, 1, 6144)]


@pytest.fixture(autouse=True)
def _extended():
    acc.require_longdouble()


@contextlib.contextmanager
def options(ctx, **kw):
    old = {k: ctx.get_option(k) for k in kw}
    try:
        for k, v in kw.items():
            ctx.set_option(k, v)
        yield
    finally:
        for k, v in old.items():
            ctx.set_option(k, v)


FORMAT_OPTS = {
    "plain": dict(patterns=0, offsets=0, window=0),
    "pattern": dict(patterns=1, patterns_min_nnz=0, offsets=0, window=0),
    "offset": dict(patterns=0, offsets=1, offsets_min_nnz=0, window=0),
    "window": dict(patterns=0, offsets=0, window=1, window_min_nnz=0),
}


def assert_stored(A, fmt):
    on = {"pattern": A.patterns()["pattern_indexed"], "offset": A.offsets()["offset_indexed"],
          "window": A.window()["windowed"]}
    if fmt == "plain":
        assert not any(on.values()), on
    else:
        assert on[fmt], (fmt, on)


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def kernels_run(fn):
    """Names of the CUDA kernels fn() launched (torch.profiler records every launch of the
    process)."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.name for e in prof.events())


def dvec(ctx, a, dt):
    return ctx.vector(np.asarray(a, dtype=F64)) if dt == F64 else _f32vec(ctx, a)


def get(v, dt):
    return v.numpy() if dt == F64 else v.numpy32()


def upload(ctx, nr, nc, ptr, col, val, tv):
    return ctx.csr(nr, nc, ptr, col, val) if tv == F64 else _f32csr(ctx, nr, nc, ptr, col, val)


class Case:
    """One uploaded operator + its host data, reused across modes."""

    def __init__(self, ctx, ptr, col, val, x, prec="DD", seed=0):
        self.ctx, self.ptr, self.col, self.x = ctx, ptr, col, x
        self.nr, self.nc = ptr.size - 1, x.size
        (self.TV, self.TX, self.TF, self.TY, self.TD), self.modes = PRECS[prec]
        self.val = val.astype(self.TV).astype(F64)
        self.prec = prec
        self.A = upload(ctx, self.nr, self.nc, ptr, col, val, self.TV)
        pl = self.A.plan()
        self.p = acc.plan(ptr, pl["lanes"], ctx.get_option("nnz_cap"))
        assert self.p["lanes"] == pl["lanes"] and self.p["nblocks"] >= 1
        rng = np.random.default_rng(seed + 17)
        self.y0 = rng.uniform(-1, 1, self.nr)
        self.f = rng.uniform(-1, 1, self.nr) * np.exp2(rng.uniform(-10, 10, self.nr))
        self.d = rng.uniform(0.1, 1.0, self.nr)
        self.m, self.k = acc.roundings(ptr, self.p)
        self._sums = None

    def run(self, mode):
        ctx, TX, TY = self.ctx, self.TX, self.TY
        vx = dvec(ctx, self.x, TX)
        if mode in ("spmv", "spmv_acc"):
            beta = 0.0 if mode == "spmv" else BETA
            vy = dvec(ctx, self.y0 if beta else np.full(self.nr, np.nan), TY)   # beta = 0: never read
            ctx.spmv(ALPHA, self.A, vx, beta, vy)
            return get(vy, TY)
        if mode == "resid":
            vr = dvec(ctx, np.full(self.nr, np.nan), TY)
            ctx.residual(dvec(ctx, self.f, self.TF), self.A, vx, vr)
            return get(vr, TY)
        vt = dvec(ctx, np.zeros(self.nr), self.TD if self.prec == "FD" else TY)
        ctx.relax(self.A, dvec(ctx, self.f, self.TF), vx, vt, dvec(ctx, self.d, self.TD), OMEGA)
        return get(vx, TX)

    def want(self, mode, xg=None):
        """(reference, bound) of one mode, in longdouble from the operands as stored."""
        TY = self.TY
        if xg is None and self._sums is not None:
            S, M = self._sums
        else:
            xs = np.asarray(self.x if xg is None else xg).astype(self.TX).astype(TY)   # (TS)x, as summed
            S, M = acc.row_sums(self.ptr, self.col, self.val, xs)
            if xg is None:
                self._sums = S, M
        u = acc.unit(TY)
        kw = {}
        if mode == "spmv":
            kw = dict(alpha=ALPHA)
        elif mode == "spmv_acc":
            kw = dict(alpha=ALPHA, beta=BETA, y0=self.y0.astype(TY))
        elif mode == "resid":
            kw = dict(f=self.f.astype(self.TF))
        else:
            kw = dict(f=self.f.astype(self.TF), x0=self.x.astype(self.TX), omega=OMEGA, d=self.d.astype(self.TD))
        return acc.reference(mode, S, **kw), acc.bound(mode, self.m, self.k, u, M, **kw)

    def check(self, mode, got, what):
        want, bnd = self.want(mode)
        acc.assert_rows(got, want, bnd, "%s %s %s" % (what, self.prec, mode), self.ptr, self.p)
        if self.prec == "DD" and mode in ("spmv", "resid"):
            # rows of at most one entry: exact up to the epilogue
            one = self.k <= 1
            e = self.ptr[:-1][one]
            has = self.k[one] == 1
            prod = np.where(has, self.val[np.minimum(e, self.val.size - 1)] *
                            self.x[self.col[np.minimum(e, self.col.size - 1)]], 0.0)
            exact = ALPHA * prod if mode == "spmv" else self.f[one] - prod
            assert np.array_equal(got[one], exact), "%s: a row of <= 1 entry is not exact" % what

    def check_all(self, what, modes=None):
        for mode in modes or self.modes:
            if mode == "relax" and self.nr != self.nc:
                continue
            self.check(mode, self.run(mode), what)


def ragged(nr, nc, cap=2048, seed=0, long_blocks=True):
    return acc.ragged_csr(nr, nc, nnz_cap=cap, seed=seed, long_blocks=long_blocks)


BAND_OFFS = [-41, -40, -3, -1, 0, 1, 3, 40, 41]


# ---------------------------------------------------------------------------------------------
# CSR passes: modes x lanes x scheduler at the default knobs
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 0])
@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 16, 32])
def test_modes_all_lane_widths(ctx, lanes, variant):
    with options(ctx, lanes=lanes, spmv_variant=variant, **FORMAT_OPTS["plain"]):
        for nr, nc in ((4099, 4099), (4098, 3001), (3805, 5003)):
            ptr, col, val, x = ragged(nr, nc, seed=lanes * 10 + variant + nr)
            c = Case(ctx, ptr, col, val, x, seed=nr)
            assert c.A.plan()["lanes"] == lanes and c.A.plan()["long_blocks"] >= 2
            names = kernels_run(lambda: c.check_all("lanes=%d variant=%d %dx%d" % (lanes, variant, nr, nc)))
            assert ("csr_ring_kernel" if variant else "csr_block_kernel") in names


@pytest.mark.parametrize("lanes", [1, 2, 4])
def test_fused_first_sweep(ctx, lanes):
    """clear -> relax -> residual of the same system is one pass (MODE_RESID_SCALED): x is
    written exactly as relax_zero_kernel writes it, r within the residual bound."""
    with options(ctx, lanes=lanes, spmv_variant=1, fuse_first_sweep=1, coarse_tail=0, **FORMAT_OPTS["plain"]):
        ptr, col, val, x = ragged(4098, 4098, seed=40 + lanes, long_blocks=False)
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        assert c.A.plan()["long_blocks"] == 0
        vf, vd = ctx.vector(c.f), ctx.vector(c.d)
        vx, vt, vr = ctx.vector(c.nr), ctx.vector(c.nr), ctx.vector(c.nr)
        ctx.clear(vx)
        l0 = ctx.launches
        ctx.relax(c.A, vf, vx, vt, vd, OMEGA)
        ctx.residual(vf, c.A, vx, vr)
        assert ctx.launches - l0 == 1, "the first sweep was not fused into the residual"
        xh = vx.numpy()
        assert np.array_equal(xh, (OMEGA * c.d) * c.f)
        S, M = acc.row_sums(ptr, col, c.val, xh)
        acc.assert_rows(vr.numpy(), c.f - S, acc.bound("resid", c.m, c.k, acc.U64, M, f=c.f),
                        "fused first sweep", ptr, c.p)


@pytest.mark.parametrize("lanes", [1, 8, 32])
def test_in_kernel_scalars(ctx, lanes):
    """<q,p> of cg_step, <t,s> and <t,t> of bicg_step_r, <r,r> of Krylov.residual and the
    sweep's <rhs, x_new>, each against the sum over the vectors the GPU produced."""
    with options(ctx, lanes=lanes, spmv_variant=1, coarse_tail=0, **FORMAT_OPTS["plain"]):
        n = 4099
        ptr, col, val, x = ragged(n, n, seed=60 + lanes)
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        pl = c.A.plan()
        csb = lambda s: acc.csr_scalar_bound(s, pl["blocks"], c.p["rows_cap"], lanes, sms(),
                                             ctx.get_option("ctas_per_sm"))
        K = ab.Krylov(ctx, n)
        try:
            rng = np.random.default_rng(lanes)
            vf, vx = ctx.vector(c.f), ctx.vector(x)
            r, s, p, q = (ctx.vector(n) for _ in range(4))
            rr = K.residual(vf, c.A, vx, r)
            rh = r.numpy()
            c.check("resid", rh, "Krylov.residual")
            S, A = acc.dot_ref(rh, rh)
            acc.assert_scalar(rr, S, csb(A), "<r,r> of Krylov.residual")
            s.upload(rng.uniform(-1, 1, n))
            K.cg_direction(r, s, p)
            l0 = ctx.launches
            K.cg_step(c.A, p, q, vx, r)
            assert ctx.launches - l0 == 2, "q = A p and <q,p> took a separate reduction"
            qh, ph = q.numpy(), p.numpy()
            want, bnd = c.want("spmv", ph)
            acc.assert_rows(qh, want / LD(ALPHA), bnd / ALPHA, "cg_step q", ptr, c.p)
            S, A = acc.dot_ref(qh, ph)
            acc.assert_scalar(K.scalars()["qp"], S, csb(A), "<q,p> of cg_step")
            # BiCGStab: t = A T with <t,s>, <t,t>
            T, t, s2, rh2 = ctx.vector(rng.uniform(-1, 1, n)), ctx.vector(n), ctx.vector(rng.uniform(-1, 1, n)), ctx.vector(n)
            K.bicg_start(r, rh2)
            Th, sh = T.numpy(), s2.numpy()
            K.bicg_step_r(c.A, rh2, T, t, s2, r, vx)
            th = t.numpy()
            want, bnd = c.want("spmv", Th)
            acc.assert_rows(th, want / LD(ALPHA), bnd / ALPHA, "bicg_step_r t", ptr, c.p)
            sc = K.scalars()
            S, A = acc.dot_ref(th, sh)
            acc.assert_scalar(sc["ts"], S, csb(A), "<t,s> of bicg_step_r")
            S, A = acc.dot_ref(th, th)
            acc.assert_scalar(sc["tt"], S, csb(A), "<t,t> of bicg_step_r")
            # the sweep leaves <rhs, x_new> behind while a Krylov solver of its size lives
            vxx, vt, vd = ctx.vector(x), ctx.vector(n), ctx.vector(c.d)
            ctx.relax(c.A, vf, vxx, vt, vd, OMEGA)
            l0 = ctx.launches
            got = ctx.dot(vf, vxx)
            assert ctx.launches == l0, "<rhs, x_new> was not produced by the sweep"
            xn = vxx.numpy()
            c.check("relax", xn, "sweep with <rhs,x>")
            S, A = acc.dot_ref(c.f, xn)
            acc.assert_scalar(got, S, csb(A), "<rhs, x_new> of the sweep")
        finally:
            K.close()


# ---------------------------------------------------------------------------------------------
# ring knobs, formats, precisions
# ---------------------------------------------------------------------------------------------
def ring_stages(fmt, rows_cap, cap, val_size, stages, ctas):
    """Stages the ring kernel really runs (csr_launch.cuh ring_smem over csr_kernels.cuh
    stage_layout): fewer than requested when they do not fit the CTA's shared memory."""
    r16 = lambda b: (b + 15) & ~15
    stage = (r16(cap * val_size + 16) + {"plain": r16((cap + 8) * 4), "offset": r16(cap + 32), "pattern": 0}[fmt]
             + r16((rows_cap + 4) * 4) + (r16(rows_cap + 32) if fmt == "pattern" else 0))
    extra = {"plain": 0, "offset": 256 * 4, "pattern": 1024 * 4 + (257 * 2 + 15) // 16 * 16}[fmt]
    budget = 228 * 1024 // ctas - 1024 - 1536
    s = stages
    while s > 1 and 448 + s * stage + extra > budget:
        s -= 1
    return s


def walks_the_ring(c, knobs, fmt):
    """Every CTA owns more than 2 * stages blocks, so the ring refills every stage and the
    parity flips (csr_ring_kernel: `i + nstages < mine`); and the requested stages all fit."""
    stages, ctas, cap = knobs
    blocks = c.A.plan()["blocks"]
    grid = min(blocks, sms() * ctas)
    assert -(-blocks // grid) > 2 * stages, (blocks, grid, stages)
    if fmt != "window":
        assert ring_stages(fmt, c.p["rows_cap"], cap, 8, stages, ctas) == stages


def sized(make, knobs, lanes, residue):
    """make(nr) -> operator; nr (= residue mod 4) large enough for > 2 * stages blocks per CTA
    (estimated from the plan of a 20000-row sample, with a margin)."""
    stages, ctas, cap = knobs
    need = 2 * stages * sms() * ctas + 1
    sample = make(20001)
    per = 20001 / acc.plan(sample[0], lanes, cap)["nblocks"]
    nr = max(4 * int(math.ceil(need * per * 1.25 / 4)) + residue, 4 * 1000 + residue)
    while True:
        op = make(nr)
        have = acc.plan(op[0], lanes, cap)["nblocks"]
        if have >= need:
            return op
        nr = 4 * int(math.ceil(nr * need / have * 1.1 / 4)) + residue


@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: "S%d-C%d-cap%d" % k)
def test_ring_knobs_plain(ctx, knobs):
    stages, ctas, cap = knobs
    with options(ctx, stages=stages, ctas_per_sm=ctas, nnz_cap=cap, spmv_variant=1, **FORMAT_OPTS["plain"]):
        for i, lanes in enumerate((1, 2, 32)):
            with options(ctx, lanes=lanes):
                ptr, col, val, x = sized(lambda nr: ragged(nr, nr, cap=cap, seed=cap + lanes + stages),
                                         knobs, lanes, 1 + i)
                c = Case(ctx, ptr, col, val, x, seed=lanes)
                assert c.A.plan()["long_blocks"] >= 2
                walks_the_ring(c, knobs, "plain")
                c.check_all("stages=%d ctas=%d cap=%d lanes=%d" % (stages, ctas, cap, lanes))


@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: "S%d-C%d-cap%d" % k)
@pytest.mark.parametrize("fmt", ["pattern", "offset", "window"])
def test_ring_knobs_compressed(ctx, knobs, fmt):
    """The decoupled refill (pattern / offset: the last warp refills a stage) and the windowed
    block barrier on rings of 1, 2, 3 and 8 stages, one to four CTAs per SM each walking more
    than 2 * stages blocks, 256..6144 entries per block."""
    stages, ctas, cap = knobs
    i = KNOBS.index(knobs)
    keep = 1.0 if fmt == "pattern" else 0.9
    skew = (0, 997, 0, -997)[i % 4]                     # square, wide, square, tall
    with options(ctx, stages=stages, ctas_per_sm=ctas, nnz_cap=cap, spmv_variant=1, lanes=0, **FORMAT_OPTS[fmt]):
        ptr, col, val, x = sized(lambda nr: acc.band_csr(nr, nr + skew, BAND_OFFS, seed=nr + cap, keep=keep),
                                 knobs, 0, 1 + i % 3)
        nr, nc = ptr.size - 1, x.size
        c = Case(ctx, ptr, col, val, x, seed=nr)
        # a 6144-entry stage leaves no shared memory for a block's window beside two stages
        # (csr_upload sizes windows for 4 CTAs per SM): such an operator stays plain
        assert_stored(c.A, "plain" if fmt == "window" and cap > 2048 else fmt)
        walks_the_ring(c, knobs, "plain" if fmt == "window" and cap > 2048 else fmt)
        c.check_all("%s stages=%d ctas=%d cap=%d %dx%d" % (fmt, stages, ctas, cap, nr, nc))
        if nr == nc:
            # and the fused first sweep on the compressed format
            vf, vd = ctx.vector(c.f), ctx.vector(c.d)
            vx, vt, vr = ctx.vector(nr), ctx.vector(nr), ctx.vector(nr)
            ctx.clear(vx)
            l0 = ctx.launches
            ctx.relax(c.A, vf, vx, vt, vd, OMEGA)
            ctx.residual(vf, c.A, vx, vr)
            assert ctx.launches - l0 == 1
            xh = vx.numpy()
            assert np.array_equal(xh, (OMEGA * c.d) * c.f)
            S, M = acc.row_sums(ptr, col, c.val, xh)
            acc.assert_rows(vr.numpy(), c.f - S, acc.bound("resid", c.m, c.k, acc.U64, M, f=c.f),
                            "%s fused first sweep" % fmt, ptr, c.p)


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("lanes", [1, 4, 32])
def test_precisions_plain(ctx, prec, lanes):
    with options(ctx, lanes=lanes, spmv_variant=1, **FORMAT_OPTS["plain"]):
        ptr, col, val, x = ragged(4099, 4099, seed=80 + lanes)
        c = Case(ctx, ptr, col, val, x, prec=prec, seed=lanes)
        assert c.A.plan()["long_blocks"] >= 2
        c.check_all("plain lanes=%d" % lanes)


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("fmt", ["pattern", "offset", "window"])
def test_precisions_compressed(ctx, prec, fmt):
    with options(ctx, spmv_variant=1, lanes=0, **FORMAT_OPTS[fmt]):
        ptr, col, val, x = acc.band_csr(9001, 9001, BAND_OFFS, seed=90, keep=1.0)
        c = Case(ctx, ptr, col, val, x, prec=prec, seed=3)
        assert_stored(c.A, fmt)
        c.check_all(fmt)


# ---------------------------------------------------------------------------------------------
# the other schedulers of the same arithmetic give the ring kernel's bits
# ---------------------------------------------------------------------------------------------
def _all_modes(c):
    return np.concatenate([np.asarray(c.run(m), dtype=F64) for m in MODES])


@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 16, 32])
def test_schedulers_are_bit_identical(ctx, lanes):
    with options(ctx, lanes=lanes, **FORMAT_OPTS["plain"]):
        ptr, col, val, x = ragged(3803, 3803, seed=100 + lanes, long_blocks=False)
        c = Case(ctx, ptr, col, val, x, seed=lanes)
        assert c.A.plan()["long_blocks"] == 0
        with options(ctx, spmv_variant=1):
            ring = _all_modes(c)
            for m in MODES:
                c.check(m, c.run(m), "ring lanes=%d" % lanes)
        with options(ctx, spmv_variant=0):
            assert "csr_block_kernel" in kernels_run(lambda: np.testing.assert_array_equal(_all_modes(c), ring))
        with options(ctx, spmv_variant=1, small_kernel_max_nnz=1 << 40):
            names = kernels_run(lambda: np.testing.assert_array_equal(_all_modes(c), ring))
            assert "small_csr_kernel" in names and "csr_ring_kernel" not in names
        with options(ctx, spmv_variant=1, coarse_tail=1, tail_max_nnz=1 << 40, tail_max_vec=1 << 40):
            f0, c0 = ctx.tail_stats()
            got = _all_modes(c)
            f1, c1 = ctx.tail_stats()
            assert c1 - c0 == len(MODES) and f1 - f0 >= 1, "the calls were not deferred into the tail"
            np.testing.assert_array_equal(got, ring)


def test_tail_and_small_kernel_refuse_long_blocks(ctx):
    with options(ctx, lanes=4, spmv_variant=1, **FORMAT_OPTS["plain"]):
        ptr, col, val, x = ragged(4099, 4099, seed=7)
        c = Case(ctx, ptr, col, val, x)
        assert c.A.plan()["long_blocks"] >= 2
        ring = _all_modes(c)
        with options(ctx, small_kernel_max_nnz=1 << 40, coarse_tail=1, tail_max_nnz=1 << 40):
            f0, c0 = ctx.tail_stats()
            names = kernels_run(lambda: np.testing.assert_array_equal(_all_modes(c), ring))
            assert ctx.tail_stats()[1] == c0
            assert "small_csr_kernel" not in names and "csr_ring_kernel" in names


@pytest.mark.parametrize("mix", ["DD", "FF", "FD"])
def test_relax_from_zero_is_exact(ctx, mix):
    """relax_zero_kernel: x = fma(TX(omega*d), TX(f), 0) == numpy's (omega*d)*f in the same types."""
    n = 100003
    rng = np.random.default_rng(5)
    d, f = rng.uniform(0.1, 1.0, n), rng.uniform(-1, 1, n) * np.exp2(rng.uniform(-30, 30, n))
    TD, TF, TX = {"DD": (F64, F64, F64), "FF": (F32, F32, F32), "FD": (F32, F64, F64)}[mix]
    ptr, col, val = np.arange(n + 1, dtype=np.int64), np.arange(n, dtype=np.int64), np.ones(n)
    A = upload(ctx, n, n, ptr, col, val, F64 if mix == "DD" else F32)
    want = (TX(OMEGA * d.astype(TD).astype(F64)) if TX == F64 else (OMEGA * d.astype(TD).astype(F64)).astype(F32)) \
        * f.astype(TF).astype(TX)
    with options(ctx, fuse_first_sweep=0, coarse_tail=0):
        vx = dvec(ctx, np.zeros(n), TX)
        ctx.clear(vx)
        tmp = dvec(ctx, np.zeros(n), TD if mix == "FD" else TX)
        vf, vd = dvec(ctx, f, TF), dvec(ctx, d, TD)
        # (a full sweep from x = 0 would give the same bits: the library's per-launch profile
        # tells the two apart)
        ctx.profile_begin()
        try:
            ctx.relax(A, vf, vx, tmp, vd, OMEGA)
        finally:
            ran = [e["mode"] for e in ctx.profile_end()]
        assert ran == ["relax_zero"], ran
        got = get(vx, TX)
    assert np.array_equal(got, want)
    if mix == "DD":
        # and its coarse-tail command
        with options(ctx, fuse_first_sweep=0, coarse_tail=1, tail_max_vec=1 << 40):
            c0 = ctx.tail_stats()[1]
            vx2 = ctx.vector(n)
            ctx.clear(vx2)
            ctx.relax(A, ctx.vector(f), vx2, ctx.vector(n), ctx.vector(d), OMEGA)
            got = vx2.numpy()                          # (flushes the deferred command)
            assert ctx.tail_stats()[1] == c0 + 1
            assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------
# element-wise kernels and reductions
# ---------------------------------------------------------------------------------------------
def _sizes():
    S = sms() * 8 * 256                  # threads of the largest grid grid_for launches
    small = list(range(10)) + [15, 16, 17, 255, 256, 257]
    # 2-per-thread loop of the 16-byte path (FP64: 2 per vector, FP32: 4), 4-per-thread dot loop
    edges = [4 * S - 2, 4 * S, 4 * S + 3, 8 * S - 1, 8 * S + 5, 16 * S + 3]
    return small, edges


def _ew_check(got, want, scale, c, u, what):
    bnd = acc.gamma(c, u) * np.asarray(scale, dtype=F64)
    acc.assert_rows(got, want, bnd, what)


def _ew_ops(ctx, n, dt, seed, wrap=None, full=True):
    """full=False: only the plain forms of the operations (the largest sizes)."""
    rng = np.random.default_rng(seed)
    x, y, z = (rng.uniform(-1, 1, n) * np.exp2(rng.uniform(-8, 8, n)) for _ in range(3))
    x, y, z = (v.astype(dt) for v in (x, y, z))
    u = acc.unit(dt)
    mk = wrap or (lambda a: dvec(ctx, a, dt))
    X, Y, Z = (a.astype(LD) for a in (x, y, z))
    a, b, c = -1.25, 0.5, 0.125                        # exact in FP32 (the kernels cast them to T)
    what = "n=%d %s%s" % (n, np.dtype(dt).name, " offset" if wrap else "")
    vx, vy = mk(x), mk(y)
    ctx.axpby(a, vx, b, vy)
    _ew_check(get(vy, dt), a * X + b * Y, np.abs(a * X) + np.abs(b * Y), 2, u, "axpby " + what)
    vz = mk(z)
    vy = mk(y)
    ctx.axpbypcz(a, vx, b, vy, c, vz)
    _ew_check(get(vz, dt), a * X + b * Y + c * Z, np.abs(a * X) + np.abs(b * Y) + np.abs(c * Z), 3, u,
              "axpbypcz " + what)
    vz = mk(z)
    ctx.vmul(a, vx, vy, c, vz)
    _ew_check(get(vz, dt), a * X * Y + c * Z, np.abs(a * X * Y) + np.abs(c * Z), 3, u, "vmul " + what)
    if not full:
        vc = mk(np.full(n, np.nan))
        ctx.copy(vx, vc)
        assert np.array_equal(get(vc, dt), x), "copy " + what
        return
    vz = mk(np.full(n, np.nan))
    ctx.vmul(a, vx, vy, 0.0, vz)                        # beta = 0: the NaNs are never read
    _ew_check(get(vz, dt), a * X * Y, np.abs(a * X * Y), 2, u, "vmul beta=0 " + what)
    vz = mk(np.full(n, np.nan))
    ctx.axpby(a, vx, 0.0, vz)
    _ew_check(get(vz, dt), a * X, np.abs(a * X), 1, u, "axpby b=0 " + what)
    vz = mk(np.full(n, np.nan))
    ctx.axpbypcz(a, vx, b, vy, 0.0, vz)
    _ew_check(get(vz, dt), a * X + b * Y, np.abs(a * X) + np.abs(b * Y), 2, u, "axpbypcz c=0 " + what)
    # aliasing the reference allows
    va = mk(x)
    ctx.axpby(a, va, b, va)
    _ew_check(get(va, dt), (a + b) * X, np.abs(a * X) + np.abs(b * X), 2, u, "axpby x==y " + what)
    va, vy = mk(x), mk(y)
    ctx.axpbypcz(a, va, b, vy, c, va)
    _ew_check(get(va, dt), (a + c) * X + b * Y, np.abs(a * X) + np.abs(b * Y) + np.abs(c * X), 3, u,
              "axpbypcz z==x " + what)
    vc = mk(np.full(n, np.nan))
    ctx.copy(vx, vc)
    assert np.array_equal(get(vc, dt), x), "copy " + what
    with options(ctx, zero_shortcut=0):
        ctx.clear(vc)                                  # (materialised at once, not lazily)
    assert n == 0 or not get(vc, dt).any()
    got = ctx.dot(vx, vy)
    S, Aabs = acc.dot_ref(x, y)
    acc.assert_scalar(got, S, acc.kahan_bound(Aabs, sms() * 8), "dot " + what)


@pytest.mark.parametrize("dt", [F64, F32], ids=["f64", "f32"])
def test_elementwise_and_dot_small_sizes(ctx, dt):
    small, _ = _sizes()
    for n in small:
        _ew_ops(ctx, n, dt, n)


@pytest.mark.parametrize("dt", [F64, F32], ids=["f64", "f32"])
def test_elementwise_and_dot_unroll_edges(ctx, dt):
    _, edges = _sizes()
    for n in edges:
        _ew_ops(ctx, n, dt, n)
    _ew_ops(ctx, (1 << 24) + 3, dt, 24, full=False)


def _wrap_offset(ctx, keep):
    """FP64 vectors wrapped from a torch slice t[1:]: 8- but not 16-byte aligned (vec_ok false)."""
    import torch

    def mk(a):
        a = np.asarray(a, dtype=F64)
        t = torch.zeros(a.size + 1, dtype=torch.float64, device="cuda")
        t[1:] = torch.from_numpy(a)
        torch.cuda.synchronize()
        s = t[1:]
        v = ab.Vector.__new__(ab.Vector)
        v.ctx, v.h, v.n = ctx, ctypes.c_void_p(), a.size
        assert s.data_ptr() % 16 == 8 or a.size == 0
        assert ab.lib().b200_vec_wrap(ctx.h, ctypes.c_void_p(s.data_ptr()), v.n, ctypes.byref(v.h)) == 0
        keep.append(t)
        return v
    return mk


def test_elementwise_scalar_fallback_on_offset_vectors(ctx):
    keep = []
    mk = _wrap_offset(ctx, keep)
    small, edges = _sizes()
    for n in small[1:] + [edges[0], edges[3]]:
        _ew_ops(ctx, n, F64, 1000 + n, wrap=mk)
        keep.clear()


def test_precision_changing_copy(ctx):
    for n in (1, 3, 257, 100003):
        rng = np.random.default_rng(n)
        x = rng.uniform(-1, 1, n) * np.exp2(rng.uniform(-60, 60, n))
        v64, v32 = ctx.vector(x), _f32vec(ctx, np.full(n, np.nan))
        ctx.copy(v64, v32)
        assert np.array_equal(v32.numpy32(), x.astype(F32))
        w64 = ctx.vector(np.full(n, np.nan))
        ctx.copy(v32, w64)
        assert np.array_equal(w64.numpy(), x.astype(F32).astype(F64))


def test_fused_krylov_steps_on_offset_vectors(ctx):
    keep = []
    mk = _wrap_offset(ctx, keep)
    n = 30001
    ptr, col, val, xh = acc.band_csr(n, n, BAND_OFFS, seed=3, keep=1.0)
    A = ctx.csr(n, n, ptr, col, val)
    rng = np.random.default_rng(8)
    r0, s0, x0 = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    K = ab.Krylov(ctx, n)
    try:
        r, s, p, q, x = mk(r0), mk(s0), mk(np.zeros(n)), mk(np.zeros(n)), mk(x0)
        K.cg_direction(r, s, p)
        ph = p.numpy()
        assert np.array_equal(ph, s0)
        rr = K.cg_step(A, p, q, x, r)
        sc = K.scalars()
        qh, al = q.numpy(), sc["alpha"]
        S, Aabs = acc.dot_ref(r0, s0)
        acc.assert_scalar(sc["rho"], S, acc.kahan_bound(Aabs, sms() * 8), "rho on offset vectors")
        X, R, P, Q = (v.astype(LD) for v in (x0, r0, ph, qh))
        _ew_check(x.numpy(), X + LD(al) * P, np.abs(X) + np.abs(LD(al) * P), 2, acc.U64, "cg x update")
        rh = r.numpy()
        _ew_check(rh, R - LD(al) * Q, np.abs(R) + np.abs(LD(al) * Q), 2, acc.U64, "cg r update")
        S, Aabs = acc.dot_ref(rh, rh)
        acc.assert_scalar(rr, S, acc.kahan_bound(Aabs, sms() * 8), "<r,r> on offset vectors")
    finally:
        K.close()


def test_reductions_at_scale(ctx):
    n = (1 << 24) + 3
    rng = np.random.default_rng(1)
    x, y = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    S, Aabs = acc.dot_ref(x, y)
    acc.assert_scalar(ctx.dot(ctx.vector(x), ctx.vector(y)), S, acc.kahan_bound(Aabs, sms() * 8), "2^24+3")
    # ill-conditioned: sum x*y ~ 1e-12 * sum |x*y|
    y2 = y.copy()
    y2[1:n - 1:2] = -x[0:n - 2:2] * y[0:n - 2:2] / x[1:n - 1:2]   # neighbours cancel pairwise
    y2[-1] = 0.0
    y2[0] += 1e-12 * float(np.abs(x * y2).sum()) / x[0]
    S, Aabs = acc.dot_ref(x, y2)
    assert 0.5e-12 < abs(float(S)) / float(Aabs) < 2e-12
    got = ctx.dot(ctx.vector(x), ctx.vector(y2))
    acc.assert_scalar(got, S, acc.kahan_bound(Aabs, sms() * 8), "ill-conditioned")


def test_cg_step_on_the_128_cube_pattern_operator(ctx):
    """Every CTA owns many blocks: the uncompensated in-kernel <q,p> of the finest operator."""
    with options(ctx, **FORMAT_OPTS["pattern"]):
        ptr, col, val, rhs = ab.poisson3d(128)
        n = ptr.size - 1
        A = ctx.csr(n, n, ptr, col, val)
        assert_stored(A, "pattern")
        pl = A.plan()
        rng = np.random.default_rng(2)
        K = ab.Krylov(ctx, n)
        try:
            r, s, p, q, x = (ctx.vector(rng.uniform(-1, 1, n)) for _ in range(5))
            K.cg_direction(r, s, p)
            K.cg_step(A, p, q, x, r)
            qh, ph = q.numpy(), p.numpy()
            S, M = acc.row_sums(ptr, col, val, ph)
            p_ = acc.plan(ptr, pl["lanes"], ctx.get_option("nnz_cap"))
            m, k = acc.roundings(ptr, p_)
            acc.assert_rows(qh, S, acc.bound("spmv", m, k, acc.U64, M), "128^3 q", ptr, p_)
            S, Aabs = acc.dot_ref(qh, ph)
            bnd = acc.csr_scalar_bound(Aabs, pl["blocks"], p_["rows_cap"], pl["lanes"], sms(),
                                       ctx.get_option("ctas_per_sm"))
            assert pl["blocks"] > 4 * sms() * ctx.get_option("ctas_per_sm")
            acc.assert_scalar(K.scalars()["qp"], S, bnd, "128^3 <q,p>")
        finally:
            K.close()


# ---------------------------------------------------------------------------------------------
# coarse solver: Gauss-Jordan inverse + GEMV
# ---------------------------------------------------------------------------------------------
# ||x^ - x||inf / ||x||inf <= C_COARSE * n * u * kappa_inf(A).  Gauss-Jordan elimination with
# partial pivoting is forward stable: its error is bounded by c_n * rho * u * kappa(A), with c_n
# linear in n and rho the growth factor (Higham, "Accuracy and Stability of Numerical Algorithms",
# 14.4 and 9.4).  The matrix families below (diagonally dominant -- also row-permuted --, SPD, and
# the tie matrices, whose pivot column is dominant after the first step) keep rho <= 2, and the
# first-order term with n*u covers c_n * rho here: C_COARSE = 1 is a stated tolerance for these
# families, not a constant proven for every matrix.
C_COARSE = 1.0


def _dense(kind, n, rng):
    if kind == "dominant":
        A = rng.uniform(-1, 1, (n, n))
        A[np.arange(n), np.arange(n)] = np.abs(A).sum(axis=1) + 1.0
    elif kind == "spd":
        B = rng.uniform(-1, 1, (n, n))
        A = B @ B.T + n * np.eye(n)
    elif kind == "permuted":
        A = rng.uniform(-1, 1, (n, n))
        A[np.arange(n), np.arange(n)] = np.abs(A).sum(axis=1) + 1.0
        A = A[::-1].copy()                   # partial pivoting exchanges rows at every step
    else:                                    # exact ties in the first pivot column
        A = rng.uniform(-1, 1, (n, n))
        A[np.arange(n), np.arange(n)] += 4.0 * np.sign(A[np.arange(n), np.arange(n)])
        A[:, 0] = rng.choice([-1.0, 1.0], n) * 8.0
        A[0, 0] = 8.0
    return A


def _csr_of(A, duplicate=False):
    import scipy.sparse as sp
    M = sp.csr_matrix(A)
    ptr, col, val = M.indptr.astype(np.int64), M.indices.astype(np.int64), M.data
    if duplicate:
        # every entry as two halves (the upload sums duplicates)
        ptr = ptr * 2
        col = np.repeat(col, 2)
        val = np.repeat(val / 2, 2)
    return ptr, col, val


def _refined_solve(A, b):
    x = np.linalg.solve(A, b)
    r = b.astype(LD) - (A.astype(LD) @ x.astype(LD))
    return x + np.linalg.solve(A, r.astype(F64))


def _coarse_check(ctx, A, b, dup, what, dt=F64):
    n = A.shape[0]
    ptr, col, val = _csr_of(A, dup)
    if dt == F64:
        S = ctx.coarse(n, ptr, col, val)
    else:
        S = _coarse_f32(ctx, n, ptr, col, val)
    vb, vx = dvec(ctx, b, dt), dvec(ctx, np.zeros(n), dt)
    ctx.coarse_solve(S, vb, vx)
    got = get(vx, dt).astype(F64)
    A_ = A.astype(dt).astype(F64)
    x = _refined_solve(A_, b.astype(dt).astype(F64))
    kappa = np.abs(A_).sum(axis=1).max() * np.abs(np.linalg.inv(A_)).sum(axis=1).max()
    err = np.abs(got - x).max() / np.abs(x).max()
    # FP32 vectors: the inverse is formed and kept in FP64 from the FP32-rounded matrix, and
    # coarse_gemv_kernel accumulates in FP64 and rounds once into the FP32 x -- so the error is the
    # FP64 one plus one FP32 rounding of x, far below an FP32-scaled n * u32 * kappa
    bnd = C_COARSE * n * acc.U64 * kappa + (acc.U32 if dt == F32 else 0.0)
    assert err <= bnd, "%s: error %.3g > bound %.3g (kappa %.3g)" % (what, err, bnd, kappa)
    return S, got


def _coarse_f32(ctx, n, ptr, col, val):
    L = ab.lib()
    S = ab.Coarse.__new__(ab.Coarse)
    S.ctx, S.h, S.n = ctx, ctypes.c_void_p(), n
    ptr, col = np.ascontiguousarray(ptr, dtype=np.int64), np.ascontiguousarray(col, dtype=np.int64)
    val = np.ascontiguousarray(val, dtype=F32)
    rc = L.b200_coarse_create_i64_f32(ctx.h, n, ptr.ctypes.data, col.ctypes.data, val.ctypes.data,
                                      ctypes.byref(S.h))
    if rc:
        raise ab.B200Error(L.b200_last_error().decode())
    return S


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 255, 256, 257, 1000, 3000])
def test_coarse_solver(ctx, n):
    rng = np.random.default_rng(n)
    kinds = ["dominant", "spd", "permuted", "ties"] if n <= 257 else (["dominant", "ties"] if n <= 1000 else ["permuted"])
    for kind in kinds:
        A = _dense(kind, n, rng)
        b = rng.uniform(-1, 1, n)
        S, got = _coarse_check(ctx, A, b, dup=(kind == "spd"), what="%s n=%d" % (kind, n))
        if n <= 1000:
            # the coarse tail's GEMV gives the stand-alone kernel's bits
            with options(ctx, coarse_tail=1, tail_max_nnz=1 << 40):
                c0 = ctx.tail_stats()[1]
                vb, vx = ctx.vector(b), ctx.vector(n)
                ctx.coarse_solve(S, vb, vx)
                tail = vx.numpy()                      # (flushes the deferred command)
                assert ctx.tail_stats()[1] == c0 + 1
                assert np.array_equal(tail, got), "tail GEMV n=%d" % n
    if n <= 1000:
        A = _dense("dominant", n, rng)
        _coarse_check(ctx, A, rng.uniform(-1, 1, n), False, "fp32 n=%d" % n, dt=F32)


def test_coarse_singularity_threshold(ctx):
    def make(A):
        ptr, col, val = _csr_of(np.asarray(A, dtype=F64))
        return ctx.coarse(len(A), ptr, col, val)
    S = make([[1.0, 0.0], [0.0, 1e-13]])                       # pivot ratio 1e-13: accepted
    vx = ctx.vector(2)
    ctx.coarse_solve(S, ctx.vector([1.0, 1.0]), vx)
    assert np.allclose(vx.numpy(), [1.0, 1e13], rtol=1e-14, atol=0)
    with pytest.raises(ab.B200Error):
        make([[1.0, 0.0], [0.0, 1e-15]])                       # 1e-15: rejected
    with pytest.raises(ab.B200Error):                          # an empty row
        ctx.coarse(3, np.array([0, 1, 1, 2]), np.array([0, 2]), np.array([1.0, 1.0]))
    with pytest.raises(ab.B200Error):                          # a NaN entry
        make([[1.0, 0.5, 0.0], [0.0, np.nan, 0.0], [0.0, 0.0, 1.0]])
    with pytest.raises(ab.B200Error):
        make([[2.0, 1.0, 0.0], [1.0, 2.0, np.nan], [0.0, 1.0, 2.0]])
