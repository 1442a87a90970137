"""Banded-LU coarse solver, host side (no GPU): the symbolic phase (b200_coarse_lu_plan_i64), a
numpy model of the tiled sweeps in the order coarse_lu_sweep_kernel documents, and the ticket
schedule of the persistent sweep kernels."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import amgcl_b200 as ab
import _accuracy as acc

# ||x^ - x||inf / ||x||inf <= C_LU * n * u * kappa_inf(A), as for the dense coarse solver
# (test_gpu_accuracy.py): LU without pivoting is backward stable with growth factor rho
# (Higham, "Accuracy and Stability of Numerical Algorithms", 9.3), and rho <= 2 for the
# diagonally dominant matrices below (9.5); the diagonal-block inverses are triangular inverses
# of 64 x 64 blocks of such a factor, whose application adds a term of the same order
# (Higham 14.2).  C_LU = 1 is a stated tolerance for these families.
C_LU = 1.0


def poisson2d(m, convection=0.0):
    T = sp.diags([-1.0 - convection, 2.0 + convection, -1.0], [-1, 0, 1], shape=(m, m))
    return (sp.kron(sp.eye(m), T) + sp.kron(sp.diags([-1.0, 2.0, -1.0], [-1, 0, 1], shape=(m, m)),
                                             sp.eye(m))).tocsr()


def shuffled(A, seed):
    """The same matrix with its rows' entries in random order (the symbolic phase must not care)."""
    A = A.tocsr()
    rng = np.random.default_rng(seed)
    col = A.indices.copy()
    val = A.data.copy()
    for i in range(A.shape[0]):
        s = slice(A.indptr[i], A.indptr[i + 1])
        p = rng.permutation(s.stop - s.start)
        col[s], val[s] = col[s][p], val[s][p]
    return A.indptr.astype(np.int64), col.astype(np.int64), val


def matrices():
    rng = np.random.default_rng(7)
    out = {"poisson2d": poisson2d(30), "convection": poisson2d(24, convection=0.7)}
    # a random sparse diagonally dominant matrix with two components and an isolated vertex
    n = 700
    R = sp.random(n, n, density=4.0 / n, random_state=3, format="csr")
    R = R + R.T * 0.5
    R.setdiag(0)
    R.eliminate_zeros()
    R = R.tolil()
    R[:350, 350:] = 0
    R[350:, :350] = 0
    R[100, :] = 0
    R[:, 100] = 0
    R = R.tocsr()
    D = sp.diags(np.asarray(abs(R).sum(axis=1)).ravel() + 1.0 + rng.uniform(0, 1, n))
    out["random"] = (R + D).tocsr()
    return out


def plan_of(A):
    ptr, col, _ = shuffled(A, 0)
    return ab.coarse_lu_plan(A.shape[0], ptr, col)


def tile_extents(lower, upper, t):
    """The tile extents the library documents, for any tile size t: L panel of tile k from the
    tile of the first column its rows reach; U panel of tile k up to the tile of the last column
    whose first row lies in tile k or before."""
    n = lower.size
    nt = (n + t - 1) // t
    r = np.arange(n)
    first_col = r - lower
    lfirst = np.array([first_col[k * t:(k + 1) * t].min() // t for k in range(nt)])
    reach = np.full(nt, -1)
    np.maximum.at(reach, (r - upper) // t, r // t)
    ulast = np.maximum(np.maximum.accumulate(reach), np.arange(nt))
    return lfirst, ulast


@pytest.mark.parametrize("name", ["poisson2d", "convection", "random"])
def test_plan_profile_covers_permuted_matrix(name):
    A = matrices()[name]
    n = A.shape[0]
    p = plan_of(A)
    perm = p["perm"].astype(np.int64)
    assert np.array_equal(np.sort(perm), np.arange(n))
    P = A[perm][:, perm].tocoo()
    r, c = P.row, P.col
    lo, up = p["lower"], p["upper"]
    assert np.all(r - c <= lo[r])                # every entry lies in its row's lower profile
    assert np.all(c - r <= up[c])                # ... and in its column's upper profile
    assert np.all(lo[r[r > c]] >= 0)
    # the profile is tight: each row's lower and each column's upper bandwidth is attained
    lo_t = np.zeros(n, dtype=np.int64)
    up_t = np.zeros(n, dtype=np.int64)
    np.maximum.at(lo_t, r, np.maximum(r - c, 0))
    np.maximum.at(up_t, c, np.maximum(c - r, 0))
    assert np.array_equal(lo, lo_t) and np.array_equal(up, up_t)
    assert p["bandwidth"] == max(lo.max(), up.max())
    lf, ul = tile_extents(lo, up, p["tile_rows"])
    assert np.array_equal(lf, p["lfirst"]) and np.array_equal(ul, p["ulast"])
    # the ordering pays: the bandwidth is far below n for these matrices
    if name == "poisson2d":
        assert p["bandwidth"] <= 2 * 30


def test_plan_reduces_poisson_bandwidth_and_counts_bytes():
    A = poisson2d(130)                                   # just above the dense inverse's 16384 rows
    p = plan_of(A)
    assert p["bandwidth"] <= 140
    t = p["tile_rows"]
    nt = len(p["lfirst"])
    chunks = (np.arange(nt) - p["lfirst"]).sum() + (p["ulast"] - np.arange(nt)).sum() + 2 * nt
    assert p["factor_bytes"] >= chunks * t * t * 8
    band = p["lower"].max() + p["upper"].max() + 1
    assert p["setup_bytes"] >= A.shape[0] * band * 8     # the band the factorisation runs in


def test_plan_rejects_bad_input():
    with pytest.raises(ab.B200Error):
        ab.coarse_lu_plan(3, np.array([0, 1, 2, 3]), np.array([0, 3, 2]))
    with pytest.raises(ab.B200Error):
        ab.coarse_lu_plan(2, np.array([0, 2, 1]), np.array([0, 1]))


def tiled_solve_model(A, b, p):
    """What the device computes: LU without pivoting of the permuted matrix (padded to whole
    tiles with identity rows), then the forward and backward sweeps tile by tile, each tile's
    panel chunks in consumption order (farthest tile first) and its diagonal block applied
    through the explicit inverse."""
    n = A.shape[0]
    t = p["tile_rows"]
    nt = (n + t - 1) // t
    N = nt * t
    perm = p["perm"].astype(np.int64)
    M = np.eye(N)
    M[:n, :n] = A[perm][:, perm].toarray()
    for k in range(N - 1):
        M[k + 1:, k] /= M[k, k]
        M[k + 1:, k + 1:] -= np.outer(M[k + 1:, k], M[k, k + 1:])
    Lf = np.tril(M, -1) + np.eye(N)
    Uf = np.triu(M)
    # the panels hold every non-zero of the factor
    for k in range(nt):
        rows = slice(k * t, (k + 1) * t)
        assert not Lf[rows, :p["lfirst"][k] * t].any()
        assert not Uf[rows, (p["ulast"][k] + 1) * t:].any()
    blk = lambda k: slice(k * t, (k + 1) * t)
    z = np.zeros(N)
    bp = np.zeros(N)
    bp[:n] = b[perm]
    for k in range(nt):
        s = np.zeros(t)
        for d in range(p["lfirst"][k], k):
            s += Lf[blk(k), blk(d)] @ z[blk(d)]
        z[blk(k)] = np.linalg.inv(Lf[blk(k), blk(k)]) @ (bp[blk(k)] - s)
    for k in range(nt - 1, -1, -1):
        s = np.zeros(t)
        for d in range(p["ulast"][k], k, -1):
            s += Uf[blk(k), blk(d)] @ z[blk(d)]
        z[blk(k)] = np.linalg.inv(Uf[blk(k), blk(k)]) @ (z[blk(k)] - s)
    x = np.zeros(n)
    x[perm] = z[:n]
    return x


@pytest.mark.parametrize("name", ["poisson2d", "convection", "random"])
def test_tiled_sweeps_model_matches_spsolve(name):
    A = matrices()[name]
    n = A.shape[0]
    b = np.random.default_rng(1).uniform(-1, 1, n)
    p = plan_of(A)
    got = tiled_solve_model(A, b, p)
    x = spla.spsolve(A.tocsc(), b)
    Ad = A.toarray()
    kappa = np.abs(Ad).sum(axis=1).max() * np.abs(np.linalg.inv(Ad)).sum(axis=1).max()
    err = np.abs(got - x).max() / np.abs(x).max()
    assert err <= C_LU * n * acc.U64 * kappa, (err, kappa)


def schedule_waits(nt, G, lfirst, ulast, epoch):
    """The persistent sweep kernels' schedule: launch `epoch` hands out tickets
    [epoch*(nt+G), (epoch+1)*(nt+G)); ticket -> position loc; forward tile loc, backward tile
    nt-1-loc; loc >= nt makes the CTA exit.  Yields (ticket, ticket waited on) for every wait."""
    per = nt + G
    for backward in (False, True):
        ticket_of = {}
        for tk in range(epoch * per, (epoch + 1) * per):
            loc = tk % per
            if loc < nt:
                ticket_of[nt - 1 - loc if backward else loc] = tk
        for k, tk in ticket_of.items():
            deps = range(k + 1, ulast[k] + 1) if backward else range(lfirst[k], k)
            for d in deps:
                assert tk // per == ticket_of[d] // per == epoch
                yield backward, tk, ticket_of[d]


def run_schedule(nt, G, lfirst, ulast):
    """Simulate G CTAs, each holding one ticket at a time and finishing it only when every tile
    it waits on is done; returns True when every tile of both sweeps finishes."""
    per = nt + G
    for backward in (False, True):
        done = np.zeros(nt, dtype=bool)
        next_ticket = 0
        held = []
        exited = 0
        while exited < G:
            while len(held) + exited < G:              # every running CTA holds a ticket
                held.append(next_ticket)
                next_ticket += 1
            progressed = False
            for tk in list(held):
                loc = tk % per
                if loc >= nt:
                    held.remove(tk)
                    exited += 1
                    progressed = True
                    continue
                k = nt - 1 - loc if backward else loc
                deps = range(k + 1, ulast[k] + 1) if backward else range(lfirst[k], k)
                if all(done[d] for d in deps):
                    done[k] = True
                    held.remove(tk)
                    progressed = True
            if not progressed:
                return False
        if not done.all():
            return False
    return True


def test_schedule_waits_only_on_smaller_tickets():
    rng = np.random.default_rng(11)
    mats = matrices()
    for trial in range(40):
        A = mats[("poisson2d", "convection", "random")[trial % 3]]
        p = plan_of(A)
        t = int(rng.integers(1, 97))
        G = int(rng.integers(1, 300))
        lf, ul = tile_extents(p["lower"], p["upper"], t)
        nt = lf.size
        for epoch in (0, 1, 5):
            for backward, tk, dep in schedule_waits(nt, G, lf, ul, epoch):
                assert dep < tk, (t, G, backward, tk, dep)
        assert run_schedule(nt, G, lf, ul), (t, G)
