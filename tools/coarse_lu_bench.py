"""Setup and per-solve time of the coarsest-level solvers on one GPU.

  python tools/coarse_lu_bench.py [--reps 200] [--warmup 20]

Cases: the banded LU on a 2-D Poisson level just above the dense inverse's 16384 rows and on the
reference's smoothed-aggregation level-1 operator of 3-D Poisson 64^3 (about 3e4 rows), and the
dense inverse at n = 16384 (2-D Poisson 128^2) for scale.  Setup is timed on the host around the create call (it
synchronises); a solve is timed with CUDA events over `reps` back-to-back solves after `warmup`
untimed ones.  The bytes a solve streams come from the plan (panel chunks and diagonal-block
inverses, 8 bytes per entry) or, for the dense inverse, n^2 * 8.  Every line names the card and
its power limit.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import amgcl_b200 as ab  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def poisson2d(m):
    T = sp.diags([-1.0, 2.0, -1.0], [-1, 0, 1], shape=(m, m))
    return (sp.kron(sp.eye(m), T) + sp.kron(T, sp.eye(m))).tocsr()


def sa_level1(m):
    import oracle
    ptr, col, val, _ = ab.poisson3d(m)
    R = oracle.RefSolver(ptr, col, val, "damped_jacobi", "cg")
    n, _, (p, c, v) = R.level_matrix(1, "A")
    R.close()
    return sp.csr_matrix((v, c, p), shape=(n, n))


def streamed_bytes(A, kind):
    n = A.shape[0]
    if kind == "dense_inverse":
        return n * n * 8
    p = ab.coarse_lu_plan(n, A.indptr, A.indices)
    nt = len(p["lfirst"])
    t = p["tile_rows"]
    k = np.arange(nt)
    chunks = int((k - p["lfirst"]).sum() + (p["ulast"] - k).sum() + 2 * nt)
    return chunks * t * t * 8


def measure(ctx, name, A, reps, warmup, gpu):
    import torch
    n = A.shape[0]
    ptr, col = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    ctx.sync()
    t0 = time.perf_counter()
    S = ctx.coarse(n, ptr, col, A.data)
    ctx.sync()
    setup = time.perf_counter() - t0
    info = S.info()
    vb, vx = ctx.vector(np.random.default_rng(0).uniform(-1, 1, n)), ctx.vector(n)
    for _ in range(warmup):
        ctx.coarse_solve(S, vb, vx)
    ctx.sync()
    stream = torch.cuda.ExternalStream(ctx_stream(ctx))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        ctx.coarse_solve(S, vb, vx)
    ctx.flush()
    e1.record(stream)
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    nbytes = streamed_bytes(A, info["kind"])
    out = {"case": name, "kind": info["kind"], "n": n, "bandwidth": info["bandwidth"],
           "tiles": info["tiles"], "factor_bytes": S.bytes(), "setup_s": round(setup, 4),
           "solve_ms": round(ms, 4), "streamed_bytes": nbytes,
           "streamed_GBps": round(nbytes / (ms * 1e-3) / 1e9, 1), "gpu": gpu[0], "power_limit": gpu[1]}
    print(json.dumps(out), flush=True)
    return out


def ctx_stream(ctx):
    s = ab._c.c_void_p()
    ab._check(ab.lib().b200_ctx_get_stream(ctx.h, ab._c.byref(s)))
    return s.value or 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    gpu = card()
    ctx = ab.Context(0)
    measure(ctx, "poisson2d_130", poisson2d(130), args.reps, args.warmup, gpu)
    measure(ctx, "sa_level1_poisson3d_64", sa_level1(64), args.reps, args.warmup, gpu)
    # the dense inverse's solve does not depend on A's sparsity: 2-D Poisson 128^2 = 16384 rows
    measure(ctx, "poisson2d_128_dense", poisson2d(128), args.reps, args.warmup, gpu)
    ctx.close()


if __name__ == "__main__":
    main()
