#!/usr/bin/env python
"""A/B of the value width the streaming passes read (option "narrow_values": FP32 copy of an FP64
operator whose values are all exact FP32, else an 8- / 16-bit index into the table of its distinct
values), of values kept in the pattern table (option "pattern_values": no per-entry stream at all)
and of the ring shape beside them, on the real solve (one GPU, SA + damped Jacobi + CG on
Poisson n^3).  For each option set: the solution hash against the first set, the solve time, and
per big operator and pass the value bytes (1, 2, 4 or 8), the bytes one pass streams and its
device time (JSON lines on stdout, the card's name and power limit first).

    python tools/values_ab.py [n] [solves] [configs]     # configs: comma-separated indices of CONFIGS
"""
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import amgcl_b200 as ab  # noqa: E402

CONFIGS = [
    ("fp64 values", {"narrow_values": 0}),
    ("fp32 values", {"narrow_values": 1}),
    ("fp32 values, nnz_cap 4096", {"narrow_values": 1, "nnz_cap": 4096}),
    ("fp32 values, 3 stages", {"narrow_values": 1, "stages": 3}),
    ("fp64 values, nnz_cap 4096", {"narrow_values": 0, "nnz_cap": 4096}),
    ("pattern values", {"pattern_values": 1}),
    ("streamed values", {"pattern_values": 0}),
]
DEFAULTS = {"narrow_values": 1, "pattern_values": 1, "nnz_cap": 2048, "stages": 2}

# bytes of column information per entry and of row information per row each stored format streams
COL_BYTES = {"plain": 4, "window": 2, "offset": 1, "pattern": 0, "col16": 2, "col24": 3, "pattern_values": 0}
ROW_BYTES = {"pattern": 3,      # 16-bit block-relative row pointer (+ 1 B pattern id)
             "pattern_values": 1}
VALUES_STREAMED = {"pattern_values": False}   # (values from the pattern table in shared memory)


def streamed_bytes(p):
    """Bytes one pass moves: the stored matrix stream plus the vectors, counted as bench.py counts
    them (x once, y written, rhs / diagonal / old iterate read once per row)."""
    vb = p["value_bytes"] if VALUES_STREAMED.get(p["format"], True) else 0
    b = p["nnz"] * (vb + COL_BYTES[p["format"]]) + p["nrows"] * ROW_BYTES.get(p["format"], 2)
    b += p["ncols"] * 8 + p["nrows"] * 8
    if p["mode"] in ("residual", "spmv_acc"):
        b += p["nrows"] * 8
    elif p["mode"] in ("relax", "residual_scaled"):
        b += 2 * p["nrows"] * 8
    return b


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:     # (the timings below still carry the device events' numbers)
        return "unknown (%s)" % e


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    solves = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    which = [int(v) for v in sys.argv[3].split(",")] if len(sys.argv) > 3 else range(len(CONFIGS))
    import torch
    print(json.dumps({"card": card()}), flush=True)
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    ctx = ab.Context(0, stream=side.cuda_stream)

    def time_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(side)
        fn()
        e1.record(side)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    ptr, col, val, rhs = ab.poisson3d(n)
    ref_hash = None
    for k in which:
        name, opts = CONFIGS[k]
        for key, v in {**DEFAULTS, **opts}.items():
            ctx.set_option(key, v)
        t0 = time.time()
        S = ab.DropinSolver(ptr, col, val, "damped_jacobi", "cg", ctx=ctx)
        setup = time.time() - t0
        x, it, res = S.solve(rhs)
        h = hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest()[:16]
        if ref_hash is None:
            ref_hash = h
        S.upload_rhs(rhs)
        for _ in range(2):
            S.solve_resident()
        ts = [time_ms(lambda: S.solve_resident()) for _ in range(solves)]
        ctx.profile_begin()
        S.solve_resident()
        prof = ctx.profile_end()
        big = sorted([p for p in prof if p["nnz"] >= 5000000 and p["value_bytes"]], key=lambda p: -p["total_ms"])
        ops = []
        for p in big:
            us = 1e3 * p["total_ms"] / p["launches"]
            b = streamed_bytes(p)
            ops.append({"rows": p["nrows"], "nnz": p["nnz"], "mode": p["mode"], "format": p["format"],
                        "value_bytes": p["value_bytes"], "launches": p["launches"], "avg_us": round(us, 1),
                        "streamed_MB": round(b / 1e6, 1), "GBs": round(b / (us * 1e-6) / 1e9)})
        rec = {"config": name, "opts": opts, "setup_s": round(setup, 2), "iters": it, "resid": res,
               "x_sha": h, "same_bits_as_first": h == ref_hash, "solve_ms_median": round(float(np.median(ts)), 3),
               "solve_ms_min": round(float(np.min(ts)), 3), "ops": ops}
        print(json.dumps(rec), flush=True)
        S.close()


if __name__ == "__main__":
    main()
