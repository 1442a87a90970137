#!/usr/bin/env python
"""bench.py -- solve-phase benchmark of the amgcl_b200 backend on an H100 (BASELINE.json metric).

Workload (config #2 of BASELINE.json): 3-D 7-point Poisson 256^3 (16.8 M unknowns,
117 M non-zeros), FP64, AMGCL smoothed_aggregation + damped_jacobi + CG with all
reference defaults, hierarchy built on the host by AMGCL itself, solve phase on the
GPU through amgcl::backend::b200 (the drop-in).  One "step" = one complete solve
(rhs == 1, x0 == 0, tol 1e-8).  Metric: CG iterations per second (and solve seconds).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--n 256] [--impl b200|reference]
                    [--dump-outputs DIR]

One JSON line on stdout (rank 0).  See DESIGN.md "Measurement" for every field.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "cg_iterations_per_second"
UNIT = "iter/s"


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10, help="timed solves (at least 1)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--n", type=int, default=256, help="grid points per dimension")
    ap.add_argument("--relax", default="damped_jacobi", choices=["damped_jacobi", "spai0"])
    ap.add_argument("--krylov", default="cg", choices=["cg", "bicgstab"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--precision", default="f64", choices=["f64", "mixed"],
                    help="f64 (BASELINE config, default) or mixed = FP32 hierarchy under an FP64 "
                         "Krylov solver (the reference's mixed-precision composition; not the headline)")
    ap.add_argument("--partition", default="all", choices=["finest", "all"],
                    help="N>1: partition only the finest level (north star) or every level "
                         "with at least --partition-min-rows rows")
    ap.add_argument("--partition-min-rows", type=int, default=50000,
                    help="levels with at least this many rows are partitioned, smaller ones replicated "
                         "(256^3: levels 0-2; measured 2-3 %% faster than 10^6 at 4 and 8 GPUs)")
    ap.add_argument("--p2p", type=int, default=1, choices=[0, 1],
                    help="N>1: 1 = peer-memory exchange kernels over NVLink, 0 = NCCL collectives")
    ap.add_argument("--graph", type=int, default=0, choices=[0, 1],
                    help="1: amgcl::preconditioner::b200_cycle_graph<amg<...>> -- every V-cycle is one "
                         "CUDA graph launch (single GPU)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed solves, write what the last one computed (either --impl) as "
                         "DIR/<name>.npy (float64): iters, resid and the solution x (a fixed seeded sample of it when "
                         "it is larger than %d entries, with the sampled indices)" % DUMP_MAX_X)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    return args


def workload_name(args):
    prec = "fp64" if args.precision == "f64" else "mixed_fp64krylov_fp32amg"
    return "poisson3d_%d^3_%s_sa_%s_%s" % (args.n, prec, args.relax, args.krylov)


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        with open(path) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not measured"


# --------------------------------------------------------------------------- clocks
class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    QUERY = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
             "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, device):
        self.device = device
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.device), "--query-gpu=" + self.QUERY,
                 "--format=csv,noheader,nounits", "-lms", "100"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._pump, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, smax, power, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in self.lines:
            parts = [p.strip() for p in line.split(",")]
            if len(parts) < 8:
                continue
            try:
                sm.append(float(parts[0]))
                smax.append(float(parts[1]))
                power.append(float(parts[2]))
            except ValueError:
                continue
            for name, flag in zip(names, parts[4:8]):
                if flag.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(max(smax)),
                "power_w_max": float(max(power)), "samples": len(sm), "reasons": sorted(reasons)}


def pin_openmp():
    """BASELINE.md section 3 protocol for the CPU arm: threads bound to cores, neighbours
    close.  Must run before the first OpenMP runtime is loaded (libgomp reads the
    environment once), i.e. before torch / oracle are imported."""
    cpu_topology()      # BEFORE binding: afterwards this thread's affinity mask is one core
    os.environ.setdefault("OMP_PROC_BIND", "close")
    os.environ.setdefault("OMP_PLACES", "cores")


_TOPOLOGY = None


def cpu_topology():
    """(logical cpus, physical cores, sockets) this process may use; evaluated once, before the
    OpenMP runtime binds the calling thread."""
    global _TOPOLOGY
    if _TOPOLOGY is None:
        _TOPOLOGY = _cpu_topology()
    return _TOPOLOGY


def cgroup_cpu_limit():
    """CPUs' worth of time the container may use (cgroup v2 cpu.max / v1 cfs quota), or None."""
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()[:2]
        if quota != "max":
            return max(1, int(int(quota) / int(period)))
    except Exception:
        pass
    try:
        with open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us") as f:
            quota = int(f.read())
        with open("/sys/fs/cgroup/cpu/cpu.cfs_period_us") as f:
            period = int(f.read())
        if quota > 0:
            return max(1, quota // period)
    except Exception:
        pass
    return None


def setup_threads(world):
    """OpenMP threads for AMGCL's host-side setup inside the drop-in library: the CPUs this
    process may really use, shared between the ranks, at most 32 (the coarsening does not scale
    further; 128 spinning threads on a container with a CPU quota are far slower than 32)."""
    logical, cores, _ = cpu_topology()
    limit = cgroup_cpu_limit()
    avail = min(cores, limit) if limit else cores
    return max(1, min(32, avail // max(world, 1)))


def _cpu_topology():
    logical = os.cpu_count() or 1
    try:
        out = subprocess.run(["lscpu", "-p=CPU,CORE,SOCKET"], stdout=subprocess.PIPE,
                             stderr=subprocess.DEVNULL, text=True, timeout=10).stdout
        rows = [tuple(int(v) for v in line.split(",")[:3]) for line in out.splitlines()
                if line and not line.startswith("#")]
        avail = None
        try:
            avail = os.sched_getaffinity(0)
        except Exception:
            pass
        if avail:
            rows = [r for r in rows if r[0] in avail] or rows
        cores = len({(c, sk) for _, c, sk in rows}) or logical
        sockets = len({sk for _, _, sk in rows}) or 1
        return len(rows) or logical, cores, sockets
    except Exception:
        return logical, logical, 1


def pick_threads(ref, step):
    """Sweep the OpenMP thread count over {all logical cpus, all physical cores, one socket's
    cores, half a socket} and keep the fastest (memory-bound kernels often peak below the
    hardware thread count): one settling step, then the median of three per candidate."""
    logical, cores, sockets = cpu_topology()
    limit = cgroup_cpu_limit()
    cands = sorted({c for c in (logical, cores, cores // sockets, max(1, cores // (2 * sockets)),
                                max(1, cores // (4 * sockets)), limit)
                    if c and c >= 1}, reverse=True)
    if limit:
        # a CPU quota far below the thread count only produces spinning threads (measured: 128
        # bound threads on a 16-CPU quota are 17x slower than 16): do not waste minutes on them
        cands = [c for c in cands if c <= 4 * limit] or [limit]
    best, best_t, seen = cands[0], None, {}
    for c in cands:
        ref.set_threads(c)
        step()                                   # settle
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            step()
            ts.append(time.perf_counter() - t0)
        dt = float(np.median(ts))
        seen[c] = dt
        if best_t is None or dt < best_t:
            best, best_t = c, dt
    ref.set_threads(best)
    return best, {"logical": logical, "physical_cores": cores, "sockets": sockets, "cgroup_cpu_limit": limit,
                  "binding": "OMP_PROC_BIND=%s OMP_PLACES=%s" % (os.environ.get("OMP_PROC_BIND"),
                                                                 os.environ.get("OMP_PLACES")),
                  "sweep_s_per_sample": {str(k): round(v, 4) for k, v in seen.items()}}


def timed_reference_solves(S, rhs, count):
    """`count` solves of the reference; solve() alone is timed (inside the library, vectors
    first-touched in parallel beforehand).  Returns (x, iters, resid, seconds[])."""
    secs = []
    for _ in range(count):
        x, it, res, dt = S.solve_timed(rhs)
        secs.append(dt)
    return x, it, res, secs


def bounded_reference_sample(args, ptr, col, val, rhs, steps, budget_s, sweep):
    """`steps` timed solves of the reference within `budget_s` seconds of CPU time: FULL solves
    when they fit (every box with a many-core host), else solves truncated to as many Krylov
    iterations as fit (each iteration does the same work, so iterations/s is the same metric;
    boxes that expose 2 host cores need 26 s per full 256^3 solve).  `sweep`: seconds of one
    4-iteration solve at the chosen thread count.  Returns (x, iters, resid, seconds[], full?,
    setup_s)."""
    import oracle
    t0 = time.time()
    S = oracle.RefSolver(ptr, col, val, args.relax, args.krylov, precision=args.precision)
    t_setup = time.time() - t0
    x, it_full, res, dt = S.solve_timed(rhs)           # one full solve: settles, gives the count
    per_iter = dt / max(it_full, 1)
    fit = int(budget_s / max(steps, 1) / max(per_iter, 1e-9))
    if fit >= it_full:
        x, it, res, secs = timed_reference_solves(S, rhs, steps)
        S.close()
        return x, it, res, secs, True, t_setup, x, it_full, res
    S.close()
    k = max(2, min(it_full, fit))
    Sk = oracle.RefSolver(ptr, col, val, args.relax, args.krylov, maxiter=k, precision=args.precision)
    xk, it, resk, secs = timed_reference_solves(Sk, rhs, steps)
    Sk.close()
    return xk, it, resk, secs, False, t_setup, x, it_full, res


# --------------------------------------------------------------------------- reference arm
def reference_arm(args, rank, world):
    """The reference's own CPU implementation of the path: AMGCL builtin (OpenMP) backend
    compiled from the reference sources (oracle/_ref), same workload.  Protocol (BASELINE.md
    section 3): threads bound (OMP_PROC_BIND=close, OMP_PLACES=cores), thread count swept over
    {logical, physical, per-socket}, every timed step ONE FULL solve, solve() alone timed,
    value = iterations / median solve time.  Warm-up steps are truncated (4-iteration)
    solves: they touch exactly the same memory."""
    if rank != 0:
        return
    import oracle
    from amgcl_b200 import poisson3d
    if not oracle.have_ref():
        emit({"impl": "reference", "unavailable":
              "oracle/_ref/libamgcl_ref.so missing and /root/reference not present"})
        return
    ref = oracle.ref()
    t0 = time.time()
    ptr, col, val, rhs = poisson3d(args.n)
    t_gen = time.time() - t0
    Sq = oracle.RefSolver(ptr, col, val, args.relax, args.krylov, maxiter=4, precision=args.precision)
    cores, topo = pick_threads(ref, lambda: Sq.solve(rhs))
    for _ in range(args.warmup):
        Sq.solve(rhs)
    Sq.close()
    x_last, it, res_last, secs, full, t_setup, x, it_full, res = bounded_reference_sample(
        args, ptr, col, val, rhs, args.steps, 150.0, topo)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, x_last, it, res_last, rank)
    med = float(np.median(secs))
    value = it / med
    sample = "%d %s %s solves (%d iterations each%s), solve() only; median %.3f s, min %.3f, max %.3f" % (
        args.steps, "full" if full else "truncated", workload_name(args), it,
        "" if full else " of %d: a full solve does not fit the time budget on %d host threads" % (it_full, cores),
        med, min(secs), max(secs))
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * med,
        "mean_ms_per_step": 1e3 * float(np.mean(secs)),
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f64" if args.precision == "f64" else "f64 krylov + f32 hierarchy",
        "data": "synthetic",
        "config": config_block(args, int(ptr.size - 1), int(ptr[-1]), t_setup, t_gen,
                               backend="amgcl::backend::builtin<double> (OpenMP)"),
        "iters": it_full, "resid": res,
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": cores, "kind": "reference",
                         "sample": sample, "topology": topo},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    emit(line)


def config_block(args, nrows, nnz, t_setup, t_gen, backend=None, parallelism="host cores (OpenMP)",
                 extra=None):
    """`config` of the JSON line: the same keys for both arms (the driver compares them)."""
    cfg = {"workload": workload_name(args), "rows": nrows, "nnz": nnz,
           "relax": args.relax, "krylov": args.krylov, "tol": 1e-8,
           "step": "one complete solve, rhs=1, x0=0",
           "l2": "inputs_exceed_l2 (finest matrix %.2f GB >> 50 MB)" % (nnz * 12 / 1e9),
           "parallelism": parallelism,
           "setup_s": t_setup, "generate_s": t_gen,
           "hierarchy": "host (AMGCL smoothed_aggregation)"}
    if backend:
        cfg["backend"] = backend
    if extra:
        cfg.update(extra)
    return cfg


# --------------------------------------------------------------------------- our arm
def cpu_baseline_leg(args, ptr, col, val, rhs, full_iters):
    """Reference builtin backend on the box's host cores: same protocol as --impl reference
    (bound threads, swept thread count, solve() only), median of three full solves."""
    import oracle
    if not oracle.have_ref():
        return None
    ref = oracle.ref()
    Sq = oracle.RefSolver(ptr, col, val, args.relax, args.krylov, maxiter=4, precision=args.precision)
    threads, topo = pick_threads(ref, lambda: Sq.solve(rhs))
    Sq.close()
    _, it, _, secs, full, t_setup, x, it_full, res = bounded_reference_sample(
        args, ptr, col, val, rhs, 3, 45.0, topo)
    med = float(np.median(secs))
    return {"value": it / med, "unit": UNIT, "cores": threads, "kind": "reference",
            "sample": "3 %s %s solves (%d iterations each), solve() only: median %.3f s (min %.3f, max %.3f); "
                      "setup %.1f s not timed" % ("full" if full else "truncated", workload_name(args), it, med,
                                                  min(secs), max(secs), t_setup),
            "topology": topo, "iters": it_full, "resid": res, "solve_s": med}, x


def golden_parity(args, iters, resid, x):
    """This run against the reference's committed known answers for the workload
    (tests/golden/large_answers.json, written by tests/golden/make_large_answers.py from the
    real reference): iteration count, final residual, and the solution at 257 sample points.
    Works at every N -- the multi-GPU lines carry it too."""
    path = os.path.join(ROOT, "tests", "golden", "large_answers.json")
    if args.precision != "f64" or not os.path.isfile(path):
        return None
    with open(path) as f:
        known = json.load(f)
    case = [c for c in known["cases"] if (c["n"], c["relax"], c["krylov"]) == (args.n, args.relax, args.krylov)]
    if not case:
        return None
    c = case[0]
    idx = np.linspace(0, x.size - 1, len(c["x_samples"])).astype(np.int64)
    want = np.asarray(c["x_samples"])
    out = {"golden": "tests/golden/large_answers.json",
           "iters": iters, "iters_golden": c["iters"],
           "resid": resid, "resid_golden": c["resid"],
           "resid_rel_diff": abs(resid - c["resid"]) / c["resid"],
           "x_samples_rel_err_inf": float(np.abs(x[idx] - want).max() / c["x_max"]),
           "x_norm2_rel_diff": abs(float(np.linalg.norm(x)) - c["x_norm2"]) / c["x_norm2"]}
    out["ok"] = bool(out["iters"] == out["iters_golden"] and out["resid_rel_diff"] <= 1e-6 and
                     out["x_samples_rel_err_inf"] <= 1e-8 and out["x_norm2_rel_diff"] <= 1e-8)
    return out


DUMP_MAX_X = 4 * 1024 * 1024     # entries of x written in full; larger solutions are sampled


def dump_outputs(out_dir, x, iters, resid, rank):
    """What a caller of the timed path receives from its last solve: the iteration count, the
    final relative residual and the solution.  A solution longer than DUMP_MAX_X is written as
    the entries at DUMP_MAX_X / 2 indices drawn with a fixed seed (x_index), so two builds run
    with the same arguments can be compared output for output; at most 64 MB in all."""
    if rank != 0:
        return
    os.makedirs(out_dir, exist_ok=True)
    out = {"iters": np.array([iters], dtype=np.float64), "resid": np.array([resid], dtype=np.float64)}
    if x.size <= DUMP_MAX_X:
        out["x"] = x.astype(np.float64)
    else:
        idx = np.sort(np.random.default_rng(0).choice(x.size, DUMP_MAX_X // 2, replace=False))
        out["x_index"] = idx.astype(np.float64)
        out["x"] = x[idx].astype(np.float64)
    for name, a in out.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def main_arm(args, rank, world, local_rank):
    import torch
    import amgcl_b200 as ab

    dist = None
    if world > 1:
        import torch.distributed as dist_mod
        dist = dist_mod
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    device = local_rank
    torch.cuda.set_device(device)
    side = torch.cuda.Stream(device=device)
    torch.cuda.set_stream(side)
    ctx = ab.Context(device, stream=side.cuda_stream)
    # host-side setup threads: share the box between the ranks (torchrun exports 1)
    ab.set_setup_threads(setup_threads(world))

    t0 = time.time()
    ptr, col, val, rhs = ab.poisson3d(args.n)
    t_gen = time.time() - t0
    nrows, nnz = int(ptr.size - 1), int(ptr[-1])

    dist_min_rows = nrows
    if world > 1:
        # one system, row-partitioned across the GPUs (SURVEY 8e): NCCL id from rank 0
        box = [ab.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        if args.partition == "all":
            dist_min_rows = args.partition_min_rows
        ctx.set_option("p2p", args.p2p)
        ctx.dist_init(box[0], world, rank, dist_min_rows)
    transport = "n/a"
    if world > 1:
        transport = "peer-memory push/wait/reduce kernels (CUDA IPC over NVLink)" \
            if ctx.dist_info()["p2p"] else "NCCL collectives"

    t0 = time.time()
    S = ab.DropinSolver(ptr, col, val, args.relax, args.krylov, ctx=ctx, precision=args.precision,
                        graph=bool(args.graph) and world == 1)
    t_setup = time.time() - t0

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- value: rhs resident in HBM, x0 = 0, K complete solves ------------------------
    S.upload_rhs(rhs)
    for _ in range(max(args.warmup, 3)):
        S.solve_resident()
    sampler = ClockSampler(device)
    barrier()
    sampler.start()
    ctx.reset_launches()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(side)
    iters_total = 0
    for _ in range(args.steps):
        it, res = S.solve_resident()
        iters_total += it
    e1.record(side)
    barrier()
    launches = ctx.launches
    clocks = sampler.stop()
    ms = e0.elapsed_time(e1)
    if dist is not None:
        t = torch.tensor([ms], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    solve_s = ms * 1e-3 / args.steps
    iters = iters_total // args.steps
    # N > 1: ONE system, row-partitioned across the GPUs -> strong scaling
    value = iters_total / (ms * 1e-3)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, S.download_x(), it, res, rank)

    # ---- roofline: same K steps again with the CSR launches bracketed by events ----------
    ctx.profile_begin()
    for _ in range(args.steps):
        S.solve_resident()
    prof = ctx.profile_end()
    # the finest-level operator (this rank's share of it when partitioned) = most non-zeros
    csr_prof = [p for p in prof if p["mode"] in ("spmv", "spmv_acc", "residual", "relax", "residual_scaled")]
    big = max([p["nnz"] for p in csr_prof if p["nrows"] * 2 > p["ncols"]] or [0])
    finest = [p for p in csr_prof if p["nnz"] == big and p["mode"] != "spmv_acc"]
    peak, peak_src = peaks()
    roof = None
    if finest and args.precision == "f64":
        def alg_bytes(p):
            b = p["nnz"] * 12 + (p["nrows"] + 1) * 4 + p["ncols"] * 8 + p["nrows"] * 8
            if p["mode"] in ("residual", "spmv_acc"):
                b += p["nrows"] * 8
            elif p["mode"] in ("relax", "residual_scaled"):      # rhs + diagonal / rhs + x written
                b += 2 * p["nrows"] * 8
            return b
        # what the kernel really streams: the finest operator is stored pattern-indexed (no
        # per-entry columns: 8 B per entry + row pointer + 1 B pattern id per row) or
        # offset-indexed (1 B of column per entry) when it qualifies -- fewer bytes than the CSR
        # figure SURVEY.md section 8(d) counts, same arithmetic
        fmt = ctx.largest_operator()[1]
        col_b, row_b = {"pattern": (0, 5), "offset": (1, 4)}.get(fmt, (4, 4))

        def streamed_bytes(p):
            return alg_bytes(p) - p["nnz"] * (4 - col_b) + (p["nrows"] + 1) * (row_b - 4)
        tot_b = sum(alg_bytes(p) * p["launches"] for p in finest)
        tot_s = sum(streamed_bytes(p) * p["launches"] for p in finest)
        tot_ms = sum(p["total_ms"] for p in finest)
        tot_l = sum(p["launches"] for p in finest)
        ach = tot_b / (tot_ms * 1e-3) / 1e9
        ach_s = tot_s / (tot_ms * 1e-3) / 1e9
        roof = {"bound": "hbm", "kernel": "csr_ring_kernel (finest level A: spmv/residual/relax)",
                "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                # achieved counts the CSR bytes of SURVEY.md 8(d) (12 B per entry); with a compressed
                # column format the kernel moves fewer, so frac can exceed what the memory system
                # delivered: `streamed` is the same launches on the bytes actually moved
                "column_format": fmt,
                "streamed": {"achieved": ach_s, "frac": ach_s / peak, "bytes_per_launch": tot_s / tot_l},
                "peak_source": peak_src, "traffic": None,
                "bytes_per_launch": tot_b / tot_l, "launches": tot_l,
                "avg_launch_ms": tot_ms / tot_l,
                "share_of_step": tot_ms / (args.steps * solve_s * 1e3),
                "by_mode": {p["mode"]: {"launches": p["launches"],
                                        "GBs": alg_bytes(p) * p["launches"] / (p["total_ms"] * 1e-3) / 1e9}
                            for p in finest}}
    all_csr_ms = sum(p["total_ms"] for p in prof if p["nnz"] > 0 and p["mode"] != "coarse_gemv")
    streams = {"vec1": 2, "vec2": 3, "vec3": 4, "vec4": 5, "vec5": 6, "vec6": 7, "vec7": 8,
               "dot": 2, "relax_zero": 3, "memset": 1, "comm": 1, "coarse_tail": 1}
    breakdown = []
    for p in sorted(prof, key=lambda q: -q["total_ms"]):
        if p["mode"] in streams:
            b = streams[p["mode"]] * p["nrows"] * 8
        elif p["mode"] == "coarse_gemv":
            b = p["nnz"] * 8
        else:
            b = p["nnz"] * 12 + (p["nrows"] + 1) * 4 + p["ncols"] * 8 + p["nrows"] * 8
            if p["mode"] in ("residual", "spmv_acc"):
                b += p["nrows"] * 8
            elif p["mode"] in ("relax", "residual_scaled"):
                b += 2 * p["nrows"] * 8
        breakdown.append({"rows": p["nrows"], "cols": p["ncols"], "nnz": p["nnz"], "kernel": p["mode"],
                          "launches_per_step": p["launches"] / args.steps,
                          "ms_per_step": round(p["total_ms"] / args.steps, 4),
                          "GBs": round(b * p["launches"] / (p["total_ms"] * 1e-3) / 1e9, 1)})
    kernels_ms_per_step = sum(p["total_ms"] for p in prof) / args.steps

    # ---- e2e: the user-facing call with pinned HOST buffers, copies inside the timed region --
    rhs_pin = torch.empty(nrows, dtype=torch.float64, pin_memory=True)
    x_pin = torch.empty(nrows, dtype=torch.float64, pin_memory=True)
    rhs_h, x_h = rhs_pin.numpy(), x_pin.numpy()
    rhs_h[:] = rhs
    e2e_iters = 0
    for _ in range(2):
        S.solve_zero_guess_into(rhs_h, x_h)
    barrier()
    t_e2e = 0.0
    for _ in range(args.steps):
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record(side)
        it, res_e2e = S.solve_zero_guess_into(rhs_h, x_h)
        a1.record(side)
        torch.cuda.synchronize()
        t_e2e += a0.elapsed_time(a1) * 1e-3
        e2e_iters += it
    if dist is not None:
        t = torch.tensor([t_e2e], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        t_e2e = float(t.item())
    # every rank uploads its rows of rhs and downloads its rows of x (one system: nrows*8 each way)
    e2e = {"value": e2e_iters / t_e2e, "unit": UNIT, "solve_s": t_e2e / args.steps,
           "h2d_bytes_per_step": nrows * 8, "d2h_bytes_per_step": nrows * 8,
           "api": "make_solver<amg<backend::b200<double>,...>, %s>::operator()(rhs, x) via "
                  "dropin_solve_zero_guess: pinned host rhs -> device, x0 = 0 created on the device as in "
                  "tutorial/1.poisson3Db/poisson3Db_cuda.cu:83-87, solution -> pinned host%s" % (
                      args.krylov, "" if world == 1 else
                      " (each rank moves the rows it owns, like amgcl::mpi's row-distributed vectors)")}
    # the complete solution for the parity check (not timed; N > 1: all-gathered to every rank)
    x_gpu = x_h.copy() if world == 1 else S.download_x()

    # ---- cpu baseline (rank 0, N == 1) ---------------------------------------------------
    cpu = None
    parity = None
    if rank == 0:
        parity = golden_parity(args, iters, res, x_gpu)
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        got = cpu_baseline_leg(args, ptr, col, val, rhs, iters)
        if got is not None:
            cpu, x_ref = got
            parity = dict(parity or {})
            parity.update({"iters_gpu": iters, "iters_ref": cpu.pop("iters"),
                           "resid_gpu": res, "resid_ref": cpu.pop("resid"),
                           "x_rel_err_inf": float(np.abs(x_gpu - x_ref).max() / np.abs(x_ref).max())})
            cpu.pop("solve_s", None)

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": max(args.warmup, 3), "ms_per_step": solve_s * 1e3, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None,       # ONE fixed-size system at every N
            "dtype": "f64" if args.precision == "f64" else "f64 krylov + f32 hierarchy",
            "data": "synthetic",
            "config": config_block(
                args, nrows, nnz, t_setup, t_gen, backend="amgcl::backend::b200<double>",
                parallelism="single GPU" if world == 1 else
                "one system row-partitioned over %d GPUs (levels with >= %d rows; exchange: %s)" % (
                    world, dist_min_rows, transport),
                ),
            "options": {"cycle_graph": {"on": bool(args.graph) and world == 1,
                                        "graphs_kernels_replays": list(S.graph_stats())},
                        "fused_krylov": bool(ctx.get_option("fused_krylov")),
                        "fuse_first_sweep": bool(ctx.get_option("fuse_first_sweep")),
                        "coarse_tail": bool(ctx.get_option("coarse_tail")),
                        "column_formats": {k: bool(ctx.get_option(k)) for k in ("patterns", "offsets", "window")},
                        "partition_min_rows": dist_min_rows if world > 1 else None},
            "solve_s": solve_s, "iters": iters, "resid": res,
            "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks,
            "roofline": roof, "csr_kernel_share_of_step": all_csr_ms / (args.steps * solve_s * 1e3),
            "kernels_ms_per_step": kernels_ms_per_step, "breakdown": breakdown,
            "cpu_baseline": cpu, "parity": parity,
        }
        emit(line)
    S.close()
    if dist is not None:
        dist.destroy_process_group()


_REAL_STDOUT = None


def emit(line):
    """The one JSON line goes to the real stdout; everything else (NCCL banners, library
    chatter) was redirected to stderr in main()."""
    data = (json.dumps(line) + "\n").encode()
    if _REAL_STDOUT is None:
        sys.stdout.write(data.decode())
        sys.stdout.flush()
    else:
        os.write(_REAL_STDOUT, data)


def main():
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)            # fd 1 -> stderr for native libraries (NCCL prints its version there)
    args = parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world == 1 or args.impl == "reference":
        pin_openmp()             # CPU legs: bound threads (before any OpenMP runtime loads)
    if args.impl == "reference":
        reference_arm(args, rank, world)
    else:
        main_arm(args, rank, world, local_rank)


if __name__ == "__main__":
    main()
