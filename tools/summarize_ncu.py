#!/usr/bin/env python
"""Turn the artefacts of tools/ncu_capture.py into summaries under profiles/ (a local output
directory: git ignores it, so captures stay out of history and are quoted with the GPU they ran on).

    python tools/summarize_ncu.py <round-tag> <launches.csv> <full.ncu-rep>

Writes profiles/<tag>_launches.csv (copy), profiles/<tag>_launch_shares.md,
profiles/<tag>_csr_kernels.md (per-kernel metrics of the --set full capture) and
profiles/traffic.json (DRAM bytes per launch of the dominant kernel)."""
import collections
import re
import csv
import io
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROF = os.path.join(ROOT, "profiles")


def short_name(full):
    """'void b200::csr_ring_kernel<3, 1, 0, Prec<double, ...>>(args)' -> 'csr_ring_kernel<3, 1> f64'."""
    name = full.split("(")[0].replace("void ", "").replace("b200::", "")
    name = name.replace("(int)", "").replace("(bool)", "")
    m = re.match(r"(csr_\w+_kernel)<(\d+), (\d+), (\d+), Prec<([^>]*)>(?:, (\d+))?>", name)
    if m:
        types = [t.strip() for t in m.group(5).split(",")]
        prec = "f64" if all(t == "double" for t in types) else \
               "f32" if all(t == "float" for t in types) else "mixed"
        fmt = {"1": " window", "2": " offset", "3": " pattern"}.get(m.group(6) or "0", "")
        return "%s<%s, %s>%s %s%s" % (m.group(1), m.group(2), m.group(3),
                                      " halo" if m.group(4) == "1" else "", prec, fmt)
    return name


def launch_shares(tag, path):
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr = rows[hi]
    data = [r for r in rows[hi + 1:] if len(r) == len(hdr)]
    kn, mv = hdr.index("Kernel Name"), hdr.index("Metric Value")
    agg = collections.OrderedDict()
    tot = 0.0
    for r in data:
        key = short_name(r[kn])
        t = float(r[mv].replace(",", ""))
        a = agg.setdefault(key, [0, 0.0])
        a[0] += 1
        a[1] += t
        tot += t
    out = ["# %s: ncu launch list (gpu__time_duration.sum, --clock-control none)" % tag, "",
           "Command: `ncu --metrics gpu__time_duration.sum --clock-control none -c 4000 --csv "
           "python tools/profile_target.py <n> 1 ...` (pass 1 of tools/ncu_capture.py: every launch "
           "of the process, coarse-solver set-up included; %d launches, %.2f ms of kernel time).  "
           "Per-launch times under ncu are cold-cache and serialised: compare SHARES." % (len(data), tot / 1e6), "",
           "Template arguments of csr_ring_kernel<MODE, L>: MODE 0 spmv(beta=0), 1 spmv(beta!=0), "
           "2 residual, 3 fused relax, 4 residual fused with the smoother's first sweep; L = lanes "
           "per row (L=1 is the finest level A and P).", "",
           "| kernel | launches | total us | share | avg us |", "|---|---:|---:|---:|---:|"]
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        out.append("| `%s` | %d | %.1f | %.1f%% | %.2f |" % (k, n, t / 1e3, 100 * t / tot, t / n / 1e3))
    finest = sum(t for k, (n, t) in agg.items() if re.match(r"csr_ring_kernel<[0234], 1>", k))
    out += ["", "Finest-level A passes (`csr_ring_kernel<0|2|3|4, 1>`): %.1f%% of the captured kernel time."
            % (100 * finest / tot)]
    open(os.path.join(PROF, tag + "_launch_shares.md"), "w").write("\n".join(out) + "\n")
    shutil.copy(path, os.path.join(PROF, tag + "_launches.csv"))


WANT = [("gpu__time_duration.sum", "time"), ("launch__grid_size", "grid"),
        ("launch__registers_per_thread", "regs"),
        ("dram__bytes_read.sum", "dram read"), ("dram__bytes_write.sum", "dram write"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %"),
        ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %"),
        ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1TEX %"),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM %"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
        ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
        ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smem wavefronts"),
        ("lts__t_sector_hit_rate.pct", "L2 hit %"), ("l1tex__t_sector_hit_rate.pct", "L1 hit %")]


def full_capture(tag, rep):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE,
                         stderr=subprocess.DEVNULL, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    kn = hdr.index("Kernel Name")
    out = ["# %s: ncu --set full capture of the CSR streaming kernels" % tag, "",
           "Command: `ncu --set full --clock-control none --import-source on -k regex:csr_ring_kernel "
           "-c 8 python tools/profile_target.py 256 1` (first 8 launches of the first solve: "
           "residual on A0 twice, then R0, A1, R1, A2, ...).", "",
           "| kernel | " + " | ".join(n for _, n in WANT) + " |",
           "|---|" + "---:|" * len(WANT)]
    traffic = None
    for r in data:
        cells = []
        for key, _ in WANT:
            if key in hdr:
                i = hdr.index(key)
                v = r[i]
                try:
                    v = "%.4g" % float(v.replace(",", ""))
                except ValueError:
                    pass
                cells.append("%s %s" % (v, units[i]) if units[i] not in ("", "%") else v)
            else:
                cells.append("n/a")
        name = short_name(r[kn])
        out.append("| `%s` | " % name + " | ".join(cells) + " |")
        if traffic is None and name.startswith("csr_ring_kernel<2, 1>"):
            def val(key):
                i = hdr.index(key)
                scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}[units[i]]
                return float(r[i].replace(",", "")) * scale
            rd, wr = val("dram__bytes_read.sum"), val("dram__bytes_write.sum")
            traffic = {"kernel": "csr_ring_kernel<2, 1> (residual r = f - A x on the finest level, 256^3)",
                       "nnz": 117047296, "dram_bytes_read": rd, "dram_bytes_write": wr,
                       "dram_bytes_per_launch": rd + wr,
                       "algorithmic_bytes_per_launch": 117047296 * 12 + 16777217 * 4 + 3 * 16777216 * 8,
                       "source": "profiles/%s_csr_kernels.md (ncu --set full, one launch)" % tag}
    open(os.path.join(PROF, tag + "_csr_kernels.md"), "w").write("\n".join(out) + "\n")
    if traffic:
        json.dump(traffic, open(os.path.join(PROF, "traffic.json"), "w"), indent=1)


def short_any(full):
    """Readable name for every kernel of the step (CSR ring kernels and the fused vector passes)."""
    name = full.split("(")[0].replace("void ", "").replace("b200::", "")
    m = re.match(r"fused_vec_kernel<(\w+), (\d+)>", name)
    if m:
        return "fused_vec_kernel<%s>" % m.group(1)
    m = re.match(r"(\w+_kernel)<(.*)>$", name)
    if m and m.group(1).startswith("csr_"):
        return short_name(full)
    return name.split("<")[0] if name.startswith(("relax_zero", "coarse_gemv", "dot_kernel", "ew_kernel")) else name


def iteration_table(tag, raw_csv, what, peak=6586.7):
    """profiles/<tag>_kernels.md: one row per launch of ONE Krylov iteration captured with
    ncu --set full (tools/ncu_capture.py): duration, DRAM bytes, achieved DRAM GB/s against the
    measured HBM peak, and the cache / pipe utilisation that explains the gap."""
    rows = list(csv.reader(open(raw_csv)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    kn = hdr.index("Kernel Name")

    def num(r, key):
        if key not in hdr:
            return None
        i = hdr.index(key)
        try:
            v = float(r[i].replace(",", ""))
        except ValueError:
            return None
        scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "us": 1e-6, "ms": 1e-3, "ns": 1e-9,
                 "second": 1.0, "msecond": 1e-3, "usecond": 1e-6, "nsecond": 1e-9}.get(units[i], 1.0)
        return v * scale

    out = ["# %s: every kernel of one %s (ncu --set full --clock-control none)" % (tag, what), "",
           "Captured by `python tools/ncu_capture.py` (pass 2: the launches of the second iteration of "
           "the first solve).  Durations under ncu are serialised and cold-cache; `DRAM GB/s` = "
           "(dram__bytes_read.sum + dram__bytes_write.sum) / gpu__time_duration, `of peak` against the "
           "measured %.1f GB/s (MEASURED_PEAKS.json).  Kernels on operators that fit the 50 MB L2 read "
           "less from DRAM than they stream: their bound is the launch / dependency latency, see "
           "DESIGN.md." % peak, "",
           "`stall`: warps stalled per issued instruction at a CTA barrier / on a long-scoreboard (global "
           "memory) dependency; `issue %`: cycles a scheduler issued.", "",
           "| # | kernel | grid | regs | time us | DRAM read MB | DRAM write MB | DRAM GB/s | of peak | "
           "dram % | L2 % | L1TEX % | SM % | L1 hit % | L2 hit % | stall barrier | stall long sb | issue % |",
           "|---:|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for i, r in enumerate(data):
        t = num(r, "gpu__time_duration.sum")
        rd, wr = num(r, "dram__bytes_read.sum") or 0.0, num(r, "dram__bytes_write.sum") or 0.0
        gbs = (rd + wr) / t / 1e9 if t else 0.0

        def pct(key):
            v = num(r, key)
            return "%.1f" % v if v is not None else "n/a"
        out.append("| %d | `%s` | %s | %s | %.1f | %.1f | %.1f | %.0f | %.2f | %s | %s | %s | %s | %s | %s | %s | %s | %s |" % (
            i, short_any(r[kn]), r[hdr.index("launch__grid_size")] if "launch__grid_size" in hdr else "",
            r[hdr.index("launch__registers_per_thread")] if "launch__registers_per_thread" in hdr else "",
            t * 1e6, rd / 1e6, wr / 1e6, gbs, gbs / peak,
            pct("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
            pct("lts__throughput.avg.pct_of_peak_sustained_elapsed"),
            pct("l1tex__throughput.avg.pct_of_peak_sustained_elapsed"),
            pct("sm__throughput.avg.pct_of_peak_sustained_elapsed"),
            pct("l1tex__t_sector_hit_rate.pct"), pct("lts__t_sector_hit_rate.pct"),
            pct("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"),
            pct("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio"),
            pct("smsp__issue_active.avg.pct_of_peak_sustained_active")))
    open(os.path.join(PROF, tag + "_kernels.md"), "w").write("\n".join(out) + "\n")
    return data, hdr, units


if __name__ == "__main__":
    os.makedirs(PROF, exist_ok=True)
    tag = sys.argv[1]
    if sys.argv[2] == "--csr-only":
        # summarize_ncu.py <tag> --csr-only <raw.csv> "<what>": a capture filtered to the CSR kernels
        iteration_table(tag, sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else "Krylov iteration")
    elif sys.argv[2] == "--iteration":
        # summarize_ncu.py <tag> --iteration <raw.csv> <launches.csv> "<what>"
        iteration_table(tag, sys.argv[3], sys.argv[5] if len(sys.argv) > 5 else "Krylov iteration")
        launch_shares(tag, sys.argv[4])
    else:
        launch_shares(tag, sys.argv[2])
        if len(sys.argv) > 3:
            full_capture(tag, sys.argv[3])
