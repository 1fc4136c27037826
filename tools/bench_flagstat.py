#!/usr/bin/env python
"""bench_flagstat.py -- `sambamba flagstat` on the GPU (bdepth_run_flagstat) over the chr20 benchmark file of bench.py.

  python tools/bench_flagstat.py [--steps 10] [--warmup 3] [--no-cpu]

Input: bench.py's workload (synthetic 30x chr20, 2.26 GB BAM, 12,888,833 reads, seed 20), generated on first use into the same temporary
directory bench.py uses.  Nothing is written into the tree.
  resident : bdepth_stage, then `warmup` untimed and `steps` timed bdepth_run_flagstat calls: host clock around each call (it ends in a
             stream synchronise) and the library's CUDA-event times (span, K1 inflate, K2 scan, k_flagstat census).
  e2e      : bdepth_open_memory on a pinned host image of the file, then the same calls: H2D of the compressed bytes inside every call.
  cpu      : tools/flagstat_oracle.c over the same file on the host's cores (a restatement of computeFlagStatistics, not sambamba).
The counters of the last timed call of each GPU arm are checked against the CPU restatement after the timed regions.  One JSON line,
with the card's name and power limit read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power, clk = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:  # the numbers are meaningless without it, but the line still says so
        return {"name": None, "power_limit": None, "error": repr(e)[:200]}


def timed(h, warmup, steps):
    for _ in range(warmup):
        h.run_flagstat()
    host, span, k1, k2, census = [], [], [], [], []
    got = None
    for _ in range(steps):
        t0 = time.perf_counter()
        got = h.run_flagstat()
        host.append((time.perf_counter() - t0) * 1e3)
        st = h.stats()
        span.append(st["ms_span_device"]); k1.append(st["ms_inflate"]); k2.append(st["ms_scan"]); census.append(st["ms_reduce"])
    med = lambda v: round(statistics.median(v), 3)
    return got, {"host_ms_median": med(host), "host_ms_min": round(min(host), 3), "host_ms_max": round(max(host), 3), "device_span_ms_median": med(span),
                 "k1_inflate_ms_median": med(k1), "k2_scan_ms_median": med(k2), "k_flagstat_ms_median": med(census), "n_batches": st["n_batches"], "gpu_launches": st["gpu_launches"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU arm (its run also verifies the GPU counters)")
    a = ap.parse_args()
    import bench
    import flagstat_common as fc
    import sambamba_b200 as sb
    info = card()
    path = bench.ensure_workload(1, bench.READS_PER_UNIT)
    size = os.path.getsize(path)
    with sb.BDepth(path) as h:
        h.stage()
        res_counts, resident = timed(h, a.warmup, a.steps)
    img, keep = bench.pinned_file(path)
    with sb.BDepth(memory=img) as h:
        e2e_counts, e2e = timed(h, a.warmup, a.steps)
    del keep
    cpu = None
    verified = None
    if not a.no_cpu:
        t0 = time.perf_counter()
        want = fc.oracle_flagstat(path)
        cpu = {"kind": "restatement, not sambamba", "impl": "tools/flagstat_oracle.c (zlib on %d threads + serial record walk)" % min(32, os.cpu_count() or 1),
               "s": round(time.perf_counter() - t0, 3)}
        verified = res_counts == want and e2e_counts == want
    gb = size / 1e9
    line = {"metric": "bam_gb_per_s_flagstat", "unit": "GB/s", "card": info, "workload": f"{os.path.basename(path)}: {size:,} B BAM, {bench.READS_PER_UNIT:,} reads, seed 20",
            "value": round(gb / (resident["host_ms_median"] / 1e3), 3), "resident": resident,
            "e2e": dict(e2e, value=round(gb / (e2e["host_ms_median"] / 1e3), 3)),
            "cpu": dict(cpu, value=round(gb / cpu["s"], 3)) if cpu else None, "verified": verified, "total_records": sum(res_counts["total"])}
    print(json.dumps(line))
    return 0 if verified is not False else 1


if __name__ == "__main__":
    sys.exit(main())
