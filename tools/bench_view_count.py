#!/usr/bin/env python
"""bench_view_count.py -- `sambamba view -c` on the GPU (bdepth_run_view_count) over the chr20 benchmark file of bench.py.

  python tools/bench_view_count.py [--steps 10] [--warmup 3]

Input: bench.py's workload (synthetic 30x chr20, 2.26 GB BAM, 12,888,833 reads, seed 20), generated on first use into the same temporary
directory bench.py uses.  Nothing is written into the tree.
  resident   : bdepth_stage, then `warmup` untimed and `steps` timed whole-file counts: host clock around each call (it ends in a stream
               synchronise) and the library's CUDA-event times (span, K1 inflate, K2 scan, k_view_count).
  resident_f : the same with --num-filter=0/1028 -s 0.1 (flag bits and the subsampling hash on every record).
  e2e        : bdepth_open_memory on a pinned host image of the file, whole-file counts: H2D of the compressed bytes inside every call.
  sparse     : a -L query of one region covering 1 % of chr20 (its middle), the file opened by path: only the region's BAI chunks are read,
               copied and inflated in every call.
Every count of the last timed call of each arm is checked against the CPU restatement (tools/view_count_oracle.c) after the timed regions.
One JSON line, with the card's name and power limit read in the same call.
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def timed(h, warmup, steps, kw):
    for _ in range(warmup):
        h.run_view_count(**kw)
    host, span, k1, k2, census = [], [], [], [], []
    got = None
    for _ in range(steps):
        t0 = time.perf_counter()
        got = h.run_view_count(**kw)
        host.append((time.perf_counter() - t0) * 1e3)
        st = h.stats()
        span.append(st["ms_span_device"]); k1.append(st["ms_inflate"]); k2.append(st["ms_scan"]); census.append(st["ms_reduce"])
    med = lambda v: round(statistics.median(v), 3)
    return got, {"host_ms_median": med(host), "host_ms_min": round(min(host), 3), "host_ms_max": round(max(host), 3), "device_span_ms_median": med(span),
                 "k1_inflate_ms_median": med(k1), "k2_scan_ms_median": med(k2), "k_view_count_ms_median": med(census), "n_batches": st["n_batches"],
                 "gpu_launches": st["gpu_launches"], "file_bytes": st["file_bytes"], "count": got}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import bench
    import sambamba_b200 as sb
    import view_count_common as vc
    from bench_flagstat import card
    info = card()
    path = bench.ensure_workload(1, bench.READS_PER_UNIT)
    size = os.path.getsize(path)
    flt = dict(num_filter=(0, 1028), subsample=0.1, seed=20)
    with sb.BDepth(path) as h:
        L = h.refs[0][1]
        bed = [(0, L // 2, L // 2 + L // 100)]
        h.stage()
        _, resident = timed(h, a.warmup, a.steps, {})
        _, resident_f = timed(h, a.warmup, a.steps, flt)
    with sb.BDepth(path) as h:
        _, sparse = timed(h, a.warmup, a.steps, dict(bed=bed))
    img, keep = bench.pinned_file(path)
    with sb.BDepth(memory=img) as h:
        _, e2e = timed(h, a.warmup, a.steps, {})
    del keep
    want = {"resident": vc.oracle_count(path), "resident_f": vc.oracle_count(path, **flt), "sparse": vc.oracle_count(path, bed=bed)}
    verified = resident["count"] == e2e["count"] == want["resident"] and resident_f["count"] == want["resident_f"] and sparse["count"] == want["sparse"]
    gb = size / 1e9
    line = {"metric": "bam_gb_per_s_view_count", "unit": "GB/s", "card": info, "workload": f"{os.path.basename(path)}: {size:,} B BAM, {bench.READS_PER_UNIT:,} reads, seed 20",
            "value": round(gb / (resident["host_ms_median"] / 1e3), 3), "resident": resident, "resident_f": dict(resident_f, selection="--num-filter=0/1028 -s 0.1"),
            "e2e": dict(e2e, value=round(gb / (e2e["host_ms_median"] / 1e3), 3)), "sparse": dict(sparse, region="chr20:%d-%d" % (bed[0][1] + 1, bed[0][2])),
            "oracle": want, "verified": verified}
    print(json.dumps(line))
    return 0 if verified else 1


if __name__ == "__main__":
    sys.exit(main())
