#!/usr/bin/env python
"""bench_view_valid.py -- what `view -v` (bdepth_view_opts.valid: BioD's isValid on every read, k_view_valid) adds to `view -c` and to the SAM
lines on the GPU, over the chr20 benchmark file of bench.py.

  python tools/bench_view_valid.py [--steps 10] [--warmup 3]

Input: bench.py's workload (synthetic 30x chr20, 2.26 GB BAM, 12,888,833 reads, seed 20), generated on first use into the same temporary
directory bench.py uses.  Nothing is written into the tree.  The file is staged once (bdepth_stage) and the arms run alternating, call by call,
so that they share the machine's state:
  count / count_v : whole-file `view -c` without and with -v;
  sam / sam_v     : whole-file SAM lines without and with -v, handed to a sink that only counts the bytes.
Per arm: the host clock around each call (it ends in a stream synchronise), the library's CUDA-event span, and ms_reduce (k_view_count, or the
formatting kernels -- with -v, k_view_valid is inside it).  After the timed calls every arm is checked against the CPU restatement
(tools/view_count_oracle.c): the counts with and without -v, the SAM text by SHA-256 and length.  bamgen's reads are all valid and carry no tags,
so the tag walk's cost is not measured here.  One JSON line, with the card's name and power limit read in the same call.
"""
import argparse
import hashlib
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import bench
    import sambamba_b200 as sb
    import view_count_common as vc
    import view_text_common as vt
    import view_valid_common as vv
    from bench_flagstat import card
    info = card()
    path = bench.ensure_workload(1, bench.READS_PER_UNIT)
    size = os.path.getsize(path)
    arms = {"count": lambda h: h.run_view_count(), "count_v": lambda h: h.run_view_count(valid=True),
            "sam": lambda h: h.run_view_text(sink=lambda c: None), "sam_v": lambda h: h.run_view_text(valid=True, sink=lambda c: None)}
    rec = {k: {"host": [], "span": [], "reduce": []} for k in arms}
    res = {}
    with sb.BDepth(path) as h:
        h.stage()
        for i in range(a.warmup + a.steps):
            for k, f in arms.items():
                t0 = time.perf_counter()
                res[k] = f(h)
                dt = (time.perf_counter() - t0) * 1e3
                st = h.stats()
                if i >= a.warmup:
                    rec[k]["host"].append(dt); rec[k]["span"].append(st["ms_span_device"]); rec[k]["reduce"].append(st["ms_reduce"])
        sha = {}
        for k, v in (("sam", False), ("sam_v", True)):            # the text of each SAM arm, after the timed calls
            d = hashlib.sha256()
            n = h.run_view_text(valid=v, sink=d.update)
            sha[k] = (d.hexdigest(), n)
    want_sha = vt.oracle_sha256(path)
    with vv.valid_oracle():
        want_v = vc.oracle_count(path)
    want = vc.oracle_count(path)
    verified = (res["count"] == want and res["count_v"] == want_v and sha["sam"] == want_sha and sha["sam_v"] == want_sha and res["sam"] == res["sam_v"] == want_sha[1])
    med = lambda v: round(statistics.median(v), 3)      # noqa: E731
    out = {k: {"host_ms_median": med(r["host"]), "host_ms_min": round(min(r["host"]), 3), "host_ms_max": round(max(r["host"]), 3),
               "device_span_ms_median": med(r["span"]), "ms_reduce_median": med(r["reduce"]), "result": res[k]} for k, r in rec.items()}
    line = {"metric": "view_v_added_ms", "unit": "ms", "card": info, "workload": f"{os.path.basename(path)}: {size:,} B BAM, {bench.READS_PER_UNIT:,} reads, seed 20",
            "count_v_minus_count_ms": round(out["count_v"]["host_ms_median"] - out["count"]["host_ms_median"], 3),
            "sam_v_minus_sam_ms": round(out["sam_v"]["host_ms_median"] - out["sam"]["host_ms_median"], 3),
            "arms": out, "oracle": {"count": want, "count_v": want_v, "sam_sha256": want_sha[0], "sam_bytes": want_sha[1]}, "verified": verified}
    print(json.dumps(line))
    return 0 if verified else 1


if __name__ == "__main__":
    sys.exit(main())
