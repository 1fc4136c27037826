#!/usr/bin/env python
"""bench_view_text.py -- `sambamba view`'s SAM lines on the GPU (bdepth_run_view_text) over the chr20 benchmark file of bench.py.

  python tools/bench_view_text.py [--steps 5] [--warmup 2]

Arms as in bench_view_count.py: resident (bdepth_stage), e2e (bdepth_open_memory on a pinned host image) and sparse (a -L query of 1 % of
chr20, file opened by path).  Timed calls hand the text to a callback that discards it (through the C ABI, no copy into Python objects).
After the timed regions each arm runs once more with a hashing callback; its SHA-256 and byte count must equal those of the CPU restatement's
text (tools/view_count_oracle.c).  One JSON line, with the card's name and power limit read in the same call.  Nothing is written into the tree.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, d)


ENTRY = {"sam": "bdepth_run_view_text", "json": "bdepth_run_view_json"}


def timed(h, warmup, steps, bed=None, fmt="sam"):
    import sambamba_b200._lib as SL
    o = SL.ViewOpts()
    arr = (SL.Region * max(len(bed or []), 1))(*[SL.Region(*r) for r in bed or []])
    o.regions_from, o.regions, o.n_regions = (1 if bed else 0), arr, len(bed or [])
    nbytes, sha = [0], hashlib.sha256()

    def discard(_user, _ptr, n):
        nbytes[0] += n
        return 0

    def hashing(_user, ptr, n):
        sha.update(C.string_at(ptr, n))
        return 0
    run = lambda cb: h._ck(getattr(h.L, ENTRY[fmt])(h.h, C.byref(o), cb, None))      # noqa: E731
    cb = SL.TEXT_CB(discard)
    for _ in range(warmup):
        run(cb)
    host, st = [], []
    for _ in range(steps):
        nbytes[0] = 0
        t0 = time.perf_counter()
        run(cb)
        host.append((time.perf_counter() - t0) * 1e3)
        st.append(h.stats())
    run(SL.TEXT_CB(hashing))                                 # verification, after the timed region
    med = lambda k: round(statistics.median(s[k] for s in st), 3)      # noqa: E731
    return {"host_ms_median": round(statistics.median(host), 3), "host_ms_min": round(min(host), 3), "host_ms_max": round(max(host), 3),
            "k1_inflate_ms_median": med("ms_inflate"), "k2_scan_ms_median": med("ms_scan"), fmt + "_kernels_ms_median": med("ms_reduce"),
            "text_d2h_ms_median": med("ms_d2h"), "file_bytes": st[-1]["file_bytes"], "text_bytes": nbytes[0],
            "text_gb_per_s": round(nbytes[0] / 1e9 / (statistics.median(host) / 1e3), 3), "sha256": sha.hexdigest()}


def main(fmt="sam"):
    """fmt: "sam" (bdepth_run_view_text) or "json" (bdepth_run_view_json, for bench_view_json.py)."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import bench
    import sambamba_b200 as sb
    vt = __import__("view_json_common" if fmt == "json" else "view_text_common")      # the oracle's SHA-256 of the same text
    from bench_flagstat import card
    info = card()
    path = bench.ensure_workload(1, bench.READS_PER_UNIT)
    gb = os.path.getsize(path) / 1e9
    with sb.BDepth(path) as h:
        L, name = h.refs[0][1], h.refs[0][0]
        bed = [(0, L // 2, L // 2 + L // 100)]
        h.stage()
        resident = timed(h, a.warmup, a.steps, fmt=fmt)
    with sb.BDepth(path) as h:
        sparse = timed(h, a.warmup, a.steps, bed=bed, fmt=fmt)
    img, keep = bench.pinned_file(path)
    with sb.BDepth(memory=img) as h:
        e2e = timed(h, a.warmup, a.steps, fmt=fmt)
    del keep
    want = vt.oracle_sha256(path)
    want_s = vt.oracle_sha256(path, bed="%s\t%d\t%d\n" % (name, bed[0][1], bed[0][2]))
    verified = (resident["sha256"], resident["text_bytes"]) == (e2e["sha256"], e2e["text_bytes"]) == want and (sparse["sha256"], sparse["text_bytes"]) == want_s
    print(json.dumps({"metric": "bam_gb_per_s_view_" + ("json" if fmt == "json" else "text"), "unit": "GB/s", "card": info, "workload": f"{os.path.basename(path)}: {bench.READS_PER_UNIT:,} reads, seed 20",
                      "value": round(gb / (resident["host_ms_median"] / 1e3), 3), "resident": resident, "e2e": dict(e2e, value=round(gb / (e2e["host_ms_median"] / 1e3), 3)),
                      "sparse": dict(sparse, region="%s:%d-%d" % (name, bed[0][1] + 1, bed[0][2])), "oracle": [want, want_s], "verified": verified}))
    return 0 if verified else 1


if __name__ == "__main__":
    sys.exit(main())
