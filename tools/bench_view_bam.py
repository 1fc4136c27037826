#!/usr/bin/env python
"""bench_view_bam.py -- `sambamba view -f bam` on the GPU (bdepth_run_view_bam) over the chr20 benchmark file of bench.py.

  python tools/bench_view_bam.py [--steps 3] [--warmup 1]

Arms at levels 0 and -1: resident (bdepth_stage), e2e (bdepth_open_memory on a pinned host image) and sparse (a -L query of 1 % of chr20).
Timed calls hand the members to a callback that discards them (through the C ABI).  After the timed regions each arm runs once more with a
callback that keeps the file: its members' ISIZE list and the SHA-256 of the inflated stream must equal the CPU restatement's
(tools/view_count_oracle.c), and at level 0 the file must be the restatement's byte for byte.  For context it reports the compression ratio
against zlib level 6 on every 16th member of the level -1 file, and zlib's level-6 rate on those members on one host thread and on all of
them.  One JSON line, with the card's name and power limit read in the same call.  Nothing is written into the tree.
"""
import argparse
import ctypes as C
import hashlib
import json
import multiprocessing as mp
import os
import statistics
import sys
import time
import zlib

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, d)
HEADER = b"@HD\tVN:1.6\tSO:coordinate\n"


def timed(h, warmup, steps, level, bed=None):
    import sambamba_b200._lib as SL
    o = SL.ViewOpts()
    arr = (SL.Region * max(len(bed or []), 1))(*[SL.Region(*r) for r in bed or []])
    o.regions_from, o.regions, o.n_regions = (1 if bed else 0), arr, len(bed or [])
    nbytes, keep = [0], []

    def discard(_user, _ptr, n):
        nbytes[0] += n
        return 0

    def keeping(_user, ptr, n):
        keep.append(C.string_at(ptr, n))
        return 0
    run = lambda cb: h._ck(h.L.bdepth_run_view_bam(h.h, C.byref(o), HEADER, len(HEADER), level, cb, None))      # noqa: E731
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
    run(SL.TEXT_CB(keeping))                                 # verification, after the timed region
    med = lambda k: round(statistics.median(s[k] for s in st), 3)      # noqa: E731
    return {"host_ms_median": round(statistics.median(host), 3), "host_ms_min": round(min(host), 3), "host_ms_max": round(max(host), 3),
            "k1_inflate_ms_median": med("ms_inflate"), "k2_scan_ms_median": med("ms_scan"), "gather_cut_compress_ms_median": med("ms_reduce"),
            "d2h_ms_median": med("ms_d2h"), "file_bytes": st[-1]["file_bytes"], "out_bytes": nbytes[0]}, b"".join(keep)


def _z6(m):
    return len(zlib.compress(m, 6, -15)) + 26


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import bench
    import sambamba_b200 as sb
    import view_bam_common as vb
    from bench_flagstat import card
    info = card()
    path = bench.ensure_workload(1, bench.READS_PER_UNIT)
    gb = os.path.getsize(path) / 1e9
    with sb.BDepth(path) as h:
        L = h.refs[0][1]
    bed = [(0, L // 2, L // 2 + L // 100)]
    want = {}
    for key, kw in (("whole", {}), ("sparse", dict(bed=bed))):      # the oracle once per selection (level 0: its file is the raw stream framed)
        raw, sizes, f0 = vb.oracle_bam(path, HEADER, 0, **kw)
        want[key] = (sizes, hashlib.sha256(raw).hexdigest(), hashlib.sha256(f0).hexdigest())
        del raw, f0
    out, sample, verified = {}, None, True

    def verify(name, f, key, lv):
        nonlocal sample, verified
        ms = vb.members(f)
        hs = hashlib.sha256()
        for _, x in ms:
            hs.update(x)
        sizes, sha_raw, sha_file = want[key]
        ok = [len(x) for _, x in ms] == sizes and hs.hexdigest() == sha_raw and (lv != 0 or hashlib.sha256(f).hexdigest() == sha_file)
        out[name].update(members=len(ms), inflated_sha256=hs.hexdigest(), verified=ok, value=round(gb / (out[name]["host_ms_median"] / 1e3), 3))
        verified = verified and ok
        if name == "resident_l-1":
            sample = [(len(d) + 26, x) for d, x in ms[::16]]

    with sb.BDepth(path) as h:
        h.stage()
        for lv in (0, -1):
            out["resident_l%d" % lv], f = timed(h, a.warmup, a.steps, lv)
            verify("resident_l%d" % lv, f, "whole", lv)
    with sb.BDepth(path) as h:
        for lv in (0, -1):
            out["sparse_l%d" % lv], f = timed(h, a.warmup, a.steps, lv, bed=bed)
            verify("sparse_l%d" % lv, f, "sparse", lv)
    img, keep = bench.pinned_file(path)
    with sb.BDepth(memory=img) as h:
        for lv in (0, -1):
            out["e2e_l%d" % lv], f = timed(h, a.warmup, a.steps, lv)
            verify("e2e_l%d" % lv, f, "whole", lv)
    del keep, f
    ours = sum(c for c, _ in sample)
    sample = [x for _, x in sample]
    t0 = time.perf_counter(); z = sum(_z6(m) for m in sample); t1 = time.perf_counter() - t0
    n = os.cpu_count() or 1
    with mp.Pool(n) as pool:
        t0 = time.perf_counter(); pool.map(_z6, sample, chunksize=8); tn = time.perf_counter() - t0
    mb = sum(len(m) for m in sample) / 1e6
    ctx = {"sample_members": len(sample), "ratio_vs_zlib6": round(ours / z, 4), "zlib6_one_thread_mb_per_s": round(mb / t1, 1),
           "zlib6_all_threads_mb_per_s": round(mb / tn, 1), "host_threads": n}
    print(json.dumps({"metric": "bam_gb_per_s_view_bam", "unit": "GB/s (input BAM)", "card": info, "workload": f"{os.path.basename(path)}: {bench.READS_PER_UNIT:,} reads, seed 20",
                      "value": out["resident_l-1"]["value"], "arms": out, "zlib_context": ctx, "verified": verified}))
    return 0 if verified else 1


if __name__ == "__main__":
    sys.exit(main())
