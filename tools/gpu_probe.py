"""Ad-hoc timing probe (needs a GPU): per-stage device times from bdepth_stats."""
import os, sys, time, json, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import sambamba_b200 as sb
import helpers

def probe(path, reps=2, check=False):
    t0 = time.time(); b = sb.BDepth(path); t1 = time.time()
    print(f"open {path}: {t1-t0:.3f}s  file={os.path.getsize(path)/1e6:.1f} MB", flush=True)
    for r in range(reps):
        t0 = time.time(); b.run_base(collect=False); t1 = time.time()
        st = b.stats()
        print(f"  run{r}: wall {t1-t0:.3f}s  " + json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in st.items()}), flush=True)
    b.stage()
    for r in range(reps):
        t0 = time.time(); b.run_base(collect=False); t1 = time.time()
        st = b.stats()
        print(f"  staged run{r}: wall {t1-t0:.3f}s  h2d {st['ms_h2d']:.2f} k1 {st['ms_inflate']:.2f} k2 {st['ms_scan']:.2f} k3 {st['ms_coverage']:.2f} d2h {st['ms_d2h']:.2f}", flush=True)
    if check:
        t0 = time.time(); got = b.run_base(); t1 = time.time(); want, _ = helpers.oracle_counts(path, threads=16); t2 = time.time()
        print(f"  collect {t1-t0:.2f}s oracle {t2-t1:.2f}s equal={np.array_equal(got, want)}", flush=True)
    b.close()

if __name__ == "__main__":
    d = "/tmp/probe"; os.makedirs(d, exist_ok=True)
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2000000
    t0 = time.time(); helpers.gen_bam(f"{d}/tiny.bam", "--preset", "tiny", "-t", 4); print("gen tiny", time.time() - t0, flush=True)
    probe(f"{d}/tiny.bam")
    t0 = time.time(); helpers.gen_bam(f"{d}/part.bam", "-r", "chr20:64444167", "-n", n, "-s", 20, "-t", 64); print("gen part", time.time() - t0, flush=True)
    probe(f"{d}/part.bam", check=True)
