"""Run `depth base` through the C ABI on a given (or generated) BAM: a small target for profiler runs.
usage: probe_one.py BAM [n_reads_if_missing] [reps] [--staged]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import sambamba_b200 as sb
import helpers
args = [a for a in sys.argv[1:] if not a.startswith("--")]
staged = "--staged" in sys.argv
path = args[0] if args else "/tmp/probe/one.bam"
if not os.path.exists(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    n = args[1] if len(args) > 1 else "200000"
    helpers.gen_bam(path, "-r", "chr20:64444167", "-n", n, "-s", "20", "-t", "32")
reps = int(args[2]) if len(args) > 2 else 1
with sb.BDepth(path) as b:
    if staged:
        b.stage()
    for _ in range(reps):
        if staged:
            b.run_resident()
        else:
            b.run_base(collect=False)
    print(b.stats())
