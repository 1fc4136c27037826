#!/usr/bin/env python
"""bench_view_json.py -- `sambamba view -f json` on the GPU (bdepth_run_view_json) over the chr20 benchmark file of bench.py.

  python tools/bench_view_json.py [--steps 5] [--warmup 2]

The arms and the verification of bench_view_text.py: resident (bdepth_stage), e2e (bdepth_open_memory on a pinned host image) and sparse (a -L
query of 1 % of chr20, file opened by path); timed calls hand the text to a callback that discards it; after the timed regions each arm's
SHA-256 and byte count must equal those of the CPU restatement's JSON text (tools/view_count_oracle.c -f json).  One JSON line, with the card's
name and power limit read in the same call.  Nothing is written into the tree.
"""
import os
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

if __name__ == "__main__":
    import bench_view_text
    sys.exit(bench_view_text.main("json"))
