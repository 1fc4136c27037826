"""`sambamba view -f bam` on the GPU (bdepth_run_view_bam) against the CPU restatement (tools/view_count_oracle.c, pinned in
tests/test_oracle_view_bam.py), case for case as tests/test_gpu_view_text.py: in every case the member ISIZE list and each member's inflated bytes
are the oracle's, every frame field (header, BSIZE, CRC32, ISIZE) and the trailing EOF member are exact, level 0 is the oracle's file byte for
byte, and the file opened from memory gives the input's SAM lines and flagstat under the same selection."""
import hashlib
import os
import random
import struct
import sys

import numpy as np
import pytest

import flagstat_common as fc
import helpers
import test_gpu_view_text as tvt
import view_bam_common as vb
import view_text_common as vt

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
EMULATE = tvt.EMULATE
gen = tvt.gen
edge = tvt.edge


def check(b, path, level=-1, header=b"@HD\tVN:1.6\tSO:coordinate\n@CO\tview -f bam\n", **kw):
    """b.run_view_bam(header, level, **kw) against the oracle; returns the file."""
    chunks = []
    n = b.run_view_bam(header, level, sink=chunks.append, **kw)
    got = b"".join(chunks)
    assert n == len(got) and chunks[-1] == vb.BGZF_EOF
    raw, sizes, want = vb.oracle_bam(path, header, level, **kw)
    vb.check_against_oracle(got, raw, sizes, want, level)
    return got


def test_golden_levels():
    for name in ("issue_204.bam", "mate_overlaps_1_3M_4M.bam", "issue225.bam"):
        p = os.path.join(helpers.GOLDEN, name)
        with tvt.bdepth(p) as b:
            for level in (0, -1, 1, 9):
                check(b, p, level)
            for kw in (dict(num_filter=(0, 0x404)), dict(subsample=0.3, seed=77), dict(valid=True)):
                check(b, p, 0, **kw)


def test_edge_file(edge):
    p = edge["path"]
    with tvt.bdepth(p) as b:
        for case in tvt.EDGE_CASES:
            check(b, p, 0, **case)
            check(b, p, -1, **case)


@pytest.mark.parametrize("tuning", [(1 << 16, 1), (1 << 17, 3), (1 << 20, 7)])
def test_tiny_batches_members_span_sub_batches(gen, tuning):
    p = gen["pairs"]
    with tvt.bdepth(p, tuning) as b:
        for level in (0, -1):
            got = check(b, p, level)
        assert len(vb.members(got)) > 3
        for kw in (dict(num_filter=(0x41, 0x100)), dict(subsample=0.1, seed=2)):
            check(b, p, 0, **kw)


def test_round_trip(gen):
    import sambamba_b200 as sb
    p = gen["pairs"]
    with tvt.bdepth(p) as b:
        for kw in (dict(), dict(num_filter=(0x41, 0x100), subsample=0.5, seed=3)):
            got = b.run_view_bam(b"@HD\tVN:1.6\n", -1, **kw)
            with sb.BDepth(memory=np.frombuffer(got, dtype=np.uint8).copy()) as c:
                assert c.run_view_text() == b.run_view_text(**kw)
                assert c.run_view_count() == b.run_view_count(**kw)
                if not kw:
                    assert c.run_flagstat() == b.run_flagstat()


def test_bed_sorted_sparse_and_unsorted(gen, tmp_path):
    p = gen["plain"]
    bed = tvt._bed_one_percent(p, 5) + [(2, 10, 900)]
    for tuning in (None, (1 << 17, 2)):
        with tvt.bdepth(p, tuning) as b:
            check(b, p, -1, bed=bed)
            check(b, p, 0, bed=bed)
    u = helpers.oracle_inflate(p)
    first, refs = helpers.header_first_record_offset(u)
    raw = u.tobytes()
    recs = [raw[r[0]:r[0] + 4 + struct.unpack_from("<i", raw, r[0])[0]] for r in helpers.parse_records(u, first)]
    random.Random(4).shuffle(recs)
    q = helpers.write_bgzf(str(tmp_path / "raw.bam"), fc.bam_body(refs, recs), len(refs))
    os.remove(q + ".bai")
    with tvt.bdepth(q) as b:
        check(b, q, 0, bed=bed)
        check(b, q, -1)


def test_positional_regions_one_stream(gen):
    p = gen["plain"]
    bed = tvt._bed_one_percent(p, 6)
    regs = bed[:4] + ["*"] + bed[:2] + [(1, 0, 700), (0, bed[0][1], bed[0][2] + 5000), (2, 5, 6)]
    with tvt.bdepth(p) as b:
        check(b, p, 0, regions=regs)
        check(b, p, -1, regions=regs[:3] + ["*"], num_filter=(0, 4), subsample=0.4, seed=3)
    with tvt.bdepth(p, (1 << 17, 2)) as b:
        check(b, p, 0, regions=regs)


def test_staged_and_memory(gen):
    import sambamba_b200 as sb
    p = gen["pairs"]
    kw = dict(num_filter=(1, 0x400), subsample=0.5, seed=4)
    raw, sizes, want = vb.oracle_bam(p, b"", 0, **kw)
    with sb.BDepth(p) as b:
        b.stage()
        for _ in range(2):
            assert b.run_view_bam(b"", 0, **kw) == want
            st = b.stats()
            assert st["ms_reduce"] > 0 and st["ms_d2h"] > 0
    with sb.BDepth(memory=np.fromfile(p, dtype=np.uint8)) as b:
        assert b.run_view_bam(b"", 0, **kw) == want


def test_refusals(gen, tmp_path):
    import sambamba_b200 as sb
    p = gen["pairs"]
    with sb.BDepth(p) as b:
        for lv in (-2, 10):
            with pytest.raises(sb.BDepthError, match=r"Compression level must be a number in interval \[-1, 9\]"):
                b.run_view_bam(b"", lv)

        def stop(_c):
            raise KeyError("stop")
        with pytest.raises(sb.BDepthError, match="callback aborted") as e:
            b.run_view_bam(b"", -1, sink=stop)
        assert isinstance(e.value.__cause__, KeyError)
    with sb.BDepth(p) as b:
        b.set_shard(0, 2)
        with pytest.raises(sb.BDepthError, match="several ranks"):
            b.run_view_bam(b"", -1)
    with sb.BDepth(p) as b:
        b.add_input(p)
        with pytest.raises(sb.BDepthError, match="several inputs"):
            b.run_view_bam(b"", -1)
    recs = [vt.record("a", 0, 0, 5, 30, [(2, 0)], -1, -1, 0, "AC"), vt.record("x", 0, -2, 5, 30, [(2, 0)], -1, -1, 0, "AC")]
    q = vt.write_records(str(tmp_path / "bad.bam"), [("c1", 1000)], recs, index=False)
    with sb.BDepth(q) as b:
        with pytest.raises(sb.BDepthError, match="Read reference ID is out of range"):
            b.run_view_bam(b"", -1)
        assert b.run_view_bam(b"", 0, num_filter=(0x400, 0)) == vb.oracle_bam(q, b"", 0, num_filter=(0x400, 0))[2]      # (only selected reads are checked)


def test_full_size(tmp_path_factory):
    """The chr20 benchmark file (a small file of its shape under the emulation): the inflated stream by SHA-256, whole and with a 1 % -L."""
    if EMULATE:
        p = helpers.gen_bam(str(tmp_path_factory.mktemp("vbz") / "small.bam"), "-r", "chr20:300000", "-n", 20000, "-s", 20, "-t", 4)
    else:
        sys.path.insert(0, helpers.ROOT)
        import bench
        p = bench.ensure_workload(1, bench.READS_PER_UNIT)
    with tvt.bdepth(p) as b:
        L = b.refs[0][1]
        for kw in (dict(), dict(bed=[(0, L // 2, L // 2 + L // 100)])):
            got = b.run_view_bam(b"@HD\tVN:1.6\n", -1, **kw)
            ms = vb.members(got)
            raw, sizes, _ = vb.oracle_bam(p, b"@HD\tVN:1.6\n", 0, **kw)
            h = hashlib.sha256()
            for _, x in ms:
                h.update(x)
            assert [len(x) for _, x in ms] == sizes and h.hexdigest() == hashlib.sha256(raw).hexdigest()
            del raw, ms, got
