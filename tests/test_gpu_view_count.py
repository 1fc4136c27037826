"""`sambamba view -c` on the GPU (bdepth_run_view_count, the CLI's `view -c`) against the CPU restatement (tools/view_count_oracle.c, pinned in
tests/test_oracle_view_count.py).  -F is composed as in test_zz_gpu_filter.py: a Python statement of each query reduces the file, and the oracle
counts the reduced file."""
import glob
import multiprocessing as mp
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

import flagstat_common as fc
import helpers
import test_emul_filter as tef
import view_count_common as vc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
EMULATE = os.environ.get("BDEPTH_EMULATE") == "1"
GOLDEN = sorted(glob.glob(os.path.join(helpers.GOLDEN, "*.bam")))


def gpu_count(path, tuning=None, stats=False, **kw):
    import sambamba_b200 as sb
    with sb.BDepth(path) as b:
        if tuning:
            b.set_tuning(*tuning)
        n = b.run_view_count(**kw)
        return (n, b.stats()) if stats else n


@pytest.fixture(scope="module")
def gen(tmp_path_factory):
    d = tmp_path_factory.mktemp("vc")
    n = 20000 if EMULATE else 200000
    return {"plain": helpers.gen_bam(str(d / "g.bam"), "-r", "chrA:%d" % (n * 10), "-r", "chrB:700", "-r", "chrC:%d" % (n * 5), "-n", n, "-s", 31, "-t", 8),
            "pairs": helpers.gen_bam(str(d / "p.bam"), "-r", "chrA:%d" % (n * 10), "-n", n, "-s", 32, "-t", 8, "--pairs", 5), "n": n, "dir": d}


@pytest.fixture(scope="module")
def edge(tmp_path_factory):
    d = tmp_path_factory.mktemp("vce")
    s = vc.write_edge_bam(str(d / "s.bam"))
    with open(s + ".bai", "wb") as f:                # a real index: positional queries and -L stage their chunks
        f.write(helpers.oracle_build_bai(s))
    return {"sorted": s, "unsorted": vc.write_edge_bam(str(d / "u.bam"), sorted_file=False), "dir": d}


EDGE_CASES = [dict(), dict(num_filter=(0, 4)), dict(num_filter=(1, 0)), dict(subsample=0.5, seed=9), dict(bed=[(0, 500, 600), (0, 200, 300), (0, 100, 200)]),
              dict(bed=[(0, 100, 101)]), dict(bed=[(1, 149, 150), (0, 100, 200)]), dict(regions=[(0, 100, 200), (0, 150, 300), (0, 100, 200)], n_unmapped=1),
              dict(n_unmapped=2), dict(regions=[(1, 40, 41)]), dict(regions=[(0, 0, 10000)], num_filter=(0, 0x400), subsample=0.7, seed=1)]


@pytest.mark.parametrize("case", range(len(EDGE_CASES)))
def test_edge_file(edge, case):
    kw = EDGE_CASES[case]
    want = vc.oracle_count(edge["sorted"], **kw)
    assert gpu_count(edge["sorted"], **kw) == want
    if "regions" not in kw and "n_unmapped" not in kw:
        assert gpu_count(edge["unsorted"], **kw) == vc.oracle_count(edge["unsorted"], **kw) == want


def test_edge_refusals(edge):
    import sambamba_b200 as sb
    with sb.BDepth(edge["unsorted"]) as b:
        with pytest.raises(sb.BDepthError) as e:
            b.run_view_count(bed=[])                 # BedFilter over an empty region list
        assert e.value.code == -7
    with sb.BDepth(edge["sorted"]) as b:
        assert b.run_view_count(bed=[]) == 0
        with pytest.raises(sb.BDepthError, match="start must be less than end"):
            b.run_view_count(regions=[(0, 7, 7)])
    os.rename(edge["sorted"] + ".bai", edge["sorted"] + ".bak")
    try:
        with sb.BDepth(edge["sorted"]) as b:
            assert b.run_view_count() == 11          # the whole file needs no index
            for kw in (dict(regions=[(0, 1, 5)]), dict(n_unmapped=1), dict(bed=[(0, 1, 5)])):
                with pytest.raises(sb.BDepthError) as e:
                    b.run_view_count(**kw)
                assert e.value.code == -4 and "must be provided" in e.value.msg
    finally:
        os.rename(edge["sorted"] + ".bak", edge["sorted"] + ".bai")


@pytest.mark.parametrize("name", [os.path.basename(p) for p in GOLDEN])
def test_golden(name):
    p = os.path.join(helpers.GOLDEN, name)
    for kw in (dict(), dict(num_filter=(0, 0x404)), dict(subsample=0.3, seed=77)):
        n, st = gpu_count(p, stats=True, **kw)
        assert n == vc.oracle_count(p, **kw)
        assert st["gpu_launches"] > 0


@pytest.mark.parametrize("tuning", [None, (1 << 16, 1), (1 << 17, 3), (1 << 20, 7)])
def test_generated_across_batches(gen, tuning):
    p = gen["pairs"]
    for kw in (dict(), dict(num_filter=(0x41, 0x100)), dict(subsample=0.1, seed=2), dict(subsample=0.9, seed=123456789)):
        assert gpu_count(p, tuning, **kw) == vc.oracle_count(p, **kw), kw


def _bed_one_percent(path, seed):
    """Regions inside 1 % of chrA, some overlapping, some touching, in no order."""
    import sambamba_b200 as sb
    with sb.BDepth(path) as b:
        L = dict(b.refs)["chrA"]
    rnd = random.Random(seed)
    out = []
    lo = rnd.randrange(0, L - L // 100)
    for _ in range(40):
        s = rnd.randrange(lo, lo + L // 100)
        out.append((0, s, s + rnd.randrange(1, L // 4000 + 2)))
    out.append((0, out[0][1] + 5, out[0][2] + 50))
    out.append((0, out[1][2], out[1][2] + 100))
    return out


def test_bed_sorted_sparse_and_shuffled_unindexed(gen, tmp_path):
    import sambamba_b200 as sb
    p = gen["plain"]
    bed = _bed_one_percent(p, 5) + [(2, 10, 900)]
    want = vc.oracle_count(p, bed=bed)
    for tuning in (None, (1 << 17, 2)):
        n, st = gpu_count(p, tuning, stats=True, bed=bed)
        assert n == want > 0
        assert st["file_bytes"] < os.path.getsize(p) // 2, "only the regions' BAI chunks are staged"
    with sb.BDepth(p, lazy=True) as b:
        assert b.run_view_count(bed=bed) == want
    # the same records shuffled under a header without SO:coordinate, no .bai: BedFilter over the whole file
    u = helpers.oracle_inflate(p)
    first, refs = helpers.header_first_record_offset(u)
    raw, recs, o = u.tobytes(), [], first
    while o + 4 <= len(raw):
        bs, = struct.unpack_from("<i", raw, o)
        recs.append(raw[o:o + 4 + bs])
        o += 4 + bs
    random.Random(4).shuffle(recs)
    q = helpers.write_bgzf(str(tmp_path / "raw.bam"), fc.bam_body(refs, recs), len(refs))
    os.remove(q + ".bai")
    with sb.BDepth(q) as b:
        assert not b.coordinate_sorted and not b.has_index
        assert b.run_view_count(bed=bed) == vc.oracle_count(q, bed=bed) == want
        assert b.run_view_count(bed=bed, num_filter=(0, 0x10), subsample=0.5, seed=8) == vc.oracle_count(p, bed=bed, num_filter=(0, 0x10), subsample=0.5, seed=8)


def test_positional_regions_repeats_and_unmapped(gen):
    p = gen["plain"]
    bed = _bed_one_percent(p, 6)
    regs = bed[:6] + bed[:2] + [(1, 0, 700), (2, 5, 6)]
    for kw in (dict(regions=regs), dict(regions=regs, n_unmapped=2), dict(n_unmapped=1), dict(regions=regs[:3], num_filter=(0, 4), subsample=0.4, seed=3)):
        want = vc.oracle_count(p, **kw)
        assert gpu_count(p, **kw) == want and (want > 0 or kw.get("n_unmapped") == 1), kw
        assert gpu_count(p, (1 << 17, 2), **kw) == want


def test_filter_queries(tmp_path):
    """A third of test_emul_filter.QUERIES, alone and with a region and the other selections."""
    p = tef.make_bam(str(tmp_path / "f.bam"), seed=5, n=3000, empty_seq=False)
    u = helpers.oracle_inflate(p)
    _, recs = tef.parse_all(u)
    import sambamba_b200 as sb
    with sb.BDepth(p) as b:
        for k, (q, fn) in enumerate(tef.QUERIES):
            if k % 3 != 1:
                continue
            keep = [bool(fn(r)) for r in recs]
            sub = helpers.subset_bam(p, str(tmp_path / f"sub{k}.bam"), keep)
            assert b.run_view_count(query=q) == sum(keep) == vc.oracle_count(sub), q
            kw = dict(bed=[(0, 100, 3000), (1, 50, 400)], num_filter=(0, 0x10), subsample=0.6, seed=k)
            assert b.run_view_count(query=q, **kw) == vc.oracle_count(sub, **kw), q
            assert b.run_view_count(query=q, regions=[(0, 100, 3000), (0, 2000, 2500)]) == vc.oracle_count(sub, regions=[(0, 100, 3000), (0, 2000, 2500)]), q


def test_staged_memory_and_depth_settings(gen):
    import sambamba_b200 as sb
    p = gen["pairs"]
    kw = dict(num_filter=(1, 0x400), subsample=0.5, seed=4)
    want = vc.oracle_count(p, **kw)
    with sb.BDepth(p) as b:
        b.set_filter_query("mapping_quality > 30")
        b.set_regions([(0, 1000, 5000)])
        b.set_combined(True)
        b.stage()
        for _ in range(2):
            assert b.run_view_count(**kw) == want
            assert b.stats()["ms_inflate"] > 0
        assert b.run_view_count() == vc.oracle_count(p)
        rows = b.run_regions([(0, 1000, 5000)], [1])
    with sb.BDepth(p) as c:
        c.set_filter_query("mapping_quality > 30")
        c.set_combined(True)
        assert c.run_regions([(0, 1000, 5000)], [1]) == rows, "the depth settings stay set"
    img = np.fromfile(p, dtype=np.uint8)
    with sb.BDepth(memory=img) as b:
        assert b.run_view_count(**kw) == want


def test_several_inputs_are_refused(gen):
    import sambamba_b200 as sb
    with sb.BDepth(gen["plain"]) as b:
        b.add_input(gen["plain"])
        with pytest.raises(sb.BDepthError) as e:
            b.run_view_count()
        assert e.value.code == -7


_CHILD = """
import sys
sys.path.insert(0, sys.argv[1])
import sambamba_b200._lib as L
L.lib_path = lambda: sys.argv[2]
import sambamba_b200 as sb
try:
    with sb.BDepth(sys.argv[3]) as b:
        b.run_view_count(num_filter=(0, 4))
    print("ok")
except sb.BDepthError as e:
    print(e.code, e.msg)
"""


def test_malformed_input_in_its_own_process(tmp_path):
    import sambamba_b200._lib as L
    body = fc.bam_body(fc.HAND_REFS, fc.hand_records())
    cut = helpers.write_bgzf(str(tmp_path / "cut.bam"), body[:-5], len(fc.HAND_REFS))
    r = subprocess.run([sys.executable, "-c", _CHILD, helpers.ROOT, L.lib_path(), cut], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-400:]
    assert r.stdout.startswith("-2 ") and "not enough data" in r.stdout, r.stdout


def _rank_main(rank, world, path, uid, kw, q):
    try:
        sys.path.insert(0, helpers.ROOT)
        import sambamba_b200 as sb
        with sb.BDepth(path, device=rank if not EMULATE else 0) as b:
            b.set_shard(rank, world, uid)
            b.set_tuning(1 << 18, 2)
            q.put((rank, "ok", b.run_view_count(**kw)))
    except Exception as e:  # pragma: no cover
        q.put((rank, "err", repr(e)))


@pytest.mark.parametrize("world", [2, 3, 4])
def test_several_ranks_all_reduce(gen, world):
    import sambamba_b200 as sb
    if not EMULATE and sb.load_library().bdepth_device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    p = gen["pairs"]
    for kw in (dict(num_filter=(0x40, 0), subsample=0.5, seed=world), dict(bed=_bed_one_percent(p, world))):
        want = vc.oracle_count(p, **kw)
        uid = sb.nccl_unique_id()
        if EMULATE:
            import queue
            import threading
            q = queue.Queue()
            ts = [threading.Thread(target=_rank_main, args=(r, world, p, uid, kw, q)) for r in range(world)]
        else:
            ctx = mp.get_context("spawn")
            q = ctx.Queue()
            ts = [ctx.Process(target=_rank_main, args=(r, world, p, uid, kw, q)) for r in range(world)]
        for t in ts:
            t.start()
        res = sorted([q.get(timeout=1500) for _ in range(world)], key=lambda r: r[0])
        for t in ts:
            t.join(timeout=60)
        assert all(r[1] == "ok" and r[2] == want for r in res), (res, want)


def _cli_same(args, rc=0):
    r1 = helpers.run_cli(["view"] + args)
    r2 = vc.oracle_cli(args)
    assert r1[0] == r2[0] == rc and r1[1] == r2[1], (args, r1, r2)
    if rc:
        assert r1[2] == r2[2], (args, r1[2], r2[2])
    return r1[1]


def test_cli_is_the_oracle_cli(edge, gen, tmp_path):
    s, p = edge["sorted"], gen["plain"]
    bed = tmp_path / "t.bed"
    bed.write_text("c1\t500\t600\nnochr\t1\t5\nc1 200 300\nc1\t100\t200\n")
    gbed = tmp_path / "g.bed"
    gbed.write_text("".join("%s\t%d\t%d\n" % (("chrA", "chrB", "chrC")[r], a, b) for r, a, b in _bed_one_percent(p, 7)))
    assert _cli_same(["-c", s]) == b"11\n"
    _cli_same(["-c", "-L", str(bed), s])
    _cli_same(["-c", "-L", str(bed), edge["unsorted"]])
    _cli_same(["-c", "-L", str(gbed), p])
    _cli_same(["-c", s, "c1:101-200", "c1:151-300", "c1:101-200", "*"])
    _cli_same(["-c", p, "chrA:1,001-50,000", "chrB", "*", "chrA:20001-30000"])
    _cli_same(["-c", "--num-filter=/4", s])
    _cli_same(["-c", "--num-filter=65/1024", "-s", "0.25", "--subsampling-seed=99", p])
    _cli_same(["-c", "-L", str(bed), s, "c1"], rc=1)
    _cli_same(["-c", s, "c9:1-5"], rc=1)
    _cli_same(["-c", s, "c1:10-5"], rc=1)
    _cli_same(["-c", "-s", "-0.5", s], rc=1)
    _cli_same(["-c", "--num-filter=x", s], rc=1)


def test_cli_quirks_and_refusals(edge, tmp_path):
    s = edge["sorted"]
    o = tmp_path / "out.sam"
    o.write_text("old")
    assert helpers.run_cli(["view", "-c", "-o", str(o), s]) == (0, b"11\n", b"")
    assert o.read_bytes() == b"", "-o is opened w+ even with -c"
    assert helpers.run_cli(["view", "-c", "-H", s]) == (0, b"", b"")
    assert helpers.run_cli(["view", "-c", "-I", "-h", "-f", "bam", "-l", "3", "-p", "-t", "4", s]) == (0, b"11\n", b"")
    assert helpers.run_cli(["view", "-c", "-F", "mapping_quality >= 30 and not duplicate", s])[1] == b"10\n"
    assert helpers.run_cli(["view", "-c", "-s", "nan", s])[1] == b"11\n", "a NaN fraction means no subsampling"
    for args in (["view", s], ["view", "-h", s], ["view", "-f", "bam", s], ["view", "-c", "-v", s], ["view", "-c", "-S", s], ["view", "-c", "-T", "x.fa", s]):
        rc, out, err = helpers.run_cli(args)
        assert rc == 1 and out == b"" and err.startswith(b"sambamba-view: not supported"), args
    rc, out, err = helpers.run_cli(["view", "-c", "-F", "mapping_quality >>= 3", s])
    assert rc == 1 and out == b"" and err.startswith(b"sambamba-view: ")
    rc, out, err = helpers.run_cli(["view"])
    assert rc == 0 and out == b"" and err.startswith(b"Usage: sambamba-view")
    rc, out, err = helpers.run_cli(["view", "-c", "-x", s])
    assert (rc, out, err) == (1, b"", b"sambamba-view: Unrecognized option -x\n")
    rc, out, err = helpers.run_cli(["view", "-c", str(tmp_path / "missing.bam")])
    assert rc == 1 and err.startswith(b"sambamba-view: Cannot open file")


def test_full_size(tmp_path_factory):
    """The chr20 benchmark file (a small file of its shape under the emulation): whole file, filters, a 1 % -L query and positional regions."""
    if EMULATE:
        p = helpers.gen_bam(str(tmp_path_factory.mktemp("vcz") / "small.bam"), "-r", "chr20:300000", "-n", 60000, "-s", 20, "-t", 4)
    else:
        sys.path.insert(0, helpers.ROOT)
        import bench
        p = bench.ensure_workload(1, bench.READS_PER_UNIT)
    import sambamba_b200 as sb
    with sb.BDepth(p) as b:
        L = b.refs[0][1]
        bed = [(0, L // 2, L // 2 + L // 100)]
        for kw in (dict(), dict(num_filter=(0, 0x404), subsample=0.1, seed=1), dict(bed=bed), dict(regions=bed + bed, n_unmapped=1)):
            n = b.run_view_count(**kw)
            assert n == vc.oracle_count(p, **kw), kw
            if not kw:
                assert n == b.stats()["n_records"] == (60000 if EMULATE else 12888833)
