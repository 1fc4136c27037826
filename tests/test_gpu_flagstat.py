"""`sambamba flagstat` on the GPU (bdepth_run_flagstat, the CLI's `flagstat` subcommand) against the CPU restatement of
computeFlagStatistics (tools/flagstat_oracle.c, pinned in tests/test_oracle_flagstat.py)."""
import glob
import multiprocessing as mp
import os
import random
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest

import flagstat_common as fc
import helpers

pytestmark = pytest.mark.gpu
EMULATE = os.environ.get("BDEPTH_EMULATE") == "1"
GOLDEN = sorted(glob.glob(os.path.join(helpers.GOLDEN, "*.bam")))


def gpu_flagstat(path, tuning=None, **kw):
    import sambamba_b200 as sb
    with sb.BDepth(path, **kw) as b:
        if tuning:
            b.set_tuning(*tuning)
        got = b.run_flagstat()
        return got, b.stats()


@pytest.fixture(scope="module")
def gen(tmp_path_factory):
    d = tmp_path_factory.mktemp("fs")
    n = 20000 if EMULATE else 200000
    return {"plain": helpers.gen_bam(str(d / "g.bam"), "-r", "chrA:%d" % (n * 10), "-r", "chrB:700", "-r", "chrC:%d" % (n * 5), "-n", n, "-s", 21, "-t", 8),
            "pairs": helpers.gen_bam(str(d / "p.bam"), "-r", "chrA:%d" % (n * 10), "-n", n, "-s", 22, "-t", 8, "--pairs", 5)}


@pytest.mark.parametrize("name", [os.path.basename(p) for p in GOLDEN])
def test_golden(name):
    p = os.path.join(helpers.GOLDEN, name)
    got, st = gpu_flagstat(p)
    assert got == fc.oracle_flagstat(p)
    assert got["total"][0] + got["total"][1] == st["n_records"] and st["gpu_launches"] > 0


@pytest.mark.parametrize("block", [0xFF00, 150])
def test_hand_made(tmp_path, block):
    p = fc.write_hand_bam(str(tmp_path / "h.bam"), block=block)
    got, _ = gpu_flagstat(p)
    assert got == fc.oracle_flagstat(p) and all(a > 0 and b > 0 for a, b in got.values())


@pytest.mark.parametrize("kind", ["plain", "pairs"])
@pytest.mark.parametrize("tuning", [None, (1 << 16, 1), (1 << 17, 3), (1 << 20, 7)])
def test_generated_across_batches(gen, kind, tuning):
    """Tiny batches and sub-batches: records straddle BGZF members, H2D chunks (sub-batches) and batches (carried tail records)."""
    p = gen[kind]
    got, st = gpu_flagstat(p, tuning)
    assert got == fc.oracle_flagstat(p)
    assert got["total"][0] + got["total"][1] == st["n_records"]
    if tuning:
        assert st["n_batches"] > 2


def test_shuffled_unindexed_unsorted(tmp_path, gen):
    """Raw aligner output: records in no order, no SO:coordinate, no .bai."""
    import sambamba_b200 as sb
    src = gen["plain"]
    u = helpers.oracle_inflate(src)
    first, refs = helpers.header_first_record_offset(u)
    b = u.tobytes()
    recs, o = [], first
    while o + 4 <= len(b):
        bs, = struct.unpack_from("<i", b, o)
        recs.append(b[o:o + 4 + bs])
        o += 4 + bs
    random.Random(4).shuffle(recs)
    hdr = fc.bam_body([(n, l) for n, l in refs], [])          # a header without SO:coordinate, the same references
    p = helpers.write_bgzf(str(tmp_path / "raw.bam"), hdr + b"".join(recs), len(refs))
    os.remove(p + ".bai")
    with sb.BDepth(p) as h:
        assert not h.coordinate_sorted and not h.has_index
        got = h.run_flagstat()
        h.set_tuning(1 << 17, 2)
        again = h.run_flagstat()
    assert got == again == fc.oracle_flagstat(p) == fc.oracle_flagstat(src)


def test_staged_twice_and_memory(gen):
    import sambamba_b200 as sb
    p = gen["pairs"]
    want = fc.oracle_flagstat(p)
    with sb.BDepth(p) as b:
        b.stage()
        for _ in range(2):
            assert b.run_flagstat() == want
            st = b.stats()
            assert want["total"][0] + want["total"][1] == st["n_records"] and st["ms_inflate"] > 0 and st["ms_reduce"] >= 0
    img = np.fromfile(p, dtype=np.uint8)
    with sb.BDepth(memory=img) as b:
        assert b.run_flagstat() == want


def test_depth_settings_do_not_apply_and_stay_set(gen):
    """-F, regions, -m, -q, --combined change nothing of flagstat, and a depth run afterwards still uses them."""
    import sambamba_b200 as sb
    p = gen["plain"]
    want = fc.oracle_flagstat(p)
    with sb.BDepth(p) as b:
        b.set_filter_query("mapping_quality > 30 and not duplicate")
        b.set_regions([(0, 1000, 5000)])
        b.set_fix_mates(True)
        b.set_min_baseq(20)
        b.set_combined(True)
        assert b.run_flagstat() == want
        rows = b.run_regions([(0, 1000, 5000)], [1])
    with sb.BDepth(p) as c:
        c.set_filter_query("mapping_quality > 30 and not duplicate")
        c.set_fix_mates(True)
        c.set_min_baseq(20)
        c.set_combined(True)
        assert c.run_regions([(0, 1000, 5000)], [1]) == rows


def test_several_inputs_are_refused(gen):
    import sambamba_b200 as sb
    with sb.BDepth(gen["plain"]) as b:
        b.add_input(gen["plain"])
        with pytest.raises(sb.BDepthError) as e:
            b.run_flagstat()
        assert e.value.code == -7


_CHILD = """
import sys
sys.path.insert(0, sys.argv[1])
import sambamba_b200._lib as L
L.lib_path = lambda: sys.argv[2]
import sambamba_b200 as sb
try:
    with sb.BDepth(sys.argv[3]) as b:
        b.run_flagstat()
    print("ok")
except sb.BDepthError as e:
    print(e.code, e.msg)
"""


def _in_own_process(path):
    import sambamba_b200._lib as L
    r = subprocess.run([sys.executable, "-c", _CHILD, helpers.ROOT, L.lib_path(), path], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-400:]
    return r.stdout.strip()


def test_malformed_input_each_in_its_own_process(tmp_path):
    body = fc.bam_body(fc.HAND_REFS, fc.hand_records())
    cut = helpers.write_bgzf(str(tmp_path / "cut.bam"), body[:-5], len(fc.HAND_REFS))
    out = _in_own_process(cut)
    assert out.startswith("-2 ") and "not enough data" in out, out
    src = helpers.gen_bam(str(tmp_path / "src.bam"), "-r", "chrA:100000", "-n", 8000, "-s", 3, "-t", 2)
    raw = open(src, "rb").read()
    bad = tmp_path / "deflate.bam"
    for pos in range(len(raw) // 2, len(raw) // 2 + 4000, 97):          # somewhere in there a flip breaks a Huffman stream
        data = bytearray(raw)
        data[pos] ^= 0x55
        bad.write_bytes(bytes(data))
        try:
            fc.oracle_flagstat(str(bad))
        except RuntimeError as e:
            if "DEFLATE" in str(e):
                break
    else:
        pytest.fail("no flip broke a DEFLATE stream")
    out = _in_own_process(str(bad))
    assert out.startswith("-2 ") and "DEFLATE" in out, out


def _rank_main(rank, world, path, uid, tuning, q):
    try:
        sys.path.insert(0, helpers.ROOT)
        import sambamba_b200 as sb
        with sb.BDepth(path, device=rank if not EMULATE else 0) as b:
            b.set_shard(rank, world, uid)
            if tuning:
                b.set_tuning(*tuning)
            q.put((rank, "ok", b.run_flagstat(), b.stats()["n_records"]))
    except Exception as e:  # pragma: no cover
        q.put((rank, "err", repr(e), 0))


def _n_gpus():
    import sambamba_b200 as sb
    return sb.load_library().bdepth_device_count()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_several_ranks_all_reduce(gen, world):
    """Each rank counts its shard, one all-reduce sums them: every rank holds the whole file's counts.  Under the emulation the ranks
    are threads over the NCCL stand-in; on hardware, processes (one GPU each)."""
    import sambamba_b200 as sb
    if not EMULATE and _n_gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    p = gen["pairs"]
    want = fc.oracle_flagstat(p)
    uid = sb.nccl_unique_id()
    tuning = (1 << 18, 2)
    if EMULATE:
        import queue
        import threading
        q = queue.Queue()
        ts = [threading.Thread(target=_rank_main, args=(r, world, p, uid, tuning, q)) for r in range(world)]
    else:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        ts = [ctx.Process(target=_rank_main, args=(r, world, p, uid, tuning, q)) for r in range(world)]
    for t in ts:
        t.start()
    res = sorted([q.get(timeout=1500) for _ in range(world)], key=lambda r: r[0])
    for t in ts:
        t.join(timeout=60)
    assert all(r[1] == "ok" for r in res), res
    assert all(r[2] == want for r in res)
    assert sum(r[3] for r in res) == want["total"][0] + want["total"][1], "every record is counted by exactly one rank"


def test_shards_without_nccl_partition_the_file(gen):
    """A NULL NCCL id with world > 1: each rank returns its shard's own counts; together they are the file's."""
    import sambamba_b200 as sb
    p = gen["plain"]
    want = fc.oracle_flagstat(p)
    world = 3
    total = {k: [0, 0] for k in fc.FIELDS}
    for r in range(world):
        with sb.BDepth(p) as b:
            b.set_shard(r, world, None)
            b.set_tuning(1 << 18, 2)
            got = b.run_flagstat()
        assert got != want
        for k, (a, c) in got.items():
            total[k][0] += a
            total[k][1] += c
    assert {k: tuple(v) for k, v in total.items()} == want


def _cli_same(args):
    rc1, out1, err1 = helpers.run_cli(["flagstat"] + args)
    rc2, out2, err2 = fc.oracle_cli(args)
    assert rc1 == rc2 == 0 and out1 == out2 and len(out1.splitlines()) == 13, (args, err1[:300], out1[:300], out2[:300])


def test_cli_is_the_oracle_cli(tmp_path, gen):
    hand = fc.write_hand_bam(str(tmp_path / "h.bam"))
    empty = helpers.write_bgzf(str(tmp_path / "e.bam"), fc.bam_body(fc.HAND_REFS, []), len(fc.HAND_REFS))
    share = fc.write_mapped_share(str(tmp_path / "s.bam"), 23, 160)        # float arithmetic prints 14.38, double 14.37
    for p in GOLDEN + [hand, empty, share, gen["pairs"]]:
        _cli_same([p])
        _cli_same(["-b", p])
    assert b"23 + 0 mapped (14.38%:N/A)" in helpers.run_cli(["flagstat", share])[1]
    rc, out, err = helpers.run_cli(["flagstat", "-t", "4", "-p", "--tabular", hand])
    assert rc == 0 and out == fc.oracle_cli(["-b", hand])[1]


def test_cli_usage_and_errors(tmp_path):
    rc, out, err = helpers.run_cli(["flagstat"])
    assert rc == 1 and out == b"" and err.startswith(b"Usage: sambamba-flagstat [options] <input.bam>\n")
    rc, out, err = helpers.run_cli(["flagstat", "-x", "a.bam"])
    assert rc == 1 and out == b"" and err == b"Unrecognized option -x\n"
    rc, out, err = helpers.run_cli(["flagstat", "-t", "many", "a.bam"])
    assert rc == 1 and out == b"" and b"when converting from type string to type ulong" in err
    rc, out, err = helpers.run_cli(["flagstat", str(tmp_path / "missing.bam")])
    assert rc == 1 and out == b"" and err.startswith(b"Cannot open file") and b"sambamba" not in err
    body = fc.bam_body(fc.HAND_REFS, fc.hand_records())
    cut = helpers.write_bgzf(str(tmp_path / "cut.bam"), body[:-5], len(fc.HAND_REFS))
    rc, out, err = helpers.run_cli(["flagstat", cut])
    assert rc == 1 and out == b"" and b"not enough data in stream" in err and not err.startswith(b"sambamba")


@pytest.mark.timeout(1500)
def test_full_size(tmp_path_factory):
    """The chr20 benchmark file (2.26 GB BAM, 12.9 M reads; a small file of its shape under the emulation): library and CLI equal the
    oracle, streamed and staged."""
    if EMULATE:
        p = helpers.gen_bam(str(tmp_path_factory.mktemp("fsz") / "small.bam"), "-r", "chr20:300000", "-n", 60000, "-s", 20, "-t", 4)
    else:
        sys.path.insert(0, helpers.ROOT)
        import bench
        p = bench.ensure_workload(1, bench.READS_PER_UNIT)
    import sambamba_b200 as sb
    want = fc.oracle_flagstat(p)
    with sb.BDepth(p) as b:
        assert b.run_flagstat() == want
        b.stage()
        assert b.run_flagstat() == want
        assert b.stats()["n_records"] == want["total"][0] + want["total"][1] == (60000 if EMULATE else 12888833)
    for args in ([p], ["-b", p]):
        _cli_same(args)
