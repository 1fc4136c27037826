"""`sambamba view -f json` on the GPU (bdepth_run_view_json) against the CPU restatement of toJson (tools/view_count_oracle.c, pinned in
tests/test_oracle_view_json.py), case for case as tests/test_gpu_view_text.py checks the SAM lines.  Every case also checks that the number of
records is what bdepth_run_view_count counts with the same options; one more checks each parsed record against the SAM line of the same read."""
import glob
import hashlib
import json
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
import test_gpu_view_text as tvt
import view_json_common as vj
import view_text_common as vt

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
EMULATE = os.environ.get("BDEPTH_EMULATE") == "1"
GOLDEN = sorted(glob.glob(os.path.join(helpers.GOLDEN, "*.bam")))
bdepth = tvt.bdepth


def check(b, path, **kw):
    """b.run_view_json(**kw) equals the oracle's text, and has as many lines as b.run_view_count counts; returns the text."""
    got = b.run_view_json(**kw)
    want = vj.oracle_json(path, **kw)
    if got != want:
        g, w = got.split(b"\n"), want.split(b"\n")
        i = next((i for i in range(min(len(g), len(w))) if g[i] != w[i]), min(len(g), len(w)))
        pytest.fail("%s %r: %d vs %d bytes, line %d differs:\n%r\n%r" % (os.path.basename(path), kw, len(got), len(want), i, g[i][:300] if i < len(g) else None, w[i][:300] if i < len(w) else None))
    assert got.count(b"\n") == b.run_view_count(**vt.count_kw(kw)), kw
    return got


@pytest.fixture(scope="module")
def gen(tmp_path_factory):
    d = tmp_path_factory.mktemp("vj")
    n = 6000 if EMULATE else 200000
    return {"plain": helpers.gen_bam(str(d / "g.bam"), "-r", "chrA:%d" % (n * 10), "-r", "chrB:700", "-r", "chrC:%d" % (n * 5), "-n", n, "-s", 41, "-t", 8),
            "pairs": helpers.gen_bam(str(d / "p.bam"), "-r", "chrA:%d" % (n * 10), "-n", n, "-s", 42, "-t", 8, "--pairs", 5), "n": n, "dir": d}


@pytest.fixture(scope="module")
def edge(tmp_path_factory):
    d = tmp_path_factory.mktemp("vje")
    p, text = vj.write_edge_bam(str(d / "e.bam"))
    return {"path": p, "text": text, "dir": d}


@pytest.mark.parametrize("name", [os.path.basename(p) for p in GOLDEN])
def test_golden(name):
    p = os.path.join(helpers.GOLDEN, name)
    with bdepth(p) as b:
        for kw in (dict(), dict(num_filter=(0, 0x404)), dict(subsample=0.3, seed=77)):
            check(b, p, **kw)
        assert b.stats()["gpu_launches"] > 0


def test_golden_sam_round_trip(tmp_path):
    p, _ = vt.sam_to_bam(os.path.join(helpers.GOLDEN, "ex1_header.sam.gz"), str(tmp_path / "ex1.bam"))
    with bdepth(p) as b:
        got = check(b, p)
        assert got.count(b"\n") == 3270
        check(b, p, regions=[(0, 100, 400), "*", (1, 0, 1584), (0, 100, 400)])


def test_json_agrees_with_sam_and_count(gen):
    """On the same file and options: as many records as run_view_count counts, and each parsed record has the SAM line's fields."""
    p = gen["pairs"]
    with bdepth(p) as b:
        for kw in (dict(), dict(num_filter=(0x40, 0), subsample=0.5, seed=3)):
            js, sam = b.run_view_json(**kw).split(b"\n")[:-1], b.run_view_text(**kw).split(b"\n")[:-1]
            assert len(js) == len(sam) == b.run_view_count(**kw) > 0
            for j, s in zip(js, sam):
                d, f = json.loads(j), s.decode().split("\t")
                assert [d["qname"], str(d["flag"]), d["rname"], str(d["pos"]), str(d["mapq"]), d["cigar"], d["rnext"], str(d["pnext"]), str(d["tlen"]), d["seq"]] == f[:10]
                assert f[10] == ("*" if not d["qual"] or d["qual"][0] == 255 else "".join(chr(q + 33) for q in d["qual"]))
                tags = [t.split(":", 2) for t in f[11:]]
                assert [k for k, _, _ in tags] == list(d["tags"])
                for k, t, v in tags:
                    x = d["tags"][k]
                    if t == "i":
                        assert int(v) == x
                    elif t == "f":
                        assert float(v) == pytest.approx(x, rel=1e-5)
                    elif t == "B":
                        assert [float(e) for e in v.split(",")[1:]] == pytest.approx([float(e) for e in x], rel=1e-5)
                    else:
                        assert v == x


EDGE_CASES = tvt.EDGE_CASES


@pytest.mark.parametrize("case", range(len(EDGE_CASES)))
def test_edge_file(edge, case):
    with bdepth(edge["path"]) as b:
        got = check(b, edge["path"], **EDGE_CASES[case])
        if not case:
            assert got == edge["text"]


@pytest.mark.parametrize("tuning", [(1 << 16, 1), (1 << 17, 3), (1 << 20, 7)])
def test_tiny_batches_and_pieces(gen, tuning):
    """Pieces of at most one batch of text: records straddle sub-batches and text slots."""
    p = gen["pairs"]
    with bdepth(p, tuning) as b:
        chunks = []
        n = b.run_view_json(sink=chunks.append)
        want = vj.oracle_json(p)
        assert b"".join(chunks) == want and n == len(want)
        assert len(chunks) > 2 and all(c.endswith(b"\n") for c in chunks), "whole lines in every piece"
        assert max(len(c) for c in chunks) <= tuning[0] + max(len(x) + 1 for x in want.split(b"\n"))
        for kw in (dict(num_filter=(0x41, 0x100)), dict(subsample=0.1, seed=2)):
            check(b, p, **kw)


def test_bed_sorted_sparse_and_shuffled_unindexed(gen, tmp_path):
    p = gen["plain"]
    bed = tvt._bed_one_percent(p, 5) + [(2, 10, 900)]
    for tuning in (None, (1 << 17, 2)):
        with bdepth(p, tuning) as b:
            assert check(b, p, bed=bed)
            assert b.stats()["file_bytes"] < os.path.getsize(p) // 2, "only the regions' BAI chunks are staged"
    u = helpers.oracle_inflate(p)
    first, refs = helpers.header_first_record_offset(u)
    raw = u.tobytes()
    recs = [raw[r[0]:r[0] + 4 + struct.unpack_from("<i", raw, r[0])[0]] for r in helpers.parse_records(u, first)]
    random.Random(4).shuffle(recs)
    q = helpers.write_bgzf(str(tmp_path / "raw.bam"), fc.bam_body(refs, recs), len(refs))
    os.remove(q + ".bai")
    with bdepth(q) as b:
        assert not b.coordinate_sorted and not b.has_index
        check(b, q, bed=bed)
        check(b, q, bed=bed, num_filter=(0, 0x10), subsample=0.5, seed=8)
        check(b, q)


def test_positional_regions_repeats_overlaps_and_star(gen):
    p = gen["plain"]
    bed = tvt._bed_one_percent(p, 6)
    regs = bed[:4] + ["*"] + bed[:2] + [(1, 0, 700), (0, bed[0][1], bed[0][2] + 5000), (2, 5, 6)]
    with bdepth(p) as b:
        assert check(b, p, regions=regs)
        check(b, p, regions=regs[:3] + ["*"], num_filter=(0, 4), subsample=0.4, seed=3)
    with bdepth(p, (1 << 17, 2)) as b:
        check(b, p, regions=regs)


def test_filter_queries(tmp_path):
    """A third of test_emul_filter.QUERIES, alone and with a region and the other selections."""
    p = tef.make_bam(str(tmp_path / "f.bam"), seed=5, n=1500 if EMULATE else 3000, empty_seq=False)
    u = helpers.oracle_inflate(p)
    _, recs = tef.parse_all(u)
    with bdepth(p) as b:
        for k, (q, fn) in enumerate(tef.QUERIES):
            if k % 3 != 1:
                continue
            keep = [bool(fn(r)) for r in recs]
            sub = helpers.subset_bam(p, str(tmp_path / f"sub{k}.bam"), keep)
            assert b.run_view_json(query=q) == vj.oracle_json(sub), q
            kw = dict(bed=[(0, 100, 3000), (1, 50, 400)], num_filter=(0, 0x10), subsample=0.6, seed=k)
            got = b.run_view_json(query=q, **kw)
            assert got == vj.oracle_json(sub, **kw) and got.count(b"\n") == b.run_view_count(query=q, **kw), q
            rg = [(0, 100, 3000), "*", (0, 2000, 2500)]
            assert b.run_view_json(query=q, regions=rg) == vj.oracle_json(sub, regions=rg), q


def test_staged_memory_and_depth_settings(gen):
    import sambamba_b200 as sb
    p = gen["pairs"]
    kw = dict(num_filter=(1, 0x400), subsample=0.5, seed=4)
    want = vj.oracle_json(p, **kw)
    with sb.BDepth(p) as b:
        b.set_filter_query("mapping_quality > 30")
        b.set_regions([(0, 1000, 5000)])
        b.stage()
        for _ in range(2):
            assert b.run_view_json(**kw) == want
            st = b.stats()
            assert st["ms_inflate"] > 0 and st["ms_reduce"] > 0 and st["ms_d2h"] > 0
        assert b.run_view_json() == vj.oracle_json(p)
        assert b.run_view_text() == vt.oracle_text(p), "the SAM lines after a JSON run on the same handle"
    img = np.fromfile(p, dtype=np.uint8)
    with sb.BDepth(memory=img) as b:
        assert b.run_view_json(**kw) == want


def test_refusals(gen, edge):
    import sambamba_b200 as sb
    with sb.BDepth(gen["plain"]) as b:
        b.add_input(gen["plain"])
        with pytest.raises(sb.BDepthError) as e:
            b.run_view_json()
        assert e.value.code == -7
    with bdepth(edge["path"]) as b:
        with pytest.raises(sb.BDepthError, match="start must be less than end"):
            b.run_view_json(regions=[(0, 1, 5), (0, 7, 7)])
        seen = []

        class Enough(Exception):
            pass

        def stop(chunk):
            seen.append(chunk)
            raise Enough()
        with pytest.raises(sb.BDepthError) as e:
            b.run_view_json(sink=stop)
        assert e.value.code == -8 and isinstance(e.value.__cause__, Enough) and len(seen) == 1
        assert b.run_view_json() == edge["text"], "the handle is usable after a stopped run"


_CHILD = """
import sys
sys.path.insert(0, sys.argv[1])
import sambamba_b200._lib as L
L.lib_path = lambda: sys.argv[2]
import sambamba_b200 as sb
try:
    with sb.BDepth(sys.argv[3]) as b:
        b.run_view_json()
    print("ok")
except sb.BDepthError as e:
    print(e.code, e.msg)
"""


@pytest.mark.parametrize("what", [w for w, _ in vt.malformed_records()])
def test_malformed_records_in_their_own_process(tmp_path, what):
    import sambamba_b200._lib as L
    recs, _ = vt.edge_records()
    p = vt.write_records(str(tmp_path / "m.bam"), vt.EDGE_REFS, [recs[0], dict(vt.malformed_records())[what]], index=False)
    r = subprocess.run([sys.executable, "-c", _CHILD, helpers.ROOT, L.lib_path(), p], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-400:]
    assert r.stdout.startswith("-2 "), r.stdout


def _rank_main(rank, world, path, uid, kw, q):
    try:
        sys.path.insert(0, helpers.ROOT)
        import sambamba_b200 as sb
        with sb.BDepth(path, device=rank if not EMULATE else 0) as b:
            b.set_shard(rank, world, uid)
            b.set_tuning(1 << 18, 2)
            q.put((rank, "ok", b.run_view_json(**kw)))
    except Exception as e:  # pragma: no cover
        q.put((rank, "err", repr(e)))


@pytest.mark.parametrize("world", [2, 3, 4])
def test_several_ranks_concatenate(gen, world):
    """The ranks' texts, joined in rank order, are the single-GPU text; positional regions are refused on several ranks."""
    import queue
    import threading
    import sambamba_b200 as sb
    if not EMULATE and sb.load_library().bdepth_device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    p = gen["pairs"]
    for kw in (dict(num_filter=(0x40, 0), subsample=0.5, seed=world), dict(bed=tvt._bed_one_percent(p, world)), dict(regions=[(0, 0, 1000)])):
        uid, ctx = sb.nccl_unique_id(), mp.get_context("spawn")
        q = queue.Queue() if EMULATE else ctx.Queue()
        ts = [(threading.Thread if EMULATE else ctx.Process)(target=_rank_main, args=(r, world, p, uid, kw, q)) for r in range(world)]
        for t in ts:
            t.start()
        res = sorted([q.get(timeout=1500) for _ in range(world)], key=lambda r: r[0])
        for t in ts:
            t.join(timeout=60)
        if "regions" in kw:
            assert all(r[1] == "err" and "positional regions on several ranks" in r[2] for r in res), res
            continue
        assert all(r[1] == "ok" for r in res) and b"".join(r[2] for r in res) == vj.oracle_json(p, **kw), res
        assert "bed" in kw or sum(1 for r in res if r[2]) >= 2, "the records are shared out"


def test_full_size(tmp_path_factory):
    """The chr20 benchmark file (a small file of its shape under the emulation): the whole file by SHA-256, a 1 % -L query and regions."""
    if EMULATE:
        p = helpers.gen_bam(str(tmp_path_factory.mktemp("vjz") / "small.bam"), "-r", "chr20:300000", "-n", 20000, "-s", 20, "-t", 4)
    else:
        sys.path.insert(0, helpers.ROOT)
        import bench
        p = bench.ensure_workload(1, bench.READS_PER_UNIT)
    want_sha, want_len = vj.oracle_sha256(p)
    with bdepth(p) as b:
        h, lines = hashlib.sha256(), [0]

        def sink(c):
            h.update(c)
            lines[0] += c.count(b"\n")
        n = b.run_view_json(sink=sink)
        assert n == want_len and h.hexdigest() == want_sha
        assert lines[0] == (20000 if EMULATE else 12888833)
        L = b.refs[0][1]
        bed = [(0, L // 2, L // 2 + L // 100)]
        check(b, p, bed=bed)
        check(b, p, regions=bed + ["*"] + bed)
