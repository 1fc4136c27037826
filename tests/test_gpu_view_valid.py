"""`view -v` on the GPU (bdepth_view_opts.valid for bdepth_run_view_count, _text and _json) against the CPU restatement of isValid in
view_main's filter chain (tools/view_count_oracle.c, pinned in tests/test_oracle_view_valid.py): the count, the SAM lines and the JSON records
of every case, and the refusals where the reference's validator reaches a record whose tags it cannot walk."""
import glob
import hashlib
import multiprocessing as mp
import os
import random
import struct
import sys

import numpy as np
import pytest

import flagstat_common as fc
import helpers
import test_emul_filter as tef
import view_count_common as vc
import view_json_common as vj
import view_text_common as vt
import view_valid_common as vv

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
EMULATE = os.environ.get("BDEPTH_EMULATE") == "1"
GOLDEN = sorted(glob.glob(os.path.join(helpers.GOLDEN, "*.bam")))


def check(b, path, **kw):
    """The three entry points with valid=True equal the oracle with -v; returns the count."""
    ckw = vt.count_kw(kw)
    with vv.valid_oracle():
        wc, wt, wj = vc.oracle_count(path, **ckw), vt.oracle_text(path, **kw), vj.oracle_json(path, **kw)
    assert b.run_view_count(valid=True, **ckw) == wc, kw
    assert b.run_view_text(valid=True, **kw) == wt, kw
    assert b.run_view_json(valid=True, **kw) == wj, kw
    assert wt.count(b"\n") == wc == wj.count(b"\n")
    return wc


def refused(b, path, **kw):
    """Every entry point refuses with BDEPTH_ERR_FORMAT, as the oracle does."""
    import sambamba_b200 as sb
    with vv.valid_oracle():
        with pytest.raises(RuntimeError):
            vc.oracle_count(path, **vt.count_kw(kw))
    for run in (lambda: b.run_view_count(valid=True, **vt.count_kw(kw)), lambda: b.run_view_text(valid=True, **kw), lambda: b.run_view_json(valid=True, **kw)):
        with pytest.raises(sb.BDepthError) as e:
            run()
        assert e.value.code == -2, kw


def bdepth(path, tuning=None, **kw):
    import sambamba_b200 as sb
    b = sb.BDepth(path, **kw)
    if tuning:
        b.set_tuning(*tuning)
    return b


@pytest.mark.parametrize("name", [os.path.basename(p) for p in GOLDEN])
def test_golden(name):
    p = os.path.join(helpers.GOLDEN, name)
    with bdepth(p) as b:
        for kw in (dict(), dict(num_filter=(0, 0x404)), dict(subsample=0.3, seed=77)):
            check(b, p, **kw)


def test_golden_sam_with_tags(tmp_path):
    """ex1_header.sam's reads with their integer tags (NM, MF, Aq, UQ, H0, H1...)."""
    p, _ = vt.sam_to_bam(os.path.join(helpers.GOLDEN, "ex1_header.sam.gz"), str(tmp_path / "ex1.bam"))
    with bdepth(p) as b:
        n = check(b, p)
        assert 0 < n <= b.run_view_count()
        check(b, p, regions=[(0, 100, 400), "*", (1, 0, 1584), (0, 100, 400)])
        check(b, p, bed=[(0, 100, 400), (1, 10, 20)], num_filter=(0, 0x10))


def kinds_file(path, sorted_file=True):
    """A valid read, then an invalid read of each kind, each at its own position of reference 0, and unplaced reads at the end."""
    recs = [vv.rec(name="ok0", pos=0)]
    for i, (_, r) in enumerate(vv.invalid_kinds()):
        body = bytearray(r[4:])
        body[4:8] = struct.pack("<i", 20 + 10 * i)
        recs.append(r[:4] + bytes(body))
        recs.append(vv.rec(name="ok%d" % (i + 1), pos=25 + 10 * i, flag=0x10 if i % 2 else 0))
    recs += [vv.rec(name="un1", pos=-1, ref=-1, flag=4, cigar=()), vv.rec(b"XXZ", name="un@", pos=-1, ref=-1, flag=4, cigar=())]
    if sorted_file:
        return vt.write_records(path, vt.EDGE_REFS, recs), len(recs)
    random.Random(3).shuffle(recs)
    return helpers.write_bgzf(path, fc.bam_body(vt.EDGE_REFS, recs), len(vt.EDGE_REFS)), len(recs)


def test_an_invalid_read_of_each_kind(tmp_path):
    p, n = kinds_file(str(tmp_path / "k.bam"))
    with bdepth(p) as b:
        got = check(b, p)
        assert got == 2 + len(vv.invalid_kinds()) and b.run_view_count() == n
        check(b, p, num_filter=(0, 0x10))
        check(b, p, subsample=0.5, seed=5)
        check(b, p, bed=[(0, 30, 200), (0, 400, 900)])
        check(b, p, regions=[(0, 30, 200), "*", (0, 30, 200), (0, 0, 1000)])
    q, _ = kinds_file(str(tmp_path / "u.bam"), sorted_file=False)
    with bdepth(q) as b:
        check(b, q)
        check(b, q, bed=[(0, 30, 200)])


def generated(path, src, every=7, broken_at=None):
    """src's reads, every `every`-th made invalid (in turn a quality of 94 and a name that begins with '@'), and the read at broken_at given
    an unknown tag type instead (it stays valid up to its tags, so the validator reaches them)."""
    u = helpers.oracle_inflate(src)
    first, refs = helpers.header_first_record_offset(u)
    raw = u.tobytes()
    recs = []
    for k, r in enumerate(helpers.parse_records(u, first)):
        rec = bytearray(raw[r[0]:r[0] + 4 + struct.unpack_from("<i", raw, r[0])[0]])
        if k % every == every - 1 and k != broken_at:
            l_name, n_cig = rec[12], struct.unpack_from("<H", rec, 16)[0]
            l_seq = struct.unpack_from("<i", rec, 20)[0]
            kind = (k // every) % 2
            if kind == 0 and l_seq:
                rec[36 + l_name + 4 * n_cig + (l_seq + 1) // 2] = 94
            else:
                rec[36] = ord("@")
        if k == broken_at:
            rec += b"XXq\x01"
            rec[0:4] = struct.pack("<i", len(rec) - 4)
        recs.append(bytes(rec))
    return vt.write_records(path, refs, recs)


@pytest.fixture(scope="module")
def gen(tmp_path_factory):
    d = tmp_path_factory.mktemp("vv")
    n = 6000 if EMULATE else 200000
    src = helpers.gen_bam(str(d / "g.bam"), "-r", "chrA:%d" % (n * 10), "-r", "chrB:700", "-n", n, "-s", 43, "-t", 8, "--pairs", 5)
    return {"src": src, "inv": generated(str(d / "inv.bam"), src), "brk": generated(str(d / "brk.bam"), src, broken_at=n // 2 + 1), "n": n, "dir": d}


@pytest.mark.parametrize("tuning", [None, (1 << 16, 1), (1 << 17, 3)])
def test_generated_tiny_batches(gen, tuning):
    """Invalid reads in every sub-batch and at its edges; a refused one in the middle of the file."""
    p = gen["inv"]
    with bdepth(p, tuning) as b:
        n = check(b, p)
        assert 0 < n < b.run_view_count()
        check(b, p, num_filter=(0x41, 0x100), subsample=0.4, seed=6)
    with bdepth(gen["brk"], tuning) as b:
        refused(b, gen["brk"])


def test_selection_combined(gen, tmp_path):
    import test_gpu_view_count as tvc
    p = gen["inv"]
    bed = tvc._bed_one_percent(p, 5) + [(1, 10, 600)]
    with bdepth(p) as b:
        check(b, p, bed=bed)
        check(b, p, bed=bed, num_filter=(0, 0x10), subsample=0.5, seed=8)
        check(b, p, regions=bed[:3] + ["*"] + bed[:2] + [(1, 0, 700)])
        assert b.stats()["file_bytes"] > 0
    u = helpers.oracle_inflate(p)
    first, refs = helpers.header_first_record_offset(u)
    raw = u.tobytes()
    recs = [raw[r[0]:r[0] + 4 + struct.unpack_from("<i", raw, r[0])[0]] for r in helpers.parse_records(u, first)]
    random.Random(4).shuffle(recs)
    q = helpers.write_bgzf(str(tmp_path / "raw.bam"), fc.bam_body(refs, recs), len(refs))
    os.remove(q + ".bai")
    with bdepth(q) as b:
        check(b, q, bed=bed)
        check(b, q)


def test_filter_queries_through_a_reduced_file(tmp_path):
    """-F after the validator: a Python statement of each query reduces the file, and the oracle checks the reduced file with -v."""
    p = tef.make_bam(str(tmp_path / "f.bam"), seed=6, n=1000 if EMULATE else 3000, empty_seq=False)
    u = helpers.oracle_inflate(p)
    _, recs = tef.parse_all(u)
    with bdepth(p) as b:
        for k, (q, fn) in enumerate(tef.QUERIES):
            if k % 5 != 1:
                continue
            sub = helpers.subset_bam(p, str(tmp_path / f"sub{k}.bam"), [bool(fn(r)) for r in recs])
            with vv.valid_oracle():
                want = vt.oracle_text(sub)
            assert b.run_view_text(query=q, valid=True) == want, q
            assert b.run_view_count(query=q, valid=True) == want.count(b"\n"), q


def refusal_file(path, name="brk", sorted_file=True):
    recs = [vv.rec(name="g%d" % i, pos=10 + i) for i in range(5)] + [vv.rec(b"XXq\x01", name=name, pos=500, flag=0x10)] + [vv.rec(name="h", pos=600)]
    if sorted_file:
        return vt.write_records(path, vt.EDGE_REFS, recs)
    return helpers.write_bgzf(path, fc.bam_body(vt.EDGE_REFS, recs[::-1]), len(vt.EDGE_REFS))


def test_refusal_scope(tmp_path):
    p = refusal_file(str(tmp_path / "r.bam"))
    h = vc.fnv1a(b"brk", 0) & 0xFFFFFFFF
    with bdepth(p) as b:
        refused(b, p)                                                       # the validator reaches the broken tags
        refused(b, p, num_filter=(0, 0x10))                                 # --num-filter comes after it
        refused(b, p, regions=[(0, 400, 550)])
        check(b, p, subsample=h / 4294967296.0)                             # -s comes before it: "brk" is not validated
        check(b, p, bed=[(0, 0, 100)])                                      # sorted: outside the regions, though inside a staged chunk
        check(b, p, regions=[(0, 0, 100), (0, 550, 700)])
        assert b.run_view_count() == 7, "without -v the count refuses nothing"
    q = refusal_file(str(tmp_path / "n.bam"), name="a@")
    with bdepth(q) as b:
        assert check(b, q) == 6                                             # a bad name ends the read before its tags
    s = refusal_file(str(tmp_path / "s.bam"), sorted_file=False)
    with bdepth(s) as b:
        refused(b, s, bed=[(0, 0, 100)])                                    # unsorted: BedFilter comes after the validator


def test_staged_and_memory(gen):
    import sambamba_b200 as sb
    p = gen["inv"]
    kw = dict(num_filter=(1, 0x400), subsample=0.5, seed=4)
    with vv.valid_oracle():
        want = vt.oracle_text(p, **kw)
    with sb.BDepth(p) as b:
        b.stage()
        for _ in range(2):
            assert b.run_view_text(valid=True, **kw) == want
            assert b.stats()["ms_reduce"] > 0
        assert b.run_view_count(valid=True, **vt.count_kw(kw)) == want.count(b"\n")
        assert b.run_view_text(**kw) == vt.oracle_text(p, **kw), "valid=False after a run with it"
    img = np.fromfile(p, dtype=np.uint8)
    with sb.BDepth(memory=img) as b:
        assert b.run_view_text(valid=True, **kw) == want
        refused_img = np.fromfile(gen["brk"], dtype=np.uint8)
    with sb.BDepth(memory=refused_img) as b:
        refused(b, gen["brk"])


def _rank_main(rank, world, path, uid, kw, what, q):
    try:
        sys.path.insert(0, helpers.ROOT)
        import sambamba_b200 as sb
        with sb.BDepth(path, device=rank if not EMULATE else 0) as b:
            b.set_shard(rank, world, uid)
            b.set_tuning(1 << 18, 2)
            r = b.run_view_count(valid=True, **kw) if what == "count" else b.run_view_text(valid=True, **kw)
            q.put((rank, "ok", r))
    except Exception as e:  # pragma: no cover
        q.put((rank, "err", getattr(e, "code", repr(e))))


def _ranks(world, path, kw, what):
    import queue
    import threading
    import sambamba_b200 as sb
    uid, ctx = sb.nccl_unique_id(), mp.get_context("spawn")
    q = queue.Queue() if EMULATE else ctx.Queue()
    ts = [(threading.Thread if EMULATE else ctx.Process)(target=_rank_main, args=(r, world, path, uid, kw, what, q)) for r in range(world)]
    for t in ts:
        t.start()
    res = sorted([q.get(timeout=1500) for _ in range(world)], key=lambda r: r[0])
    for t in ts:
        t.join(timeout=60)
    return res


@pytest.mark.parametrize("world", [2, 3, 4])
def test_several_ranks(gen, world):
    """Every rank returns the summed count and the texts join to the single-GPU text; a rank that refuses makes the others stop
    (BDEPTH_ERR_NCCL)."""
    import sambamba_b200 as sb
    if not EMULATE and sb.load_library().bdepth_device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    p = gen["inv"]
    for kw in (dict(num_filter=(0x40, 0), subsample=0.5, seed=world), dict()):
        with vv.valid_oracle():
            wt, wc = vt.oracle_text(p, **kw), vc.oracle_count(p, **kw)
        res = _ranks(world, p, kw, "text")
        assert all(r[1] == "ok" for r in res) and b"".join(r[2] for r in res) == wt, res
        res = _ranks(world, p, kw, "count")
        assert all(r[1] == "ok" and r[2] == wc for r in res), res                 # the all-reduce gives every rank the sum
    for what in ("count", "text"):
        res = _ranks(world, gen["brk"], {}, what)
        codes = sorted(r[2] for r in res)
        assert all(r[1] == "err" for r in res) and -2 in codes and set(codes) <= {-2, -6}, res


def test_full_size(tmp_path_factory):
    """The chr20 benchmark file (a small file of its shape under the emulation): bamgen's reads are all valid, so -v changes nothing."""
    if EMULATE:
        p = helpers.gen_bam(str(tmp_path_factory.mktemp("vvz") / "small.bam"), "-r", "chr20:300000", "-n", 20000, "-s", 20, "-t", 4)
    else:
        sys.path.insert(0, helpers.ROOT)
        import bench
        p = bench.ensure_workload(1, bench.READS_PER_UNIT)
    want_sha, want_len = vt.oracle_sha256(p)
    with vv.valid_oracle():
        want_n = vc.oracle_count(p)
    with bdepth(p) as b:
        n = b.run_view_count(valid=True)
        assert n == b.run_view_count() == want_n == (20000 if EMULATE else 12888833)
        h = hashlib.sha256()
        assert b.run_view_text(valid=True, sink=h.update) == want_len and h.hexdigest() == want_sha
