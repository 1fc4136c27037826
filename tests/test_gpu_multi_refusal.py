"""Several ranks, one of which refuses its input: every rank returns.  Each run mode owes its peers collectives (the sparse decision of a
region query, the all-reduce of the flagstat counters, that of view's count or failure word); a rank that stops with an error joins the
next one it owes with a "failed" mark, so that the others end with BDEPTH_ERR_NCCL instead of waiting for it.  The boundary-table case of
depth is in test_gpu_multi.py.  Here the second rank's half of a small file holds one record whose sequence does not fit its block_size:
an ordinary BDEPTH_ERR_FORMAT refusal on that rank alone."""
import multiprocessing as mp
import os
import struct
import sys
import zlib

import pytest

import helpers

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
EMULATE = os.environ.get("BDEPTH_EMULATE") == "1"
ERR_FORMAT, ERR_NCCL = -2, -6
N_READS = 3000
BAD = N_READS - 40           # the corrupt read: near the end of the file, far inside the second rank's shard


def _patch_l_seq(path, name, l_seq):
    """Set the l_seq field of the read called `name` in a BAM of stored (level 0) BGZF members, in place: the members keep their sizes, so
    an index built for the file before still describes it."""
    data = bytearray(open(path, "rb").read())
    members, o = [], 0
    while o < len(data):
        bsize = struct.unpack_from("<H", data, o + 16)[0] + 1
        isize = struct.unpack_from("<I", data, o + bsize - 4)[0]
        if isize:
            members.append((o, o + 18 + 5, isize))       # member offset, start of its stored bytes (after the stored block's header), their length
        o += bsize
    flat = b"".join(bytes(data[s:s + n]) for _, s, n in members)
    at = flat.index(name.encode() + b"\0") - 16        # l_seq, next_refID, next_pos, tlen precede the name
    for k, byte in enumerate(struct.pack("<i", l_seq)):
        u = at + k
        for m, s, n in members:
            if u < n:
                data[s + u] = byte
                break
            u -= n
    for m, s, n in members:      # (one stored block per member: its bytes end where the member's CRC32 and ISIZE begin)
        data[s + n:s + n + 4] = struct.pack("<I", zlib.crc32(bytes(data[s:s + n])))
    open(path, "wb").write(bytes(data))


@pytest.fixture(scope="module")
def bad_bam(tmp_path_factory):
    d = tmp_path_factory.mktemp("refuse")
    reads = [(0, 20 * i, 30, 0, [(40, 0)], "ACGTA" * 8, "bad" if i == BAD else "r%d" % i) for i in range(N_READS)]
    p = helpers.write_bam(str(d / "f.bam"), [("r0", 20 * N_READS + 100)], reads, block=2048, level=0, bins="auto", index=False)
    open(p + ".bai", "wb").write(helpers.oracle_build_bai(p))       # the index of the intact file
    _patch_l_seq(p, "bad", 5000)
    return p


def _rank_main(rank, world, path, uid, what, q):
    try:
        sys.path.insert(0, helpers.ROOT)
        import sambamba_b200 as sb
        with sb.BDepth(path, device=rank if not EMULATE else 0) as b:
            b.set_shard(rank, world, uid)
            b.set_tuning(1 << 16, 2)
            if what == "flagstat":
                b.run_flagstat()
            elif what == "view_count":
                b.run_view_count()
            elif what == "view_text":
                b.run_view_text()
            else:      # a -L query on the sorted, indexed file: the ranks stage their region chunks and decide together whether the index held
                b.run_view_count(bed=[(0, 100, 3000), (0, 20 * BAD - 1000, 20 * BAD + 1000)])
            q.put((rank, "ok", 0, ""))
    except Exception as e:  # pragma: no cover
        q.put((rank, "err", getattr(e, "code", None), str(e)))


def _run(world, path, what):
    import sambamba_b200 as sb
    uid = sb.nccl_unique_id()
    if EMULATE:           # ranks as threads over the NCCL stand-in (tests/emul)
        import queue
        import threading
        q = queue.Queue()
        ts = [threading.Thread(target=_rank_main, args=(r, world, path, uid, what, q)) for r in range(world)]
    else:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        ts = [ctx.Process(target=_rank_main, args=(r, world, path, uid, what, q)) for r in range(world)]
    for t in ts:
        t.start()
    res = sorted([q.get(timeout=1500) for _ in range(world)], key=lambda r: r[0])
    for t in ts:
        t.join(timeout=60)
    return res


def test_the_file_is_refused_on_one_gpu(bad_bam):
    import sambamba_b200 as sb
    with sb.BDepth(bad_bam) as b:
        with pytest.raises(sb.BDepthError) as e:
            b.run_flagstat()
    assert e.value.code == ERR_FORMAT and "do not fit its block_size" in e.value.msg


@pytest.mark.parametrize("what", ["sparse_decision", "flagstat", "view_count", "view_text"])
def test_one_rank_refuses_the_others_return(bad_bam, what):
    import sambamba_b200 as sb
    if not EMULATE and sb.load_library().bdepth_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    res = _run(2, bad_bam, what)
    assert [r[1] for r in res] == ["err", "err"], res
    assert res[1][2] == ERR_FORMAT and "do not fit its block_size" in res[1][3], res
    assert res[0][2] == ERR_NCCL and "another rank of the run stopped with an error" in res[0][3], res
