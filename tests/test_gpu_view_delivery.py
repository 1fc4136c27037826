"""How `view` hands its output to the callback, across its three formats (SAM, JSON, BAM): one handle running every format in turn, the shape of
the chunks, what counts as output already handed out when a foreign index forces a whole-file pass, and the pipeline's statistics."""
import os
import struct

import pytest

import helpers
import test_gpu_view_text as tvt
import view_bam_common as vb
import view_json_common as vj
import view_text_common as vt

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
gen = tvt.gen
HEADER = b"@HD\tVN:1.6\tSO:coordinate\n"
TINY = (1 << 16, 1)
PIECE = 64 << 20           # VIEW_TEXT_PIECE: the most bytes of text in one chunk, besides the line that crosses it
BATCH = 6 << 30            # the default batch; a smaller one caps the piece


def run(b, fmt, sink=None):
    if fmt == "sam":
        return b.run_view_text(sink=sink)
    if fmt == "json":
        return b.run_view_json(sink=sink)
    return b.run_view_bam(HEADER, int(fmt[3:]), sink=sink)


def check_oracle(p, fmt, got):
    if fmt == "sam":
        assert got == vt.oracle_text(p)
    elif fmt == "json":
        assert got == vj.oracle_json(p)
    else:
        level = int(fmt[3:])
        raw, sizes, want = vb.oracle_bam(p, HEADER, level)
        vb.check_against_oracle(got, raw, sizes, want, level)


def member_sizes(chunk):
    """The sizes of the BGZF members that make up chunk; asserts that it ends with a member."""
    out, o = [], 0
    while o < len(chunk):
        assert chunk[o:o + 16] == vb.HEADER_START, "member header at %d" % o
        out.append(struct.unpack_from("<H", chunk, o + 16)[0] + 1)
        o += out[-1]
    assert o == len(chunk), "a chunk ends inside a member"
    return out


def test_one_handle_every_format_in_turn(gen):
    """The slots grow and their pending state carries from one format's call into the next: each output is a fresh handle's and the oracle's."""
    p = gen["pairs"]
    order = ("sam", "bam0", "json", "sam", "bam-1")
    for tuning in (TINY, None):
        fresh = {}
        for fmt in set(order):
            with tvt.bdepth(p, tuning) as b:
                fresh[fmt] = run(b, fmt)
            check_oracle(p, fmt, fresh[fmt])
        with tvt.bdepth(p, tuning) as b:
            for fmt in order:
                assert run(b, fmt) == fresh[fmt], (tuning, fmt)


@pytest.mark.parametrize("tuning", [TINY, None])
def test_chunk_shape(gen, tuning):
    p = gen["pairs"]
    with tvt.bdepth(p, tuning) as b:
        for fmt in ("sam", "json"):
            chunks = []
            run(b, fmt, chunks.append)
            text = b"".join(chunks)
            longest = max(len(x) + 1 for x in text.split(b"\n"))
            assert all(c.endswith(b"\n") for c in chunks), "whole lines in every chunk"
            assert max(len(c) for c in chunks) <= min(PIECE, tuning[0] if tuning else BATCH) + longest
            assert len(chunks) > 3 or tuning is None
        for fmt in ("bam0", "bam-1"):
            chunks = []
            run(b, fmt, chunks.append)
            assert chunks[-1] == vb.BGZF_EOF, "the EOF member comes last, on its own"
            assert all(member_sizes(c) for c in chunks[:-1]), "whole members in every chunk"
            assert len(chunks) > 3 or tuning is None
            check_oracle(p, fmt, b"".join(chunks))


def _foreign_index_pair(d):
    """(F, region 1, region 2): F carries the index of G, which differs from F in two read names (read J one byte longer, read J2 one byte
    shorter).  At level 0 with 4 KiB members the member layout of the two files is the same, but G's reads between J and J2 start one byte
    later than F's: the index puts region 2's chunk one byte into a record of F.  Reads lie 2 kbp apart and inside their 16 kbp window, so each
    region's BAI chunk is the reads of its windows; region 2 is a window whose reads share one member, where the walk meets the chunk's end."""
    refs = [("chr1", 9000000)]
    cig, seq = [(100, 0)], "ACGT" * 25
    J, J2, STEP, WIN = 400, 2500, 2048, 16384
    reads = [(0, i * STEP, 60, 0, cig, seq, "r%07d" % i) for i in range(4000)]
    g_reads = list(reads)
    g_reads[J] = reads[J][:6] + ("r%07dx" % J,)
    g_reads[J2] = reads[J2][:6] + ("r%06d" % J2,)
    f = helpers.write_bam(str(d / "f.bam"), refs, reads, level=0, block=4096, bins="auto")
    g = helpers.write_bam(str(d / "g.bam"), refs, g_reads, level=0, block=4096, bins="auto")
    assert os.path.getsize(f) == os.path.getsize(g)
    with tvt.bdepth(g) as b:
        bai = b.build_index()
    open(f + ".bai", "wb").write(bai)
    u = helpers.oracle_inflate(g)
    raw = u.tobytes()
    recs = helpers.parse_records(u, helpers.header_first_record_offset(u)[0])
    win = {}
    for o, _, pos, *_ in recs:
        win.setdefault(pos // WIN, []).append((o, o + 4 + struct.unpack_from("<i", raw, o)[0] - 1))
    w = next(w for w in sorted(win) if J * STEP < w * WIN and (w + 1) * WIN < J2 * STEP and win[w][0][0] // 4096 == win[w][-1][1] // 4096)
    region1 = (0, 100 * STEP, 199 * STEP + 50)     # reads 100-199: about 20 KB of records, five members, 400 kbp before J
    region2 = (0, w * WIN, (w + 1) * WIN)
    return f, region1, region2


def test_restart_or_refusal_under_a_foreign_index(tmp_path):
    """Once output has gone out, a region chunk that the index misplaces refuses the run; before that, the run restarts as a whole-file pass.
    BAM counts a read as output when it joins the open member: region 1's reads close no member, and the run is refused all the same."""
    import sambamba_b200 as sb
    f, region1, region2 = _foreign_index_pair(tmp_path)
    with tvt.bdepth(f, (1 << 16, 2)) as b:
        for fmt in ("sam", "bam0"):
            with pytest.raises(sb.BDepthError) as e:
                if fmt == "sam":
                    b.run_view_text(bed=[region1, region2])
                else:
                    b.run_view_bam(HEADER, 0, bed=[region1, region2])
            assert e.value.code == -2 and "found after SAM lines were delivered" in e.value.msg, (fmt, e.value.msg)
    with tvt.bdepth(f, (1 << 16, 2)) as b:
        assert b.run_view_text(bed=[region2]) == vt.oracle_text(f, bed=[region2])
        assert b.stats()["file_bytes"] >= os.path.getsize(f) - 28, "a whole-file pass"
    with tvt.bdepth(f, (1 << 16, 2)) as b:
        got = b.run_view_bam(HEADER, 0, bed=[region2])
        assert b.stats()["file_bytes"] >= os.path.getsize(f) - 28, "a whole-file pass"
    raw, sizes, want = vb.oracle_bam(f, HEADER, 0, bed=[region2])
    vb.check_against_oracle(got, raw, sizes, want, 0)


def test_stats_match_the_count(gen):
    """The output runs report the pipeline's counters as view -c does for the same selection."""
    p = gen["plain"]
    kw = dict(num_filter=(0, 0x10), bed=[(0, 1000, gen["n"] * 5)])
    keys = ("file_bytes", "n_blocks", "cdata_bytes", "inflated_bytes", "n_records", "n_batches")
    with tvt.bdepth(p, (1 << 17, 3)) as b:
        b.run_view_count(**kw)
        want = {k: b.stats()[k] for k in keys}
        assert want["cdata_bytes"] > 0 and want["inflated_bytes"] > 0
        b.run_view_text(**kw)
        assert {k: b.stats()[k] for k in keys} == want
        b.run_view_json(**kw)
        assert {k: b.stats()[k] for k in keys} == want
        b.run_view_bam(HEADER, -1, **kw)
        assert {k: b.stats()[k] for k in keys} == want
