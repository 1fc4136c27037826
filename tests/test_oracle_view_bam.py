"""The CPU restatement of `sambamba view -f bam` (tools/view_count_oracle.c, view_bam_oracle): BamWriter's member cut over BgzfOutputStream on
hand-built record sizes, the header and reference list, bin recomputation, the zeroed last name byte, the reference-ID refusal, and that the
file it writes reads back with Python's gzip to the input's selected records."""
import gzip
import os
import struct

import pytest

import helpers
import view_bam_common as vb
import view_text_common as vt

L = 0xFF00
REFS = [("c1", 100000), ("c2", 5000)]


def sized(n, name="r", ref=0, pos=10):
    """A record of exactly n bytes (block_size field included), padded with a Z tag."""
    base = vt.record(name, 0, ref, pos, 30, [(10, 0)], -1, -1, 0, "ACGTACGTAC")
    pad = n - len(base)
    assert pad == 0 or pad >= 4, n
    return base if pad == 0 else vt.record(name, 0, ref, pos, 30, [(10, 0)], -1, -1, 0, "ACGTACGTAC", aux=b"XZZ" + b"a" * (pad - 4) + b"\0")


def no_name(rec):
    """rec with l_read_name 0 (no name, not even its NUL)."""
    r = bytearray(rec)
    del r[36]
    r[12] = 0
    struct.pack_into("<i", r, 0, len(r) - 4)
    return bytes(r)


def run(tmp_path, recs, header=b"@HD\tVN:1.6\n", level=-1, refs=REFS, **kw):
    p = vt.write_records(str(tmp_path / "s.bam"), refs, recs, index=False)
    return vb.oracle_bam(p, header, level, **kw)


def header_len(header=b"@HD\tVN:1.6\n", refs=REFS):
    return 12 + len(header) + sum(9 + len(n) for n, _ in refs)


@pytest.mark.parametrize("sizes,want", [
    ([L // 2, L // 2], [L]),                            # exact fill: one member, flushed when it reaches 0xFF00
    ([L // 2, L // 2 + 1], [L // 2, L // 2 + 1]),      # one byte over: the second read opens a member
    ([L, 100], [L, 100]),                               # a read of exactly 0xFF00
    ([100, L + 500, 64, 64], [100, L, 500, 128]),        # larger than a member: spans two; the next read flushes the rest
    ([3 * L + 70, 64], [L, L, L, 70, 64]),
    ([100, 100, L - 150, 64], [200, L - 150 + 64]),
])
def test_member_cut(tmp_path, sizes, want):
    raw, ms, f = run(tmp_path, [sized(n, "r%d" % i) for i, n in enumerate(sizes)])
    assert ms == [header_len()] + want
    assert sum(ms) == len(raw)
    assert gzip.decompress(f) == raw


def test_header_larger_than_a_member(tmp_path):
    h = b"@HD\tVN:1.6\n" + b"".join(b"@CO\t%s\n" % (b"x" * 1000) for _ in range(100))
    raw, ms, f = run(tmp_path, [sized(300)], header=h)
    n = header_len(h)
    assert ms == [L] * (n // L) + ([n % L] if n % L else []) + [300]
    assert raw[:4] == b"BAM\1" and struct.unpack_from("<i", raw, 4)[0] == len(h) and raw[8:8 + len(h)] == h


def test_no_selected_read(tmp_path):
    raw, ms, f = run(tmp_path, [sized(300)], num_filter=(0x400, 0))
    assert ms == [header_len()] and f.endswith(vb.BGZF_EOF)
    assert gzip.decompress(f) == raw


def test_bin_and_name_byte(tmp_path):
    recs = [vt.record("u", 4, -1, -1, 0, [], -1, -1, 0, "AC", bin_=0),                       # unmapped at -1: bin 4680
            vt.record("z", 0, 0, 1000, 30, [(5, 1)], -1, -1, 0, "ACGTA", bin_=0),           # covers nothing: reg2bin(1000, 1000)
            vt.record("nd", 0, 0, 16380, 30, [(2, 0), (10, 3), (3, 2)], -1, -1, 0, "AC", bin_=0),      # N / D spans cross 16384
            no_name(vt.record("", 0, 0, 5, 30, [(2, 0)], -1, -1, 0x7F010203, "AC", bin_=0))]      # l_read_name 0: the top byte of tlen goes
    raw, ms, f = run(tmp_path, recs)
    o = header_len()
    got = []
    while o < len(raw):
        bs = struct.unpack_from("<i", raw, o)[0]
        got.append(raw[o:o + 4 + bs]); o += 4 + bs
    bins = [struct.unpack_from("<H", r, 14)[0] for r in got]
    assert bins == [4680, helpers.reg2bin(1000, 1001), helpers.reg2bin(16380, 16395), helpers.reg2bin(5, 7)]
    for r, src in zip(got, recs):
        ln = src[12]
        fixed = bytearray(src); fixed[14:16] = r[14:16]; fixed[35 + ln] = 0
        assert r == bytes(fixed)
    assert struct.unpack_from("<i", got[3], 32)[0] == 0x00010203


def test_reference_id_refusal(tmp_path):
    with pytest.raises(RuntimeError, match="Read reference ID is out of range"):
        run(tmp_path, [sized(300), vt.record("x", 0, -2, 5, 30, [(2, 0)], -1, -1, 0, "AC")])
    with pytest.raises(RuntimeError, match="Read reference ID is out of range"):
        run(tmp_path, [vt.record("x", 0, 2, 5, 30, [(2, 0)], -1, -1, 0, "AC")])
    run(tmp_path, [vt.record("x", 0, 0, 5, 30, [(2, 0)], 7, 5, 0, "AC")])      # the mate's reference is not checked


def test_level_refusal(tmp_path):
    for lv in (-2, 10):
        with pytest.raises(RuntimeError, match=r"Compression level must be a number in interval \[-1, 9\]"):
            run(tmp_path, [sized(300)], level=lv)


@pytest.mark.parametrize("name", ["issue_204.bam", "mate_overlaps_1_3M_4M.bam"])
@pytest.mark.parametrize("level", [0, -1])
def test_golden_reads_back(name, level):
    p = os.path.join(helpers.GOLDEN, name)
    u = gzip.open(p).read()
    lt = struct.unpack_from("<i", u, 4)[0]
    raw, ms, f = vb.oracle_bam(p, u[8:8 + lt], level, num_filter=(0, 0x400))
    back = gzip.decompress(f)
    assert back == raw and [len(x) for _, x in vb.members(f)] == ms
    assert raw[:8 + lt] == u[:8 + lt]
