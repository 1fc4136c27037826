"""The CPU restatement of `sambamba view`'s SAM lines (tools/view_count_oracle.c, TEST INFRASTRUCTURE) pinned on the reference's own SAM file and
on hand-written lines: every tag type, floats at rounding ties and at the ends of the range, missing sequences and qualities, CIGAR op codes
9-15, unplaced reads, mates on another reference and a stray trailing aux byte."""
import gzip
import os
import struct
import subprocess

import pytest

import helpers
import view_count_common as vc
import view_text_common as vt

SAM = os.path.join(helpers.GOLDEN, "ex1_header.sam.gz")      # the reference's test/ex1_header.sam


def test_golden_sam_round_trip(tmp_path):
    body = [x for x in gzip.open(SAM).read().split(b"\n") if x and not x.startswith(b"@")]
    assert len(body) == 3270
    for x in body:                                   # what makes the round trip exact: integer tags only, no RNEXT spelled as the RNAME
        f = x.split(b"\t")
        assert f[6] != f[2] and all(t.split(b":")[1] == b"i" for t in f[11:])
    p, want = vt.sam_to_bam(SAM, str(tmp_path / "ex1.bam"))
    assert vt.oracle_text(p) == want
    assert vc.oracle_count(p) == 3270
    r = subprocess.run([vc.ORACLE_EXE, "view", p], capture_output=True)
    assert r.returncode == 0 and r.stdout == want


def test_edge_lines_by_hand(tmp_path):
    p, want = vt.write_edge_bam(str(tmp_path / "e.bam"))
    got = vt.oracle_text(p)
    assert got.split(b"\n") == want.split(b"\n")
    for bits, s in vt.EDGE_FLOATS:                   # the hand-written %g strings are what C prints
        f, = struct.unpack("<f", struct.pack("<I", bits))
        if f == f:
            assert "%g" % f == s, (hex(bits), s)


def test_edge_selection_and_order(tmp_path):
    p, want = vt.write_edge_bam(str(tmp_path / "e.bam"))
    lines = want.split(b"\n")[:-1]
    star = b"".join(x + b"\n" for x in lines if x.split(b"\t")[2] == b"*")
    assert vt.oracle_text(p, regions=["*"]) == star
    c1 = vt.oracle_text(p, regions=[(0, 0, 1000)])
    assert c1 == b"".join(x + b"\n" for x in lines if x.split(b"\t")[2] == b"c1")
    assert vt.oracle_text(p, regions=[(0, 0, 1000), "*", (0, 0, 1000)]) == c1 + star + c1
    assert vt.oracle_text(p, num_filter=(0, 4)) == b"".join(x + b"\n" for x in lines if not int(x.split(b"\t")[1]) & 4)
    assert vt.oracle_text(p, bed=[(1, 0, 10)]) == lines[7] + b"\n"
    for kw in (dict(), dict(regions=[(0, 15, 45), "*", (0, 15, 45)]), dict(bed=[(0, 0, 35), (1, 0, 500)]), dict(subsample=0.5, seed=3)):
        assert vt.oracle_text(p, **kw).count(b"\n") == vc.oracle_count(p, **vt.count_kw(kw)), kw


@pytest.mark.parametrize("what", [w for w, _ in vt.malformed_records()])
def test_malformed_records_are_refused(tmp_path, what):
    rec = dict(vt.malformed_records())[what]
    p = vt.write_records(str(tmp_path / "m.bam"), vt.EDGE_REFS, [rec], index=False)
    with pytest.raises(RuntimeError):
        vt.oracle_text(p)


def test_oracle_cli_text(tmp_path):
    p, want = vt.write_edge_bam(str(tmp_path / "e.bam"))
    lines = want.split(b"\n")[:-1]
    r = subprocess.run([vc.ORACLE_EXE, "view", p, "c1:1-1000", "*", "c2"], capture_output=True)
    assert r.returncode == 0
    assert r.stdout == b"".join(x + b"\n" for x in lines[:7] + lines[8:] + [lines[7]])
    assert subprocess.run([vc.ORACLE_EXE, "view", "-c", p, "c1:1-1000", "*", "c2"], capture_output=True).stdout == b"10\n"
