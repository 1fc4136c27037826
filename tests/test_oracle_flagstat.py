"""The flagstat checker (tools/flagstat_oracle.c) against an independent restatement of computeFlagStatistics (sambamba/flagstat.d:31-57)
written here over a struct walk of the depth oracle's inflate, and its CLI against hand-written text.  No GPU needed."""
import glob
import os
import random
import struct

import numpy as np

import flagstat_common as fc
import helpers


def py_flagstat(path):
    """flagstat.d:31-57, record by record."""
    u = helpers.oracle_inflate(path)
    o, _ = helpers.header_first_record_offset(u)
    b = u.tobytes()
    c = {n: [0, 0] for n in fc.FIELDS}
    while o + 4 <= len(b):
        bs, = struct.unpack_from("<i", b, o)
        assert o + 4 + bs <= len(b)
        ref_id, _pos, bmn, fnc, _lseq, mate_ref_id = struct.unpack_from("<iiIIii", b, o + 4)
        flag, mapq = fnc >> 16, (bmn >> 8) & 0xFF
        q = 1 if flag & 0x200 else 0
        c["total"][q] += 1
        if not flag & 0x4:
            c["mapped"][q] += 1
        if flag & 0x400:
            c["duplicates"][q] += 1
        if flag & 0x100:
            c["secondary"][q] += 1
        elif flag & 0x800:
            c["supplementary"][q] += 1
        elif flag & 0x1:
            c["paired"][q] += 1
            if flag & 0x2 and not flag & 0x4:
                c["proper_pair"][q] += 1
            if flag & 0x40:
                c["read1"][q] += 1
            if flag & 0x80:
                c["read2"][q] += 1
            if flag & 0x8 and not flag & 0x4:
                c["singletons"][q] += 1
            if not flag & 0x4 and not flag & 0x8:
                c["both_mapped"][q] += 1
                if ref_id != mate_ref_id:
                    c["mate_diff_chr"][q] += 1
                    if mapq >= 5:
                        c["mate_diff_chr_mapq5"][q] += 1
        o += 4 + bs
    return {k: tuple(v) for k, v in c.items()}


def test_oracle_equals_the_restatement(tmp_path):
    paths = sorted(glob.glob(os.path.join(helpers.GOLDEN, "*.bam")))
    paths.append(fc.write_hand_bam(str(tmp_path / "hand.bam")))
    paths.append(fc.write_hand_bam(str(tmp_path / "hand_small_blocks.bam"), block=150))          # records cut by BGZF members
    paths.append(helpers.gen_bam(str(tmp_path / "g.bam"), "-r", "chrA:200000", "-r", "chrB:90000", "-n", 20000, "-s", 7, "-t", 4))
    paths.append(helpers.gen_bam(str(tmp_path / "p.bam"), "-r", "chrA:200000", "-n", 20000, "-s", 8, "-t", 4, "--pairs", 3))
    for p in paths:
        assert fc.oracle_flagstat(p) == py_flagstat(p), p


def test_hand_made_file_reaches_every_category_in_both_classes(tmp_path):
    got = fc.oracle_flagstat(fc.write_hand_bam(str(tmp_path / "hand.bam")))
    assert all(p > 0 and f > 0 for p, f in got.values()), got
    assert got["total"] != (got["total"][1], got["total"][1]), "the two QC classes differ"
    assert got["mate_diff_chr"] != got["mate_diff_chr_mapq5"], "MAPQ 4 and 5 with the mate on another reference"


HAND_TEXT = """\
23 + 19 in total (QC-passed reads + QC-failed reads)
2 + 2 secondary
2 + 2 supplementary
2 + 2 duplicates
17 + 15 mapped (73.91%:78.95%)
15 + 13 paired in sequencing
9 + 8 read1
6 + 5 read2
4 + 2 properly paired (26.67%:15.38%)
10 + 8 with itself and mate mapped
1 + 1 singletons (6.67%:7.69%)
4 + 4 with mate mapped to a different chr
3 + 3 with mate mapped to a different chr (mapQ>=5)
"""
HAND_TABULAR = """\
in total (QC-passed reads + QC-failed reads),23,19
secondary,2,2
supplementary,2,2
duplicates,2,2
mapped,17:73.91%,15:78.95%
paired in sequencing,15,13
read1,9,8
read2,6,5
properly paired,4:26.67%,2:15.38%
with itself and mate mapped,10,8
singletons,1:6.67%,1:7.69%
with mate mapped to a different chr,4,4
with mate mapped to a different chr (mapQ>=5),3,3
"""
EMPTY_TEXT = """\
0 + 0 in total (QC-passed reads + QC-failed reads)
0 + 0 secondary
0 + 0 supplementary
0 + 0 duplicates
0 + 0 mapped (N/A:N/A)
0 + 0 paired in sequencing
0 + 0 read1
0 + 0 read2
0 + 0 properly paired (N/A:N/A)
0 + 0 with itself and mate mapped
0 + 0 singletons (N/A:N/A)
0 + 0 with mate mapped to a different chr
0 + 0 with mate mapped to a different chr (mapQ>=5)
"""
EMPTY_TABULAR = """\
in total (QC-passed reads + QC-failed reads),0,0
secondary,0,0
supplementary,0,0
duplicates,0,0
mapped,0:N/A,0:N/A
paired in sequencing,0,0
read1,0,0
read2,0,0
properly paired,0:N/A,0:N/A
with itself and mate mapped,0,0
singletons,0:N/A,0:N/A
with mate mapped to a different chr,0,0
with mate mapped to a different chr (mapQ>=5),0,0
"""


def test_oracle_cli_text(tmp_path):
    hand = fc.write_hand_bam(str(tmp_path / "hand.bam"))
    empty = helpers.write_bgzf(str(tmp_path / "empty.bam"), fc.bam_body(fc.HAND_REFS, []), len(fc.HAND_REFS))
    for path, plain, tab in ((hand, HAND_TEXT, HAND_TABULAR), (empty, EMPTY_TEXT, EMPTY_TABULAR)):
        assert fc.oracle_cli([path]) == (0, plain.encode(), b"")
        assert fc.oracle_cli(["-b", path]) == (0, tab.encode(), b"")


def percent_float(a, b):
    """percent (flagstat.d:66): to!float(a) / b * 100.0 returned as float."""
    return float(np.float32(float(np.float32(a) / np.float32(b)) * 100.0))


def test_percent_is_float_arithmetic(tmp_path):
    """The search for the smallest denominator (and, for it, the smallest numerator) at which the reference's float formula and plain
    double arithmetic print different %.2f; denominators up to 1000 are searched."""
    found = next(((a, b) for b in range(1, 1001) for a in range(b + 1) if "%.2f" % percent_float(a, b) != "%.2f" % (a / b * 100.0)), None)
    assert found == (23, 160), found
    assert "%.2f" % percent_float(23, 160) == "14.38" and "%.2f" % (23 / 160 * 100.0) == "14.37"
    p = fc.write_mapped_share(str(tmp_path / "share.bam"), 23, 160)
    rc, out, _ = fc.oracle_cli([p])
    assert rc == 0 and out.splitlines()[4] == b"23 + 0 mapped (14.38%:N/A)"


def test_shuffled_records_give_the_same_counts(tmp_path):
    """flagstat does not depend on the order of the records."""
    src = helpers.gen_bam(str(tmp_path / "g.bam"), "-r", "chrA:200000", "-n", 5000, "-s", 9, "-t", 2)
    u = helpers.oracle_inflate(src)
    first, refs = helpers.header_first_record_offset(u)
    b = u.tobytes()
    recs, o = [], first
    while o + 4 <= len(b):
        bs, = struct.unpack_from("<i", b, o)
        recs.append(b[o:o + 4 + bs])
        o += 4 + bs
    random.Random(3).shuffle(recs)
    p = helpers.write_bgzf(str(tmp_path / "shuf.bam"), b[:first] + b"".join(recs), len(refs))
    assert fc.oracle_flagstat(p) == fc.oracle_flagstat(src) == py_flagstat(p)


def test_errors(tmp_path):
    rc, out, err = fc.oracle_cli([str(tmp_path / "missing.bam")])
    assert rc == 1 and out == b"" and b"Cannot open file" in err
    body = fc.bam_body(fc.HAND_REFS, fc.hand_records())
    p = helpers.write_bgzf(str(tmp_path / "cut.bam"), body[:-5], len(fc.HAND_REFS))
    rc, out, err = fc.oracle_cli([p])
    assert rc == 1 and out == b"" and b"not enough data in stream" in err
