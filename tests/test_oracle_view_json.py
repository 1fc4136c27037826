"""The CPU restatement of `sambamba view -f json` (tools/view_count_oracle.c, TEST INFRASTRUCTURE) pinned on hand-written lines, and checked
against an independent decoding of the raw records: on the reference's own SAM file and on the edge lines that are valid JSON, json.loads of
each line must give the fields decoded from the record in Python."""
import json
import os
import subprocess

import pytest

import helpers
import view_count_common as vc
import view_json_common as vj
import view_text_common as vt

SAM = os.path.join(helpers.GOLDEN, "ex1_header.sam.gz")      # the reference's test/ex1_header.sam


def records_of(path):
    """The raw records of a BAM file (block_size included), in file order."""
    import struct
    u = helpers.oracle_inflate(path)
    first, _ = helpers.header_first_record_offset(u)
    raw = u.tobytes()
    return [raw[r[0]:r[0] + 4 + struct.unpack_from("<i", raw, r[0])[0]] for r in helpers.parse_records(u, first)]


def test_edge_lines_by_hand(tmp_path):
    p, want = vj.write_edge_bam(str(tmp_path / "e.bam"))
    got = vj.oracle_json(p)
    assert got.split(b"\n") == want.split(b"\n")


def test_edge_lines_parse_to_the_decoded_fields(tmp_path):
    p, want = vj.write_edge_bam(str(tmp_path / "e.bam"))
    recs, _, valid = vj.edge_records()
    lines = vj.oracle_json(p).split(b"\n")[:-1]
    refs = [n.decode("latin-1") for n, _ in vj.EDGE_REFS]
    for i, line in enumerate(lines):
        if i not in valid:                             # raw control bytes or lone high bytes: not JSON, as the reference writes them
            with pytest.raises(ValueError):
                json.loads(line.decode("utf-8"))
            continue
        assert vj.same_fields(vj.loads(line), vj.decode(recs[i], refs)) is None, line
    assert len(valid) >= 9


def test_golden_sam_parses_to_the_decoded_fields(tmp_path):
    p, _ = vt.sam_to_bam(SAM, str(tmp_path / "ex1.bam"))
    refs = [n for n, _ in helpers.header_first_record_offset(helpers.oracle_inflate(p))[1]]
    recs = records_of(p)
    lines = vj.oracle_json(p).split(b"\n")
    assert lines[-1] == b"" and len(lines) - 1 == len(recs) == 3270
    for line, rec in zip(lines, recs):
        assert vj.same_fields(vj.loads(line), vj.decode(rec, refs)) is None, line
    sam = vt.oracle_text(p).split(b"\n")
    for line, s in zip(lines[:-1], sam):                    # the same fields as the SAM line, where SAM spells them alike
        d, f = json.loads(line), s.decode().split("\t")
        assert [d["qname"], str(d["flag"]), d["rname"], str(d["pos"]), str(d["mapq"]), d["cigar"], d["rnext"], str(d["pnext"]), str(d["tlen"]), d["seq"]] == f[:10]


def every_byte_name():
    """A record whose read name is the bytes 1-254, every byte a name can hold (l_name 255)."""
    r = bytearray(vt.record("x" * 254, 0, 0, 9, 60, [(1, 0)], -1, -1, 0, "A"))
    r[36:36 + 254] = bytes(range(1, 255))
    return bytes(r)


def test_every_byte_of_a_read_name(tmp_path):
    """Only '"', '\\', '/' and bytes 8, 9, 10, 12, 13 are escaped; every other byte is written as it is."""
    p = vt.write_records(str(tmp_path / "n.bam"), vt.EDGE_REFS, [every_byte_name()])
    line = vj.oracle_json(p)
    q = b'"' + b"".join({8: b"\\b", 9: b"\\t", 10: b"\\n", 12: b"\\f", 13: b"\\r", 34: b'\\"', 47: b"\\/", 92: b"\\\\"}.get(c, bytes([c])) for c in range(1, 255)) + b'"'
    assert q == vj.quote(bytes(range(1, 255)))
    assert line == b'{"qname":' + q + b',"flag":0,"rname":"c1","pos":10,"mapq":60,"cigar":"1M","rnext":"*","pnext":0,"tlen":0,"seq":"A","qual":[30],"tags":{}}\n'


def test_edge_selection_and_order(tmp_path):
    p, want = vj.write_edge_bam(str(tmp_path / "e.bam"))
    lines = want.split(b"\n")[:-1]
    star = b"".join(x + b"\n" for x in lines if b'"rname":"*"' in x)
    assert vj.oracle_json(p, regions=["*"]) == star
    c1 = vj.oracle_json(p, regions=[(0, 0, 1000)])
    assert c1 == b"".join(x + b"\n" for x in lines if b'"rname":"c1"' in x)
    assert vj.oracle_json(p, regions=[(0, 0, 1000), "*", (0, 0, 1000)]) == c1 + star + c1
    for kw in (dict(), dict(regions=[(0, 15, 45), "*", (0, 15, 45)]), dict(bed=[(0, 0, 35), (1, 0, 500)]), dict(subsample=0.5, seed=3), dict(num_filter=(0, 4))):
        assert vj.oracle_json(p, **kw).count(b"\n") == vc.oracle_count(p, **vt.count_kw(kw)), kw      # (every '\n' in a value is escaped)


@pytest.mark.parametrize("what", [w for w, _ in vt.malformed_records()])
def test_malformed_records_are_refused(tmp_path, what):
    rec = dict(vt.malformed_records())[what]
    p = vt.write_records(str(tmp_path / "m.bam"), vt.EDGE_REFS, [rec], index=False)
    with pytest.raises(RuntimeError):
        vj.oracle_json(p)


def test_oracle_cli_json(tmp_path):
    p, want = vj.write_edge_bam(str(tmp_path / "e.bam"))
    r = subprocess.run([vc.ORACLE_EXE, "view", "-f", "json", p], capture_output=True)
    assert r.returncode == 0 and r.stdout == want
    r = subprocess.run([vc.ORACLE_EXE, "view", "-f", "json", p, "c1:1-1000", "*"], capture_output=True)
    assert r.returncode == 0 and r.stdout == vj.oracle_json(p, regions=[(0, 0, 1000), "*"])
    assert subprocess.run([vc.ORACLE_EXE, "view", "-f", "sam", p], capture_output=True).stdout == vt.oracle_text(p)
    assert vj.oracle_sha256(p)[1] == len(want)
