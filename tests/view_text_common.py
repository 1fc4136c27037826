"""Shared pieces of the `view` SAM-text tests: the binding of the CPU restatement's text entry point (tools/view_count_oracle.c, TEST
INFRASTRUCTURE), a SAM-to-BAM encoder for the golden SAM file, a raw record encoder, and a hand-made edge file whose lines are written out by
hand (every tag type, float rounding ties, missing sequences and qualities, CIGAR op codes 9-15, unplaced reads, a different mate reference and
a stray trailing aux byte)."""
import ctypes as C
import gzip
import hashlib
import os
import re
import struct
import subprocess

import flagstat_common as fc
import helpers
import view_count_common as vc

UNMAPPED = 0xFFFFFFFF
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(vc.ORACLE_LIB)
        _lib.view_text_oracle.argtypes = [C.c_char_p, C.c_uint, C.c_uint, C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(C.c_uint32), C.c_size_t,
                                          C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        _lib.view_text_oracle_free.argtypes = [C.c_void_p]
        _lib.view_count_oracle_error.restype = C.c_char_p
    return _lib


def oracle_text(path, num_filter=(0, 0), subsample=None, seed=0, bed=None, regions=None):
    """The same arguments as BDepth.run_view_text ("*" entries in `regions` in their place)."""
    L = _L()
    rg = bed if bed is not None else (regions or [])
    rg = [(UNMAPPED, 0, 0) if r == "*" else r for r in rg]
    flat = (C.c_uint32 * max(3 * len(rg), 1))(*[v for r in rg for v in r])
    mode = 1 if bed is not None else (2 if rg else 0)
    buf, n = C.c_void_p(), C.c_size_t()
    rc = L.view_text_oracle(os.fsencode(path), num_filter[0], num_filter[1], 0 if subsample is None else 1, 0 if subsample is None else vc.threshold(subsample),
                            seed, mode, flat, len(rg), C.byref(buf), C.byref(n))
    if rc:
        raise RuntimeError(L.view_count_oracle_error().decode())
    out = C.string_at(buf, n.value) if n.value else b""
    L.view_text_oracle_free(buf)
    return out


def oracle_sha256(path, bed=None):
    """(SHA-256, length) of the oracle CLI's text, streamed (the chr20 file prints about 5 GB); bed: the text of a BED file for -L."""
    import tempfile
    h, n = hashlib.sha256(), 0
    with tempfile.NamedTemporaryFile("w", suffix=".bed") as f:
        f.write(bed or "")
        f.flush()
        with subprocess.Popen([vc.ORACLE_EXE, "view"] + (["-L", f.name] if bed else []) + [path], stdout=subprocess.PIPE) as pr:
            for c in iter(lambda: pr.stdout.read(1 << 24), b""):
                h.update(c)
                n += len(c)
    assert pr.returncode == 0
    return h.hexdigest(), n


def count_kw(kw):
    """run_view_count's keywords for run_view_text's: the "*" entries become n_unmapped."""
    kw = dict(kw)
    if "regions" in kw:
        rg = kw["regions"]
        kw["regions"] = [r for r in rg if r != "*"]
        kw["n_unmapped"] = sum(1 for r in rg if r == "*")
    return kw


# ---- raw records
CODE = {c: i for i, c in enumerate("=ACMGRSVTWYHKDBN")}
FMT = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "I"}      # (floats are given as bit patterns)


def record(name, flag, ref, pos, mapq, cigar, nref, npos, tlen, seq, qual=None, aux=b"", bin_=None):
    """One BAM record, block_size included.  cigar: [(len, op code)]; qual: bytes (default 30 each); bin_: the alignment's BAI bin unless given."""
    if bin_ is None:
        span = 0 if flag & 4 else sum(l for l, op in cigar if op in (0, 2, 3, 7, 8))
        bin_ = helpers.reg2bin(max(pos, 0), max(pos, 0) + max(span, 1))
    nm = name.encode() + b"\0"
    packed = bytes((CODE[seq[i]] << 4) | (CODE[seq[i + 1]] if i + 1 < len(seq) else 0) for i in range(0, len(seq), 2))
    body = struct.pack("<iiIIiiii", ref, pos, (bin_ << 16) | (mapq << 8) | len(nm), (flag << 16) | len(cigar), len(seq), nref, npos, tlen)
    body += nm + b"".join(struct.pack("<I", (l << 4) | op) for l, op in cigar) + packed + (bytes([30] * len(seq)) if qual is None else bytes(qual)) + aux
    return struct.pack("<i", len(body)) + body


def tag(key, t, v):
    """Raw aux bytes of one tag; B arrays as (element type, values)."""
    k = key.encode() + t.encode()
    if t in FMT:
        return k + struct.pack("<" + FMT[t], v)
    if t == "A":
        return k + v.encode()
    if t in "ZH":
        return k + v.encode() + b"\0"
    return k + v[0].encode() + struct.pack("<I", len(v[1])) + b"".join(struct.pack("<" + FMT[v[0]], x) for x in v[1])


def write_records(path, refs, recs, index=True):
    p = helpers.write_bgzf(path, fc.bam_body(refs, recs, sorted_header=True), len(refs))
    if index:
        with open(p + ".bai", "wb") as f:
            f.write(helpers.oracle_build_bai(p))
    return p


def sam_to_bam(sam_gz, bam_path):
    """Encode a gzipped SAM file (integer tags only) as BAM with its own header; returns (bam path, its body lines, '\\n' after each)."""
    lines = [x for x in gzip.open(sam_gz).read().split(b"\n") if x]
    hdr, body = [x for x in lines if x.startswith(b"@")], [x for x in lines if not x.startswith(b"@")]
    refs = [(f[b"SN"].decode(), int(f[b"LN"])) for f in (dict(x.split(b":", 1) for x in h.split(b"\t")[1:]) for h in hdr if h.startswith(b"@SQ"))]
    rid = {n: i for i, (n, _) in enumerate(refs)}
    recs = []
    for line in body:
        f = line.decode().split("\t")
        ref = rid.get(f[2], -1)
        cigar = [(int(n), "MIDNSHP=X".index(op)) for n, op in re.findall(r"(\d+)([MIDNSHP=X])", f[5])]
        seq = "" if f[9] == "*" else f[9]
        qual = bytes([0xFF] * len(seq)) if f[10] == "*" else bytes(ord(c) - 33 for c in f[10])
        aux = b""
        for x in f[11:]:
            key, t, v = x.split(":", 2)
            n = int(v)
            assert t == "i", x
            aux += tag(key, "c" if -128 <= n < 128 else "C" if 0 <= n < 256 else "s" if -32768 <= n < 32768 else "S" if 0 <= n < 65536 else "i", n)
        recs.append(record(f[0], int(f[1]), ref, int(f[3]) - 1, int(f[4]), cigar, ref if f[6] == "=" else rid.get(f[6], -1), int(f[7]) - 1, int(f[8]), seq, qual, aux))
    text = b"\n".join(hdr) + b"\n"
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    out += b"".join(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l) for n, l in refs)
    p = helpers.write_bgzf(bam_path, out + b"".join(recs), len(refs))
    with open(p + ".bai", "wb") as fb:
        fb.write(helpers.oracle_build_bai(p))
    return p, b"".join(x + b"\n" for x in body)


# ---- the edge file
EDGE_REFS = [("c1", 1000), ("c2", 500)]
_F = lambda x: struct.unpack("<I", struct.pack("<f", x))[0]      # noqa: E731 -- the float's bit pattern
EDGE_FLOATS = [(_F(1234565.0), "1.23456e+06"), (_F(1234575.0), "1.23458e+06"), (_F(999999.5), "1e+06"), (_F(0.5), "0.5"), (_F(100000.0), "100000"),
               (_F(1e6), "1e+06"), (_F(123.456), "123.456"), (_F(0.0001), "0.0001"), (_F(1e-5), "1e-05"), (0x00000001, "1.4013e-45"),
               (0x007FFFFF, "1.17549e-38"), (0x7F7FFFFF, "3.40282e+38"), (0x7F800000, "inf"), (0xFF800000, "-inf"), (0x7FC00000, "nan"),
               (0xFFC00000, "-nan"), (0x80000000, "-0"), (0, "0"), (_F(-2.5), "-2.5"), (_F(0.00012345), "0.00012345"), (_F(123456.0), "123456"),
               (_F(1234567.0), "1.23457e+06"), (_F(0.1), "0.1")]


def edge_records():
    """(records, the lines `sambamba view` prints for them), written out by hand."""
    R, L = [], []
    allt = (tag("XA", "A", "x") + tag("Xc", "c", -5) + tag("XC", "C", 200) + tag("Xs", "s", -300) + tag("XS", "S", 60000) + tag("Xi", "i", -70000)
            + tag("XI", "I", 4000000000) + tag("XZ", "Z", "hello world") + tag("XH", "H", "1AE3") + tag("Bc", "B", ("c", [-1, 2]))
            + tag("BC", "B", ("C", [255, 0])) + tag("Bs", "B", ("s", [-1000])) + tag("BS", "B", ("S", [65535])) + tag("Bi", "B", ("i", [-2147483648, 7]))
            + tag("BI", "B", ("I", [4294967295])) + tag("Bf", "B", ("f", [_F(1.5), _F(-0.25)])) + tag("Be", "B", ("c", [])) + tag("XE", "Z", ""))
    R.append(record("all_tags", 0, 0, 9, 60, [(5, 0)], -1, -1, 0, "ACGTN", bytes([30, 31, 32, 33, 34]), allt))
    L.append("all_tags\t0\tc1\t10\t60\t5M\t*\t0\t0\tACGTN\t?@ABC\tXA:A:x\tXc:i:-5\tXC:i:200\tXs:i:-300\tXS:i:60000\tXi:i:-70000\tXI:i:4000000000"
             "\tXZ:Z:hello world\tXH:H:1AE3\tBc:B:c,-1,2\tBC:B:C,255,0\tBs:B:s,-1000\tBS:B:S,65535\tBi:B:i,-2147483648,7\tBI:B:I,4294967295"
             "\tBf:B:f,1.5,-0.25\tBe:B:c,\tXE:Z:")
    fl = b"".join(tag("F%d" % (i % 10), "f", b) for i, (b, _) in enumerate(EDGE_FLOATS)) + tag("FB", "B", ("f", []))
    fb = tag("FA", "B", ("f", [b for b, _ in EDGE_FLOATS]))
    R.append(record("floats", 16, 0, 19, 0, [(4, 0)], 0, 99, 84, "ACGT", None, fl + fb))
    L.append("floats\t16\tc1\t20\t0\t4M\t=\t100\t84\tACGT\t????" + "".join("\tF%d:f:%s" % (i % 10, s) for i, (_, s) in enumerate(EDGE_FLOATS))
             + "\tFB:B:f,\tFA:B:f," + ",".join(s for _, s in EDGE_FLOATS))
    R.append(record("no_seq", 0, 0, 29, 7, [(3, 0)], 1, 49, -123, ""))
    L.append("no_seq\t0\tc1\t30\t7\t3M\tc2\t50\t-123\t*\t*")
    R.append(record("qual_ff_first", 0, 0, 39, 7, [(3, 0)], -1, -1, 0, "ACG", bytes([0xFF, 0xFF, 0xFF])))
    L.append("qual_ff_first\t0\tc1\t40\t7\t3M\t*\t0\t0\tACG\t*")
    R.append(record("qual_ff_later", 0, 0, 49, 7, [(3, 0)], -1, -1, 0, "MRW", bytes([30, 0xFF, 93])))
    L.append("qual_ff_later\t0\tc1\t50\t7\t3M\t*\t0\t0\tMRW\t? ~")
    R.append(record("no_cigar", 4, 0, 59, 0, [], 0, 59, 0, "=ACMGRSVTWYHKDBN", None, tag("NM", "i", 0) + b"X"))
    L.append("no_cigar\t4\tc1\t60\t0\t*\t=\t60\t0\t=ACMGRSVTWYHKDBN\t" + "?" * 16 + "\tNM:i:0")
    R.append(record("odd_ops", 0, 0, 69, 60, [(1, 9), (2, 10), (3, 11), (4, 12), (5, 13), (6, 14), (7, 15), (8, 8), (9, 7), (10, 6)], -1, -1, 0, "A"))
    L.append("odd_ops\t0\tc1\t70\t60\t1?2?3?4?5?6?7?8X9=10P\t*\t0\t0\tA\t?")
    R.append(record("mate_c1", 0x41, 1, 4, 60, [(2, 4), (3, 0), (1, 1)], 0, 999, 0, "ACGTAC"))
    L.append("mate_c1\t65\tc2\t5\t60\t2S3M1I\tc1\t1000\t0\tACGTAC\t??????")
    R.append(record("unplaced", 4, -1, -1, 0, [], -1, -1, 0, "ACGT", None, tag("RG", "Z", "g1")))
    L.append("unplaced\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\t????\tRG:Z:g1")
    R.append(record("unplaced_mate", 0x45, -1, -1, 0, [], 1, 9, 0, "A"))
    L.append("unplaced_mate\t69\t*\t0\t0\t*\tc2\t10\t0\tA\t?")
    return R, "".join(x + "\n" for x in L).encode()


def write_edge_bam(path):
    recs, text = edge_records()
    return write_records(path, EDGE_REFS, recs), text


# ---- malformed records: (what, record), each refused with BDEPTH_ERR_FORMAT
def malformed_records():
    ok = lambda aux=b"", **kw: record(kw.get("name", "m"), 0, kw.get("ref", 0), 10, 60, [(4, 0)], kw.get("nref", -1), -1, 0, "ACGT", None, aux)   # noqa: E731
    return [("ref", ok(ref=5)), ("mate_ref", ok(nref=7)), ("tag_type", ok(b"XXq\x01")), ("b_type", ok(b"XXBq\x01\0\0\0\x05")),
            ("no_nul", ok(b"XXZabc")), ("tag_overrun", ok(b"XXi\x01\x02")), ("b_overrun", ok(b"XXBi\x03\0\0\0\x01\0\0\0")), ("key_only", ok(b"XX"))]
