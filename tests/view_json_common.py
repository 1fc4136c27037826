"""Shared pieces of the `view -f json` tests: the binding of the CPU restatement's JSON entry point (tools/view_count_oracle.c, TEST
INFRASTRUCTURE), BioD's string escape restated in Python, an independent decoder of raw records into the fields `toJson` prints, and a hand-made
edge file whose lines are written out by hand (every tag type, every escaped byte and raw control and high bytes in a read name, a reference
name, Z, H and A values and a tag key, +-inf and NaN in f and B:f, the %g ties of EDGE_FLOATS, empty B arrays, missing sequences and
qualities, 0xFF qualities, CIGAR op codes 9-15, unplaced reads and mates on another reference)."""
import ctypes as C
import hashlib
import os
import struct
import subprocess

import helpers
import view_count_common as vc
import view_text_common as vt

_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(vc.ORACLE_LIB)
        _lib.view_json_oracle.argtypes = [C.c_char_p, C.c_uint, C.c_uint, C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(C.c_uint32), C.c_size_t,
                                          C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        _lib.view_text_oracle_free.argtypes = [C.c_void_p]
        _lib.view_count_oracle_error.restype = C.c_char_p
    return _lib


def oracle_json(path, num_filter=(0, 0), subsample=None, seed=0, bed=None, regions=None):
    """The same arguments as BDepth.run_view_json ("*" entries in `regions` in their place)."""
    L = _L()
    rg = bed if bed is not None else (regions or [])
    rg = [(vt.UNMAPPED, 0, 0) if r == "*" else r for r in rg]
    flat = (C.c_uint32 * max(3 * len(rg), 1))(*[v for r in rg for v in r])
    mode = 1 if bed is not None else (2 if rg else 0)
    buf, n = C.c_void_p(), C.c_size_t()
    rc = L.view_json_oracle(os.fsencode(path), num_filter[0], num_filter[1], 0 if subsample is None else 1, 0 if subsample is None else vc.threshold(subsample),
                            seed, mode, flat, len(rg), C.byref(buf), C.byref(n))
    if rc:
        raise RuntimeError(L.view_count_oracle_error().decode())
    out = C.string_at(buf, n.value) if n.value else b""
    L.view_text_oracle_free(buf)
    return out


def oracle_sha256(path, bed=None):
    """(SHA-256, length) of the oracle CLI's JSON text, streamed; bed: the text of a BED file for -L."""
    import tempfile
    h, n = hashlib.sha256(), 0
    with tempfile.NamedTemporaryFile("w", suffix=".bed") as f:
        f.write(bed or "")
        f.flush()
        with subprocess.Popen([vc.ORACLE_EXE, "view", "-f", "json"] + (["-L", f.name] if bed else []) + [path], stdout=subprocess.PIPE) as pr:
            for c in iter(lambda: pr.stdout.read(1 << 24), b""):
                h.update(c)
                n += len(c)
    assert pr.returncode == 0
    return h.hexdigest(), n


ESC = {8: b"\\b", 9: b"\\t", 10: b"\\n", 12: b"\\f", 13: b"\\r", ord('"'): b'\\"', ord("/"): b"\\/", ord("\\"): b"\\\\"}


def quote(s):
    """writeStringJson of the bytes s: only the eight bytes of ESC are escaped."""
    return b'"' + b"".join(ESC.get(c, bytes([c])) for c in s) + b'"'


# ---- an independent decoder: the fields of toJson from a raw record (block_size included), as Python values json.loads would give
def decode(rec, refs):
    """refs: the reference names as str.  Floats are Python floats of the stored float (NaN as None)."""
    ref, pos, bmn, fnc, l_seq, nref, npos, tlen = struct.unpack_from("<iiIIiiii", rec, 4)
    l_name, mapq, flag, n_cig = bmn & 0xFF, (bmn >> 8) & 0xFF, fnc >> 16, fnc & 0xFFFF
    o = 36
    name = rec[o:o + l_name - 1].decode()
    o += l_name
    cig = struct.unpack_from("<%dI" % n_cig, rec, o)
    o += 4 * n_cig
    seq = "".join("=ACMGRSVTWYHKDBN"[(rec[o + i // 2] >> (0 if i & 1 else 4)) & 15] for i in range(l_seq))
    o += (l_seq + 1) // 2
    qual = list(rec[o:o + l_seq])
    o += l_seq
    wrap = lambda v: (v + 1 + (1 << 31)) % (1 << 32) - (1 << 31)      # noqa: E731 -- D's int + 1
    fmt = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}

    def val(t, at):
        v, = struct.unpack_from("<" + fmt[t], rec, at)
        return (None if v != v else v), struct.calcsize(fmt[t])
    tags = []
    while o + 1 < len(rec):
        key, t = rec[o:o + 2].decode(), chr(rec[o + 2])
        o += 3
        if t == "A":
            v, o = chr(rec[o]), o + 1
        elif t in "ZH":
            e = rec.index(b"\0", o)
            v, o = rec[o:e].decode(), e + 1
        elif t == "B":
            et, n = chr(rec[o]), struct.unpack_from("<I", rec, o + 1)[0]
            o += 5
            v = []
            for _ in range(n):
                x, sz = val(et, o)
                v.append(x)
                o += sz
        else:
            v, sz = val(t, o)
            o += sz
        tags.append((key, v))
    return {"qname": name, "flag": flag, "rname": "*" if ref == -1 else refs[ref], "pos": wrap(pos), "mapq": mapq,
            "cigar": "".join("%d%s" % (c >> 4, "MIDNSHP=X???????"[c & 15]) for c in cig) or "*",
            "rnext": "*" if nref == -1 else "=" if nref == ref else refs[nref], "pnext": wrap(npos), "tlen": tlen, "seq": seq or "*",
            "qual": qual, "tags": tags}


def _close(a, b):
    if isinstance(b, float) and not isinstance(a, bool) and isinstance(a, (int, float)):
        if b in (float("inf"), float("-inf")):
            return a == b
        return abs(a - b) <= 1e-5 * abs(b) + 1e-45      # %g keeps 6 significant digits
    if isinstance(b, list):
        return isinstance(a, list) and len(a) == len(b) and all(_close(x, y) for x, y in zip(a, b))
    return a == b and type(a) is type(b)


def loads(line):
    """json.loads of a line, with the tags as a list of (key, value) pairs: a record may hold a tag key twice."""
    import json
    return json.loads(line, object_pairs_hook=lambda kv: dict(kv) if kv and kv[0][0] == "qname" else [tuple(x) for x in kv])


def same_fields(parsed, want):
    """loads() of a line against decode(); returns the first field that differs, or None."""
    for k, v in want.items():
        got = parsed[k]
        if k == "tags":
            if len(got) != len(v) or any(g[0] != w[0] or not _close(g[1], w[1]) for g, w in zip(got, v)):
                return k
        elif not _close(got, v):
            return k
    return None if list(parsed) == list(want) else "keys"


# ---- the edge file
EDGE_REFS = [(b"c1", 1000), (b'w/"\\\t\x01\xe9', 500), (b'c/3"\\', 300)]      # ref 1: escapes, a raw control and a raw high byte
_F = vt._F
JSON_FLOAT = {"inf": "1.0e+1024", "-inf": "-1.0e+1024", "nan": "null", "-nan": "null"}
EDGE_FLOATS = [(b, JSON_FLOAT.get(s, s)) for b, s in vt.EDGE_FLOATS] + [(0x7F800001, "null"), (0xFFFFFFFF, "null")]


def raw_tag(key, t, v):
    """Raw aux bytes of one tag given as bytes (any byte in the key and the value); Z / H get their NUL."""
    return key + t + v + (b"\0" if t in b"ZH" else b"")


def bam_body(refs, records):
    """fc.bam_body with reference names as bytes."""
    text = b"@HD\tVN:1.6\tSO:coordinate\n"
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for n, ln in refs:
        out += struct.pack("<i", len(n) + 1) + n + b"\0" + struct.pack("<i", ln)
    return out + b"".join(records)


def edge_records():
    """(records, the lines `sambamba view -f json` prints for them, the indices of the lines that are valid JSON), written out by hand."""
    R, L, valid = [], [], []

    def add(rec, line, ok=True):
        if ok:
            valid.append(len(R))
        R.append(rec)
        L.append(line)
    allt = (vt.tag("XA", "A", "x") + vt.tag("Xc", "c", -5) + vt.tag("XC", "C", 200) + vt.tag("Xs", "s", -300) + vt.tag("XS", "S", 60000)
            + vt.tag("Xi", "i", -70000) + vt.tag("XI", "I", 4000000000) + vt.tag("XZ", "Z", "hello world") + vt.tag("XH", "H", "1AE3")
            + vt.tag("Bc", "B", ("c", [-1, 2])) + vt.tag("BC", "B", ("C", [255, 0])) + vt.tag("Bs", "B", ("s", [-1000])) + vt.tag("BS", "B", ("S", [65535]))
            + vt.tag("Bi", "B", ("i", [-2147483647, 7])) + vt.tag("BI", "B", ("I", [4294967295])) + vt.tag("Bf", "B", ("f", [_F(1.5), _F(-0.25)]))
            + vt.tag("Be", "B", ("c", [])) + vt.tag("XE", "Z", ""))
    add(vt.record("all_tags", 0, 0, 9, 60, [(5, 0)], -1, -1, 0, "ACGTN", bytes([30, 31, 32, 33, 34]), allt),
        b'{"qname":"all_tags","flag":0,"rname":"c1","pos":10,"mapq":60,"cigar":"5M","rnext":"*","pnext":0,"tlen":0,"seq":"ACGTN",'
        b'"qual":[30,31,32,33,34],"tags":{"XA":"x","Xc":-5,"XC":200,"Xs":-300,"XS":60000,"Xi":-70000,"XI":4000000000,"XZ":"hello world",'
        b'"XH":"1AE3","Bc":[-1,2],"BC":[255,0],"Bs":[-1000],"BS":[65535],"Bi":[-2147483647,7],"BI":[4294967295],"Bf":[1.5,-0.25],"Be":[],"XE":""}}')
    esc = (raw_tag(b'/"', b"Z", b'a"b\\c/d\be\tf\ng\fh\ri\x01j\x1fk\x7fl\xffm\x80') + raw_tag(b"\xe9\\", b"Z", b"\xc3\xa9") + raw_tag(b"A1", b"A", b'"')
           + raw_tag(b"A2", b"A", b"\\") + raw_tag(b"A3", b"A", b"/") + raw_tag(b"A4", b"A", b"\n") + raw_tag(b"A5", b"A", b"\xe9")
           + raw_tag(b"A6", b"A", b"\x01") + raw_tag(b"XH", b"H", b"0A/F\r") + raw_tag(b"\b\t", b"i", struct.pack("<i", 3)))
    add(vt.record('e/"s\\c\b\t\n\f\r\x01\x7f\xe9', 0x41, 0, 14, 20, [(3, 0)], 1, 99, 0, "ACG", None, esc),
        b'{"qname":"e\\/\\"s\\\\c\\b\\t\\n\\f\\r\x01\x7f\xc3\xa9","flag":65,"rname":"c1","pos":15,"mapq":20,"cigar":"3M",'
        b'"rnext":"w\\/\\"\\\\\\t\x01\xe9","pnext":100,"tlen":0,"seq":"ACG","qual":[30,30,30],"tags":{"\\/\\"":"a\\"b\\\\c\\/d\\be\\tf\\ng\\fh\\ri\x01j\x1fk\x7fl\xffm\x80",'
        b'"\xe9\\\\":"\xc3\xa9","A1":"\\"","A2":"\\\\","A3":"\\/","A4":"\\n","A5":"\xe9","A6":"\x01","XH":"0A\\/F\\r","\\b\\t":3}}', ok=False)
    fl = b"".join(vt.tag("F%d" % (i % 10), "f", b) for i, (b, _) in enumerate(EDGE_FLOATS)) + vt.tag("FB", "B", ("f", []))
    fb = vt.tag("FA", "B", ("f", [b for b, _ in EDGE_FLOATS]))
    add(vt.record("floats", 16, 0, 19, 0, [(4, 0)], 0, 99, 84, "ACGT", None, fl + fb),
        b'{"qname":"floats","flag":16,"rname":"c1","pos":20,"mapq":0,"cigar":"4M","rnext":"=","pnext":100,"tlen":84,"seq":"ACGT",'
        b'"qual":[30,30,30,30],"tags":{' + ",".join('"F%d":%s' % (i % 10, s) for i, (_, s) in enumerate(EDGE_FLOATS)).encode()
        + b',"FB":[],"FA":[' + ",".join(s for _, s in EDGE_FLOATS).encode() + b"]}}")
    add(vt.record("no_seq", 0, 0, 29, 7, [(3, 0)], 2, 49, -123, ""),
        b'{"qname":"no_seq","flag":0,"rname":"c1","pos":30,"mapq":7,"cigar":"3M","rnext":"c\\/3\\"\\\\","pnext":50,"tlen":-123,"seq":"*","qual":[],"tags":{}}')
    add(vt.record("qual_ff", 0, 0, 39, 7, [(3, 0)], -1, -1, 0, "ACG", bytes([0xFF, 0xFF, 0xFF])),
        b'{"qname":"qual_ff","flag":0,"rname":"c1","pos":40,"mapq":7,"cigar":"3M","rnext":"*","pnext":0,"tlen":0,"seq":"ACG","qual":[255,255,255],"tags":{}}')
    add(vt.record("qual_mix", 0, 0, 49, 7, [(6, 0)], -1, -1, 0, "MRWSYK", bytes([0, 9, 10, 99, 100, 0xFF])),
        b'{"qname":"qual_mix","flag":0,"rname":"c1","pos":50,"mapq":7,"cigar":"6M","rnext":"*","pnext":0,"tlen":0,"seq":"MRWSYK","qual":[0,9,10,99,100,255],"tags":{}}')
    add(vt.record("no_cigar", 4, 0, 59, 0, [], 0, 59, 0, "=ACMGRSVTWYHKDBN", None, vt.tag("NM", "i", 0) + b"X"),
        b'{"qname":"no_cigar","flag":4,"rname":"c1","pos":60,"mapq":0,"cigar":"*","rnext":"=","pnext":60,"tlen":0,"seq":"=ACMGRSVTWYHKDBN",'
        b'"qual":[' + b",".join([b"30"] * 16) + b'],"tags":{"NM":0}}')
    add(vt.record("odd_ops", 0, 0, 69, 60, [(1, 9), (2, 10), (3, 11), (4, 12), (5, 13), (6, 14), (7, 15), (8, 8), (9, 7), (10, 6)], -1, -1, 0, "A"),
        b'{"qname":"odd_ops","flag":0,"rname":"c1","pos":70,"mapq":60,"cigar":"1?2?3?4?5?6?7?8X9=10P","rnext":"*","pnext":0,"tlen":0,"seq":"A","qual":[30],"tags":{}}')
    empt = b"".join(vt.tag("E" + t, "B", (t, [])) for t in "cCsSiIf") + vt.tag("EZ", "Z", "") + vt.tag("EH", "H", "")
    add(vt.record("empty_arrays", 0, 0, 79, 1, [(1, 0)], -1, -1, 0, "T", None, empt),
        b'{"qname":"empty_arrays","flag":0,"rname":"c1","pos":80,"mapq":1,"cigar":"1M","rnext":"*","pnext":0,"tlen":0,"seq":"T","qual":[30],'
        b'"tags":{"Ec":[],"EC":[],"Es":[],"ES":[],"Ei":[],"EI":[],"Ef":[],"EZ":"","EH":""}}')
    add(vt.record("on_w", 0, 1, 4, 60, [(2, 0)], 1, 4, 0, "AC"),
        b'{"qname":"on_w","flag":0,"rname":"w\\/\\"\\\\\\t\x01\xe9","pos":5,"mapq":60,"cigar":"2M","rnext":"=","pnext":5,"tlen":0,"seq":"AC","qual":[30,30],"tags":{}}', ok=False)
    add(vt.record("mate_c1", 0x41, 2, 4, 60, [(2, 4), (3, 0), (1, 1)], 0, 999, 0, "ACGTAC"),
        b'{"qname":"mate_c1","flag":65,"rname":"c\\/3\\"\\\\","pos":5,"mapq":60,"cigar":"2S3M1I","rnext":"c1","pnext":1000,"tlen":0,"seq":"ACGTAC",'
        b'"qual":[30,30,30,30,30,30],"tags":{}}')
    add(vt.record("unplaced", 4, -1, -1, 0, [], -1, -1, 0, "ACGT", None, vt.tag("RG", "Z", "g1")),
        b'{"qname":"unplaced","flag":4,"rname":"*","pos":0,"mapq":0,"cigar":"*","rnext":"*","pnext":0,"tlen":0,"seq":"ACGT","qual":[30,30,30,30],"tags":{"RG":"g1"}}')
    add(vt.record("unplaced_mate", 0x45, -1, -1, 0, [], 1, 9, 0, "A"),
        b'{"qname":"unplaced_mate","flag":69,"rname":"*","pos":0,"mapq":0,"cigar":"*","rnext":"w\\/\\"\\\\\\t\x01\xe9","pnext":10,"tlen":0,"seq":"A","qual":[30],"tags":{}}', ok=False)
    return R, b"".join(x + b"\n" for x in L), valid


def write_edge_bam(path):
    recs, text, _ = edge_records()
    p = helpers.write_bgzf(path, bam_body(EDGE_REFS, recs), len(EDGE_REFS))
    with open(p + ".bai", "wb") as f:
        f.write(helpers.oracle_build_bai(p))
    return p, text
