"""The JSON formatter of kernels.cuh (json_line through k_json_len, the offset scan and k_json_write) compiled for the host against the
CUDA-on-CPU emulation (tests/emul/emul_json.cpp), compared with the CPU restatement of toJson (tools/view_count_oracle.c) on
seeded random records weighted towards escaped bytes, raw control and high bytes, and infinite and NaN floats."""
import ctypes as C
import os
import random
import struct

import pytest

import helpers
import view_json_common as vj
import view_text_common as vt

LIB = os.path.join(helpers.ROOT, "tests", "emul", "libemul_json.so")
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
        _lib.emul_json_format.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.c_int,
                                          C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    return _lib


def emul_format(recs, refs):
    """The device formatter's JSON text for the records (block_size included) and reference names (bytes), the names quoted and escaped as
    the library uploads them."""
    body = b"".join(recs)
    offs, o = [], 0
    for r in recs:
        offs.append(o + 4)
        o += len(r)
    q = [vj.quote(n) for n, _ in refs]
    noff, a = [], 0
    for n in q:
        noff.append(a)
        a += len(n)
    noff.append(a)
    cap = len(body) * 8 + 4096
    out = C.create_string_buffer(cap)
    n = C.c_size_t()
    rc = _L().emul_json_format(body, len(body), (C.c_int64 * max(len(offs), 1))(*offs), len(offs), b"".join(q), (C.c_uint32 * len(noff))(*noff), len(refs),
                               out, cap, C.byref(n))
    return rc, out.raw[:n.value]


REFS = [(b"chr1", 1 << 30), (b"a/rather\\long \"reference\" name to cross a warp of lanes\t" + b"x" * 20, 5000), (b"c\x01\x7f\x80\xff", 10)]
SPECIAL = b'"\\/\b\t\n\f\r'                                   # the escaped bytes
NAME_BYTES = SPECIAL * 4 + b"\x01\x1f\x7f\x80\xe9\xff" + b"ABCxyz:_0123456789"
FLOATS = [0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x80000000, 0, 0x00000001, 0x7F7FFFFF]


def rbytes(rnd, n, alphabet):
    return bytes(rnd.choice(alphabet) for _ in range(n))


def random_record(rnd):
    nr = len(REFS)
    ref = rnd.randrange(-1, nr)
    name = rbytes(rnd, rnd.choice([0, 1, 5, 31, 32, 33, 100, 254]), NAME_BYTES)
    cigar = [(rnd.randrange(0, 1 << 28) if rnd.random() < 0.1 else rnd.randrange(1, 300), rnd.randrange(0, 16)) for _ in range(rnd.choice([0, 1, 3, 33]))]
    n = rnd.choice([0, 1, 2, 31, 32, 33, 64, 151, 300])
    qual = bytes(rnd.choice([rnd.randrange(0, 256), 0, 9, 10, 99, 100, 255]) for _ in range(n))
    if n and rnd.random() < 0.2:
        qual = b"\xff" * n
    lim = {"c": (-128, 127), "C": (0, 255), "s": (-32768, 32767), "S": (0, 65535), "i": (-(1 << 31) + 1, (1 << 31) - 1), "I": (0, (1 << 32) - 1),
           "f": (0, (1 << 32) - 1)}
    fval = lambda: rnd.choice(FLOATS) if rnd.random() < 0.5 else rnd.randrange(0, 1 << 32)      # noqa: E731
    aux = b""
    for _ in range(rnd.choice([0, 1, 3, 8])):
        k, t = rbytes(rnd, 2, b"NMXZa1" + SPECIAL + b"\x01\xe9"), rnd.choice("AcCsSiIfZHB")
        if t == "A":
            aux += vj.raw_tag(k, b"A", rbytes(rnd, 1, NAME_BYTES))
        elif t == "f":
            aux += vj.raw_tag(k, b"f", struct.pack("<I", fval()))
        elif t in lim:
            aux += k + vt.tag("XX", t, rnd.choice([lim[t][0], lim[t][1], 0, rnd.randint(*lim[t])]))[2:]
        elif t in "ZH":
            aux += vj.raw_tag(k, t.encode(), rbytes(rnd, rnd.choice([0, 1, 31, 32, 33, 100]), NAME_BYTES))
        else:
            et = rnd.choice("cCsSiIf")
            vals = [fval() if et == "f" else rnd.randint(*lim[et]) for _ in range(rnd.choice([0, 1, 31, 32, 33, 70]))]
            aux += k + vt.tag("XX", "B", (et, vals))[2:]
    if rnd.random() < 0.05:
        aux += b"Q"                                          # a stray trailing byte: ignored
    rec = bytearray(vt.record("x" * len(name), rnd.randrange(0, 1 << 16), ref, rnd.choice([-1, 0, rnd.randrange(0, 1 << 31), 0x7FFFFFFE]), rnd.randrange(0, 256),
                              cigar, rnd.choice([ref, -1, rnd.randrange(-1, nr)]), rnd.choice([-1, 0x7FFFFFFE, rnd.randrange(-1, 1 << 31)]),
                              rnd.choice([0, -(1 << 31) + 1, (1 << 31) - 1, rnd.randrange(-(1 << 31) + 1, 1 << 31)]), "".join(rnd.choice("=ACMGRSVTWYHKDBN") for _ in range(n)),
                              qual, aux, bin_=rnd.randrange(0, 1 << 16)))
    rec[36:36 + len(name)] = name
    return bytes(rec)


def test_random_records_against_the_oracle(tmp_path):
    """INT32_MIN stays out of the integers: it is the one stated deviation from BioD's itoa (DESIGN.md section 8), and the oracle prints it as
    the device does."""
    rnd = random.Random(20261017)
    total = 0
    for part in range(4):                                   # 4 x 25,000 records
        recs = [random_record(rnd) for _ in range(25000)]
        p = helpers.write_bgzf(str(tmp_path / ("r%d.bam" % part)), vj.bam_body(REFS, recs), len(REFS))
        want = vj.oracle_json(p)
        rc, got = emul_format(recs, REFS)
        assert rc == 0
        if got != want:
            g, w = got.split(b"\n"), want.split(b"\n")
            i = next(i for i in range(min(len(g), len(w))) if g[i] != w[i])
            pytest.fail("line %d differs:\n%r\n%r" % (i, g[i][:400], w[i][:400]))
        assert got.count(b"\n") == len(recs)
        total += len(recs)
    assert total >= 100000


def test_int32_min_prints_as_the_sam_line_does():
    """tlen, pnext = INT32_MAX + 1, an i tag and a B:i element at INT32_MIN: -2147483648, as in the SAM line (see the docstring above)."""
    r = vt.record("m", 0, 0, 5, 1, [(1, 0)], 0, 0x7FFFFFFF, -(1 << 31), "A", None, vt.tag("Xi", "i", -(1 << 31)) + vt.tag("Bi", "B", ("i", [-(1 << 31)])))
    rc, got = emul_format([r], REFS)
    assert rc == 0 and got == (b'{"qname":"m","flag":0,"rname":"chr1","pos":6,"mapq":1,"cigar":"1M","rnext":"=","pnext":-2147483648,"tlen":-2147483648,'
                               b'"seq":"A","qual":[30],"tags":{"Xi":-2147483648,"Bi":[-2147483648]}}\n')


def test_edge_lines_and_malformed_records():
    recs, want, _ = vj.edge_records()
    assert emul_format(recs, vj.EDGE_REFS) == (0, want)
    codes = {"ref": 1, "mate_ref": 2, "tag_type": 3, "b_type": 4, "no_nul": 5, "tag_overrun": 6, "b_overrun": 6, "key_only": 6}
    for what, rec in vt.malformed_records():
        assert emul_format([recs[0], rec], vj.EDGE_REFS)[0] == codes[what], what
