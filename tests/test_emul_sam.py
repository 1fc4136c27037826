"""The SAM formatter of kernels.cuh (sam_line through k_sam_len, the offset scan and k_sam_write; the %g routine sam_fmt_g) compiled for the host
against the CUDA-on-CPU emulation (tests/emul/emul_sam.cpp), compared with the CPU restatement (tools/view_count_oracle.c) on seeded random
records and with the C library's snprintf("%g") on float bit patterns spread over the whole range."""
import ctypes as C
import os
import random
import struct

import pytest

import flagstat_common as fc
import helpers
import view_text_common as vt

LIB = os.path.join(helpers.ROOT, "tests", "emul", "libemul_sam.so")
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
        _lib.emul_sam_format.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.c_int,
                                         C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        _lib.emul_fmt_g.argtypes = [C.c_uint32, C.c_char_p]
        _lib.emul_fmt_g.restype = C.c_uint32
        _lib.emul_check_g.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint32)]
        _lib.emul_check_g.restype = C.c_uint64
    return _lib


def emul_format(recs, refs):
    """The device formatter's text for the records (block_size included) and reference names."""
    body = b"".join(recs)
    offs, o = [], 0
    for r in recs:
        offs.append(o + 4)
        o += len(r)
    names = "".join(n for n, _ in refs).encode()
    noff, a = [], 0
    for n, _ in refs:
        noff.append(a)
        a += len(n)
    noff.append(a)
    cap = len(body) * 4 + 4096
    out = C.create_string_buffer(cap)
    n = C.c_size_t()
    rc = _L().emul_sam_format(body, len(body), (C.c_int64 * max(len(offs), 1))(*offs), len(offs), names, (C.c_uint32 * len(noff))(*noff), len(refs), out, cap, C.byref(n))
    return rc, out.raw[:n.value]


REFS = [("chr1", 1 << 30), ("a_rather_long_reference_name_to_cross_a_warp_of_lanes_" + "x" * 20, 5000), ("c", 10)]


def random_record(rnd):
    nr = len(REFS)
    ref = rnd.randrange(-1, nr)
    name = "".join(rnd.choice("ABCxyz:_0123456789") for _ in range(rnd.choice([0, 1, 5, 31, 32, 33, 100, 254])))
    cigar = [(rnd.randrange(0, 1 << 28) if rnd.random() < 0.1 else rnd.randrange(1, 300), rnd.randrange(0, 16)) for _ in range(rnd.choice([0, 1, 3, 31, 32, 33, 70]))]
    n = rnd.choice([0, 1, 2, 31, 32, 33, 64, 151, 300])
    qual = bytes(rnd.randrange(0, 256) for _ in range(n))
    if n and rnd.random() < 0.2:
        qual = b"\xff" + qual[1:]
    lim = {"c": (-128, 127), "C": (0, 255), "s": (-32768, 32767), "S": (0, 65535), "i": (-(1 << 31), (1 << 31) - 1), "I": (0, (1 << 32) - 1), "f": (0, (1 << 32) - 1)}
    aux = b""
    for _ in range(rnd.choice([0, 1, 3, 8])):
        k, t = rnd.choice(["NM", "XA", "ZZ", "a1"]), rnd.choice("AcCsSiIfZHB")
        if t == "A":
            aux += vt.tag(k, "A", chr(rnd.randrange(33, 127)))
        elif t in lim:
            aux += vt.tag(k, t, rnd.choice([lim[t][0], lim[t][1], 0, rnd.randint(*lim[t])]))
        elif t in "ZH":
            aux += vt.tag(k, t, "".join(rnd.choice("ABCDEF0123456789 xyz") for _ in range(rnd.choice([0, 1, 31, 32, 33, 100]))))
        else:
            et = rnd.choice("cCsSiIf")
            aux += vt.tag(k, "B", (et, [rnd.randint(*lim[et]) for _ in range(rnd.choice([0, 1, 31, 32, 33, 70]))]))
    if rnd.random() < 0.05:
        aux += b"Q"                                          # a stray trailing byte: ignored
    return vt.record(name, rnd.randrange(0, 1 << 16), ref, rnd.choice([-1, 0, rnd.randrange(0, 1 << 31), 0x7FFFFFFF]), rnd.randrange(0, 256), cigar,
                     rnd.choice([ref, -1, rnd.randrange(-1, nr)]), rnd.choice([-1, 0x7FFFFFFF, rnd.randrange(-1, 1 << 31)]),
                     rnd.choice([0, -(1 << 31), (1 << 31) - 1, rnd.randrange(-(1 << 31), 1 << 31)]), "".join(rnd.choice("=ACMGRSVTWYHKDBN") for _ in range(n)),
                     qual, aux, bin_=rnd.randrange(0, 1 << 16))


def test_random_records_against_the_oracle(tmp_path):
    rnd = random.Random(20261016)
    total = 0
    for part in range(4):                                   # 4 x 25,000 records
        recs = [random_record(rnd) for _ in range(25000)]
        p = helpers.write_bgzf(str(tmp_path / ("r%d.bam" % part)), fc.bam_body(REFS, recs), len(REFS))
        want = vt.oracle_text(p)
        rc, got = emul_format(recs, REFS)
        assert rc == 0
        if got != want:
            g, w = got.split(b"\n"), want.split(b"\n")
            i = next(i for i in range(min(len(g), len(w))) if g[i] != w[i])
            pytest.fail("line %d differs:\n%r\n%r" % (i, g[i][:400], w[i][:400]))
        total += len(recs)
    assert total >= 100000


def test_edge_lines_and_malformed_records():
    recs, want = vt.edge_records()
    assert emul_format(recs, vt.EDGE_REFS) == (0, want)
    codes = {"ref": 1, "mate_ref": 2, "tag_type": 3, "b_type": 4, "no_nul": 5, "tag_overrun": 6, "b_overrun": 6, "key_only": 6}
    for what, rec in vt.malformed_records():
        assert emul_format([recs[0], rec], vt.EDGE_REFS)[0] == codes[what], what


def _g(bits):
    b = C.create_string_buffer(32)
    n = _L().emul_fmt_g(bits, b)
    return b.raw[:n].decode()


def test_fmt_g_curated():
    for bits, s in vt.EDGE_FLOATS:
        assert _g(bits) == s, hex(bits)
    bad = C.c_uint32()
    for k in range(-45, 39):                                 # the neighbours of every power of ten and of every power of two
        b = struct.unpack("<I", struct.pack("<f", float("1e%d" % k)))[0]
        assert _L().emul_check_g((b - 3) & 0xFFFFFFFF, 1, 7, C.byref(bad)) == 0, hex(bad.value)
    for e in range(256):
        assert _L().emul_check_g(((e << 23) - 2) & 0xFFFFFFFF, 1, 5, C.byref(bad)) == 0, hex(bad.value)


def test_fmt_g_spread_over_all_floats():
    """2^24 bit patterns with a stride of 257 cover every exponent, both signs and NaNs, and many mantissas of each.  (emul_check_g(0, 1, 1 << 32)
    compares all 2^32 patterns: minutes per 2^30 of them on one CPU.)"""
    bad = C.c_uint32()
    n = _L().emul_check_g(0x5A5A5A5A, 257, 1 << 24, C.byref(bad))
    assert n == 0, "%d patterns differ from snprintf, the first %#x" % (n, bad.value)
