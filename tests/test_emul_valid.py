"""The validator of `view -v` (k_view_valid in kernels.cuh) compiled for the host against the CUDA-on-CPU emulation (tests/emul/emul_valid.cpp),
compared with the CPU restatement of BioD's isValid (tools/view_count_oracle.c) on the hand-written boundary records and on seeded random
records weighted towards the boundaries of each rule."""
import ctypes as C
import os
import random

import helpers
import view_valid_common as vv

LIB = os.path.join(helpers.ROOT, "tests", "emul", "libemul_valid.so")
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
        _lib.emul_view_valid.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.c_uint32, C.c_char_p]
    return _lib


def emul_status(recs):
    """k_view_valid's status of each record (block_size included): 0 valid, 255 invalid, else the SAM_ERR_* code."""
    body = b"".join(recs)
    offs, o = [], 0
    for r in recs:
        offs.append(o + 4)
        o += len(r)
    st = C.create_string_buffer(max(len(recs), 1))
    _L().emul_view_valid(body, len(body), (C.c_int64 * max(len(offs), 1))(*offs), len(recs), st)
    return list(st.raw[:len(recs)])


def oracle_status(r):
    v, why = vv.oracle_valid(r)
    return 0 if v == vv.VALID else 255 if v == vv.INVALID else vv.REFUSAL_CODE[why]


def test_boundary_records():
    cases = vv.cases()
    got = emul_status([r for _, r, _ in cases])
    for (what, r, want), g in zip(cases, got):
        assert g == oracle_status(r), what
        assert (g == 0) == (want == vv.VALID) and (g == 255) == (want == vv.INVALID), what


KEYS = ["AM", "AS", "NM", "MQ", "UQ", "RG", "BC", "MD", "OQ", "E2", "BQ", "CQ", "U2", "FZ", "PG", "XA", "XB", "xy", "H0"]
PRINT = bytes(range(0x21, 0x7F))


def random_aux(rnd, l_seq):
    aux = b""
    for _ in range(rnd.choice([0, 0, 1, 2, 4, 8, 40])):
        k = rnd.choice(KEYS)
        ty = rnd.choice("AcCsSiIfZZZZHHBB")
        if ty == "A":
            aux += k.encode() + b"A" + bytes([rnd.choice([0x20, 0x21, 0x7E, 0x7F, 0x41, rnd.randrange(256)])])
        elif ty in "cCsSiIf":
            aux += vv.t(k, ty, {"c": 1, "C": 200, "s": -3, "S": 60000, "i": -7, "I": 7, "f": 0x3F800000}[ty])
        elif ty == "Z":
            if k == "MD" or rnd.random() < 0.2:
                s = bytes(rnd.choice(b"0123456789" * 3 + b"ACGT^" + b"a -") for _ in range(rnd.choice([0, 1, 2, 3, 5, 9, 40])))
            elif rnd.random() < 0.3:
                s = rnd.choice([b"*", b"", b" ", bytes(rnd.choice(PRINT) for _ in range(l_seq)), bytes(rnd.choice(PRINT) for _ in range(max(l_seq - 1, 0)))])
            else:
                s = bytes(rnd.choice(PRINT + b" \t\x7f\x80") for _ in range(rnd.choice([1, 4, 31, 32, 33, 70])))
            aux += vv.z(k, s)
        elif ty == "H":
            aux += vv.z(k, bytes(rnd.choice(b"0123456789abcdefABCDEFgG") for _ in range(rnd.choice([0, 1, 2, 33]))), "H")
        else:
            et = rnd.choice("SSscC")
            aux += vv.t(k, "B", (et, [1] * rnd.choice([0, 1, 3])))
    r = rnd.random()
    if r < 0.01:
        aux += b"XXq\x01"
    elif r < 0.02:
        aux += b"XXBq\x01\0\0\0\x05"
    elif r < 0.03:
        aux += b"XXZabc"
    elif r < 0.04:
        aux += b"XXi\x01"
    elif r < 0.05:
        aux += b"XX"
    elif r < 0.06:
        aux += b"X"
    return aux


def random_record(rnd):
    l_seq = rnd.choice([0, 1, 4, 31, 32, 33, 100])
    n = rnd.choice([0, 1, 2, 3, 4, 5, 8, 40])
    ops = [rnd.choice([0, 0, 0, 1, 2, 3, 4, 4, 5, 5, 6, 7, 8, rnd.randrange(9, 16)]) for _ in range(n)]
    lens = [rnd.randrange(1, 6) for _ in range(n)]
    if n and rnd.random() < 0.6:                              # make the M/I/S/=/X lengths add up to l_seq
        q = [i for i, op in enumerate(ops) if op in (0, 1, 4, 7, 8)]
        if q:
            rest = l_seq - sum(lens[i] for i in q if i != q[-1])
            if rest > 0:
                lens[q[-1]] = rest
            elif rnd.random() < 0.3:
                lens[q[-1]] = (rest + (1 << 32)) % (1 << 28) or 1
    if n and rnd.random() < 0.02:                             # a length sum that wraps at 2^32
        ops, lens = [1] * 16 + [0], [(1 << 28) - 1] * 16 + [l_seq + 16]
    cigar = list(zip(lens, ops))
    if l_seq and rnd.random() < 0.3:
        qual = rnd.choice([b"\xff" * l_seq, bytes([93] * l_seq), bytes(rnd.choice([0, 30, 93, 94, 255]) for _ in range(l_seq))])
    else:
        qual = bytes(rnd.randrange(0, 94) for _ in range(l_seq))
    name = rnd.choice(["r", "read/1", "x" * 254, "a@b", "a b", "!~", "q" * 40])
    pos = rnd.choice([-2, -1, 0, 10, (1 << 29) - 2, (1 << 29) - 1])
    r = vv.rec(random_aux(rnd, l_seq), name=name, pos=pos, cigar=cigar, seq="ACGT" * (l_seq // 4) + "ACGT"[:l_seq % 4], qual=qual)
    x = rnd.random()
    if x < 0.01:
        r = vv.raw_name(r, None)
    elif x < 0.02:
        r = vv.raw_name(r, b"")
    elif x < 0.04:
        r = vv.raw_name(r, bytes([rnd.choice([0x20, 0x40, 0x7F, 0x80, 0xFF])]) + b"ab")
    return r


def test_random_records_against_the_oracle():
    rnd = random.Random(20261017)
    total, seen = 0, set()
    for part in range(4):                                    # 4 x 25,000 records
        recs = [random_record(rnd) for _ in range(25000)]
        got = emul_status(recs)
        for i, r in enumerate(recs):
            w = oracle_status(r)
            assert got[i] == w, "record %d of part %d: %d vs %d: %r" % (i, part, got[i], w, r[:200])
            seen.add(w)
        total += len(recs)
    assert total >= 100000 and seen == {0, 255, 3, 4, 5, 6}
