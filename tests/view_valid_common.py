"""Shared pieces of the `view -v` tests: the binding of the CPU restatement of BioD's isValid (tools/view_count_oracle.c, TEST
INFRASTRUCTURE), hand-written records on both sides of each of its rules with the answer the reference gives, and a file that holds an invalid
read of each kind among valid ones."""
import contextlib
import ctypes as C
import struct

import view_count_common as vc
import view_text_common as vt

VALID, INVALID, REFUSED = 0, 1, 2
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(vc.ORACLE_LIB)
        _lib.view_valid_oracle.argtypes = [C.c_char_p, C.c_uint32]
        _lib.view_count_oracle_set_valid.argtypes = [C.c_int]
        _lib.view_count_oracle_error.restype = C.c_char_p
    return _lib


def oracle_valid(rec):
    """(VALID / INVALID / REFUSED, the refusal's reason) of one record, block_size included."""
    L = _L()
    v = L.view_valid_oracle(rec[4:], len(rec) - 4)
    return v, (L.view_count_oracle_error().decode() if v == REFUSED else "")


@contextlib.contextmanager
def valid_oracle():
    """-v for the oracle's count, text and JSON entry points inside the block."""
    _L().view_count_oracle_set_valid(1)
    try:
        yield
    finally:
        _L().view_count_oracle_set_valid(0)


# the SAM_ERR_* code of the library (kernels.cuh) for each refusal reason of the oracle
REFUSAL_CODE = {"unknown tag type": 3, "unknown B array element type": 4, "Z or H value without its NUL": 5, "tag runs past the record": 6,
                "B array runs past the record": 6}


def rec(aux=b"", name="r1", pos=10, cigar=((4, 0),), seq="ACGT", qual=None, ref=0, flag=0):
    return vt.record(name, flag, ref, pos, 60, list(cigar), -1, -1, 0, seq, qual, aux)


def raw_name(r, name):
    """r with its read name replaced by the bytes `name` (l_read_name = len(name) + 1; None: l_read_name 0, no name bytes at all)."""
    body = bytearray(r[4:])
    ln = body[8]
    new = b"" if name is None else bytes(name) + b"\0"
    body = body[:32] + new + body[32 + ln:]
    body[8] = len(new)
    return struct.pack("<i", len(body)) + bytes(body)


def t(key, ty, v):
    return vt.tag(key, ty, v)


def z(key, v, ty="Z"):
    """a Z / H tag with raw bytes"""
    return key.encode() + ty.encode() + bytes(v) + b"\0"


def many_tags(n, dup=None):
    keys = ["%s%s" % (chr(65 + i // 26), chr(97 + i % 26)) for i in range(n)]
    if dup:
        keys[dup[1]] = keys[dup[0]]
    return b"".join(t(k, "C", 1) for k in keys)


BIG = (1 << 28) - 1


def cases():
    """(what, record, VALID / INVALID / REFUSED), each rule's boundary from both sides."""
    C_ = [
        # 1. name
        ("l_read_name 0", raw_name(rec(), None), INVALID), ("l_read_name 1", raw_name(rec(), b""), INVALID),
        ("name with @", rec(name="a@b"), INVALID), ("name with space", rec(name="a b"), INVALID), ("name !", rec(name="!"), VALID),
        ("name ~", rec(name="~"), VALID), ("name 0x7F", raw_name(rec(), b"a\x7f"), INVALID), ("name 0x80", raw_name(rec(), b"a\x80"), INVALID),
        ("name 254 bytes", rec(name="n" * 254), VALID), ("name ?A", rec(name="?A~!"), VALID),
        # 2. position
        ("pos -2", rec(pos=-2), INVALID), ("pos -1", rec(pos=-1, ref=-1, flag=4), VALID), ("pos 2^29-2", rec(pos=(1 << 29) - 2), VALID),
        ("pos 2^29-1", rec(pos=(1 << 29) - 1), INVALID),
        # 3. qualities
        ("no qualities", rec(cigar=(), seq=""), VALID), ("all 0xFF", rec(qual=b"\xff" * 4), VALID), ("93", rec(qual=bytes([93, 0, 1, 93])), VALID),
        ("94", rec(qual=bytes([30, 94, 30, 30])), INVALID), ("0xFF and 30", rec(qual=bytes([255, 30, 255, 255])), INVALID),
        ("30 then 0xFF", rec(qual=bytes([30, 30, 30, 255])), INVALID), ("long all 0xFF", rec(cigar=((100, 0),), seq="A" * 100, qual=b"\xff" * 100), VALID),
        ("long with one 94", rec(cigar=((100, 0),), seq="A" * 100, qual=bytes([20] * 70 + [94] + [20] * 29)), INVALID),
        # 4. CIGAR
        ("HMH", rec(cigar=((1, 5), (4, 0), (1, 5))), VALID), ("MHM", rec(cigar=((2, 0), (1, 5), (2, 0))), INVALID),
        ("HSMSH", rec(cigar=((1, 5), (1, 4), (2, 0), (1, 4), (1, 5))), VALID), ("SMS", rec(cigar=((1, 4), (2, 0), (1, 4))), VALID),
        ("MSMS", rec(cigar=((1, 0), (1, 4), (1, 0), (1, 4))), INVALID), ("HSMSMH", rec(cigar=((1, 5), (1, 4), (1, 0), (1, 4), (1, 0), (1, 5))), INVALID),
        ("HS", rec(cigar=((1, 5), (4, 4))), VALID), ("SH", rec(cigar=((4, 4), (1, 5))), VALID), ("MH", rec(cigar=((4, 0), (1, 5))), VALID),
        ("HHM", rec(cigar=((1, 5), (1, 5), (4, 0))), INVALID), ("HMS H", rec(cigar=((1, 5), (2, 0), (2, 4), (1, 5))), VALID),
        ("length mismatch", rec(cigar=((3, 0),)), INVALID), ("length with S I = X", rec(cigar=((1, 4), (1, 1), (1, 7), (1, 8))), VALID),
        ("D N P do not count", rec(cigar=((2, 0), (5, 2), (5, 3), (5, 6), (2, 0))), VALID), ("l_seq 0", rec(cigar=((3, 0),), seq=""), VALID),
        ("empty CIGAR", rec(cigar=()), VALID), ("op 9", rec(cigar=((4, 0), (5, 9))), VALID), ("op 13 is not H", rec(cigar=((2, 0), (1, 13), (2, 0))), VALID),
        ("op 12 does not count", rec(cigar=((2, 0), (7, 12), (2, 1))), VALID), ("op 15 does not count", rec(cigar=((4, 0), (3, 15), (1, 0))), INVALID),
        ("sum wraps to l_seq", rec(cigar=[(BIG, 1)] * 16 + [(20, 0)]), VALID), ("sum wraps past l_seq", rec(cigar=[(BIG, 1)] * 16 + [(19, 0)]), INVALID),
        # 5. tags: each type's own rule
        ("H empty", rec(z("XH", b"", "H")), INVALID), ("H hex", rec(z("XH", b"0123456789abcdefABCDEF", "H")), VALID), ("H G", rec(z("XH", b"1G", "H")), INVALID),
        ("A !", rec(t("XA", "A", "!")), VALID), ("A ~", rec(t("XA", "A", "~")), VALID), ("A space", rec(t("XA", "A", " ")), INVALID),
        ("A 0x7F", rec(b"XAA\x7f"), INVALID), ("Z empty", rec(z("XZ", b"")), INVALID), ("Z space ~", rec(z("XZ", b" x~")), VALID),
        ("Z 0x7F", rec(z("XZ", b"a\x7fb")), INVALID), ("Z tab", rec(z("XZ", b"a\tb")), INVALID), ("Z 0x1F", rec(z("XZ", b"\x1f")), INVALID),
        ("f B and integers", rec(t("Xf", "f", 0x7FC00000) + t("XB", "B", ("f", [1])) + t("Xi", "I", 5)), VALID),
        # predefined keys
        ("NM:i", rec(t("NM", "i", 3)), VALID), ("NM:Z", rec(z("NM", b"3")), INVALID), ("NM:f", rec(t("NM", "f", 0)), INVALID),
        ("NM:A", rec(t("NM", "A", "3")), INVALID), ("AS:C", rec(t("AS", "C", 3)), VALID), ("UQ:B", rec(t("UQ", "B", ("c", [1]))), INVALID),
        ("H0:s", rec(t("H0", "s", -1)), VALID), ("TC:H", rec(z("TC", b"AB", "H")), INVALID),
        ("RG:Z", rec(z("RG", b"g1")), VALID), ("RG:i", rec(t("RG", "i", 1)), INVALID), ("RG:H", rec(z("RG", b"AB", "H")), INVALID),
        ("MD:A", rec(t("MD", "A", "4")), INVALID), ("BC:Z", rec(z("BC", b"ACGT")), VALID), ("PG:B", rec(t("PG", "B", ("C", [1]))), INVALID),
        ("FZ:B:S", rec(t("FZ", "B", ("S", [1, 2]))), VALID), ("FZ:B:s", rec(t("FZ", "B", ("s", [1, 2]))), INVALID), ("FZ:Z", rec(z("FZ", b"1")), INVALID),
        ("FZ:B:S empty", rec(t("FZ", "B", ("S", []))), VALID),
        ("OQ *", rec(z("OQ", b"*")), VALID), ("OQ with space", rec(z("OQ", b"II I")), INVALID), ("OQ", rec(z("OQ", b"IIII")), VALID),
        ("CQ with space", rec(z("CQ", b"a b")), INVALID), ("U2 *", rec(z("U2", b"*")), VALID), ("Q2 space only", rec(z("Q2", b" ")), INVALID),
        ("BQ l_seq", rec(z("BQ", b"@@@@")), VALID), ("BQ short", rec(z("BQ", b"@@@")), INVALID), ("BQ with space", rec(z("BQ", b"@ @@")), VALID),
        ("E2 l_seq", rec(z("E2", b"ACGT")), VALID), ("E2 short", rec(z("E2", b"ACG")), INVALID), ("E2 with space", rec(z("E2", b"AC T")), INVALID),
        ("E2 * is one byte", rec(z("E2", b"*")), INVALID),
        ("unknown key f", rec(t("XY", "f", 0)), VALID), ("MD empty", rec(z("MD", b"")), INVALID),
        # the first failing tag does not stop the walk: a later malformed tag still refuses
        ("bad tag then malformed", rec(z("XZ", b"\x01") + b"XXq\x01"), REFUSED), ("bad name and malformed", rec(b"XXq\x01", name="a@"), INVALID),
        ("bad CIGAR and malformed", rec(b"XXZabc", cigar=((3, 0),)), INVALID),
        # duplicate keys
        ("NM twice", rec(t("NM", "i", 1) + t("XA", "A", "a") + t("NM", "i", 1)), INVALID), ("XA XB", rec(t("XA", "i", 1) + t("XB", "i", 1)), VALID),
        ("300 keys", rec(many_tags(300)), VALID), ("300 keys, 299 = 0", rec(many_tags(300, (0, 299))), INVALID),
        ("300 keys, 280 = 260", rec(many_tags(300, (260, 280))), INVALID), ("300 keys, 255 = 0", rec(many_tags(300, (0, 255))), INVALID),
        ("300 keys, 256 = 3", rec(many_tags(300, (3, 256))), INVALID),
        ("300 keys then malformed", rec(many_tags(300) + b"XXZab"), REFUSED),
        ("key only", rec(b"XX"), REFUSED), ("one stray byte", rec(b"X"), VALID),
    ]
    for s in ("0", "10", "4A0", "2^AC2", "0A0C0", "1^A0", "100T0^GG3", "12Z0", "0^ABCDEFGHIJKLMNOPQRSTUVWXYZ0", "3A4^T5"):
        C_.append(("MD " + s, rec(z("MD", s.encode())), VALID))
    for s in ("A1", "1a1", "1^1", "1^", "1A", "^A1", "1 A1", "12-", "1AB2", "1^AB", "1A2 ", "x"):
        C_.append(("MD " + s, rec(z("MD", s.encode())), INVALID))
    ok = lambda aux: rec(aux)      # noqa: E731
    for what, bad, twin in (("tag type", b"XXq\x01", b"XXc\x01"), ("B type", b"XXBq\x01\0\0\0\x05", b"XXBc\x01\0\0\0\x05"),
                            ("no NUL", b"XXZabc", b"XXZabc\0"), ("tag overrun", b"XXi\x01\x02", b"XXs\x01\x02"),
                            ("B overrun", b"XXBi\x03\0\0\0\x01\0\0\0", b"XXBi\x01\0\0\0\x01\0\0\0"), ("type byte missing", b"XYZa\0XX", b"XYZa\0X")):
        C_.append(("refused: " + what, ok(bad), REFUSED))
        C_.append(("twin of " + what, ok(twin), VALID))
    return C_


def invalid_kinds():
    """One invalid read of each kind, and the refused ones, as (what, record) -- every record placed at pos 10 on reference 0."""
    return [(w, r) for w, r, v in cases() if v == INVALID and "pos" not in w and "l_read_name 0" != w]
