"""Shared pieces of the `view -f bam` tests: the oracle (tools/view_count_oracle.c, view_bam_oracle) through ctypes, and a reader that splits a
BGZF file into its members and checks each member's frame (header fields, BSIZE, CRC32, ISIZE)."""
import ctypes as C
import os
import struct
import zlib

import view_count_common as vc

UNMAPPED = 0xFFFFFFFF
BGZF_EOF = bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0, 27, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0])
HEADER_START = bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0])
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(vc.ORACLE_LIB)
        _lib.view_bam_oracle.argtypes = [C.c_char_p, C.c_uint, C.c_uint, C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(C.c_uint32), C.c_size_t,
                                         C.c_char_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_void_p),
                                         C.POINTER(C.c_size_t), C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        _lib.view_text_oracle_free.argtypes = [C.c_void_p]
        _lib.view_count_oracle_error.restype = C.c_char_p
    return _lib


def _bytes_at(p, n):
    """n bytes at p (C.string_at takes an int length: files of 2 GB and more do not fit it)."""
    return (C.c_char * n).from_address(p.value).raw if n else b""


def oracle_bam(path, header_text, level=-1, num_filter=(0, 0), subsample=None, seed=0, bed=None, regions=None, valid=False):
    """(uncompressed stream, [member sizes], finished file) of `sambamba view -f bam`; the keywords are BDepth.run_view_bam's."""
    L = _L()
    ht = header_text.encode() if isinstance(header_text, str) else bytes(header_text)
    rg = bed if bed is not None else (regions or [])
    rg = [(UNMAPPED, 0, 0) if r == "*" else r for r in rg]
    flat = (C.c_uint32 * max(3 * len(rg), 1))(*[v for r in rg for v in r])
    mode = 1 if bed is not None else (2 if rg else 0)
    raw, rl, ms, nm, f, fl = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t()
    L.view_count_oracle_set_valid(1 if valid else 0)
    rc = L.view_bam_oracle(os.fsencode(path), num_filter[0], num_filter[1], 0 if subsample is None else 1, 0 if subsample is None else vc.threshold(subsample),
                           seed, mode, flat, len(rg), ht, len(ht), level, C.byref(raw), C.byref(rl), C.byref(ms), C.byref(nm), C.byref(f), C.byref(fl))
    L.view_count_oracle_set_valid(0)
    if rc:
        raise RuntimeError(L.view_count_oracle_error().decode())
    out = (_bytes_at(raw, rl.value), list((C.c_uint32 * nm.value).from_address(ms.value)) if nm.value else [], _bytes_at(f, fl.value))
    for p in (raw, ms, f):
        L.view_text_oracle_free(p)
    return out


def members(data):
    """The members of a BGZF file as (raw DEFLATE data, inflated bytes); asserts every frame field on the way and the trailing EOF member."""
    assert data.endswith(BGZF_EOF), "no BGZF EOF member at the end"
    out, o, body = [], 0, data[:-len(BGZF_EOF)]
    while o < len(body):
        assert body[o:o + 16] == HEADER_START, "member header at %d" % o
        bsize = struct.unpack_from("<H", body, o + 16)[0] + 1
        d = body[o + 18:o + bsize - 8]
        crc, isize = struct.unpack_from("<II", body, o + bsize - 8)
        u = zlib.decompressobj(-15)
        x = u.decompress(d)
        assert u.eof and not u.unused_data, "member at %d: DEFLATE stream does not end with the member" % o
        assert len(x) == isize and zlib.crc32(x) == crc, "member at %d: ISIZE / CRC32" % o
        out.append((d, x))
        o += bsize
    return out


def check_against_oracle(got, want_raw, want_sizes, want_file, level):
    """got (a finished file) has the oracle's member sizes, members, frames and EOF; at level 0 it is the oracle's file byte for byte."""
    ms = members(got)
    assert [len(x) for _, x in ms] == want_sizes
    assert b"".join(x for _, x in ms) == want_raw
    if level == 0:
        assert got == want_file
