"""Shared pieces of the `view -c` tests: the binding of the CPU restatement (tools/view_count_oracle.c, TEST INFRASTRUCTURE) and a hand-made
file whose reads sit on the edges of the selection rules (zero-length reads at and inside region starts, a read reaching two merged regions,
unmapped reads with a position, the unplaced tail)."""
import ctypes as C
import os
import random
import subprocess

import flagstat_common as fc
import helpers

ORACLE_LIB = os.path.join(helpers.ROOT, "tools", "_build", "libview_count_oracle.so")
ORACLE_EXE = os.path.join(helpers.ROOT, "tools", "_build", "view_count_oracle")
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(ORACLE_LIB)
        _lib.view_count_oracle.argtypes = [C.c_char_p, C.c_uint, C.c_uint, C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(C.c_uint32), C.c_size_t,
                                           C.c_uint, C.POINTER(C.c_uint64)]
        _lib.view_count_oracle_error.restype = C.c_char_p
        _lib.view_count_oracle_hash.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64]
        _lib.view_count_oracle_hash.restype = C.c_uint64
    return _lib


def threshold(frac):
    import sambamba_b200._lib as SL
    return SL.subsample_threshold(frac)


def oracle_count(path, num_filter=(0, 0), subsample=None, seed=0, bed=None, regions=None, n_unmapped=0):
    """The same arguments as BDepth.run_view_count."""
    L = _L()
    rg = bed if bed is not None else (regions or [])
    flat = (C.c_uint32 * max(3 * len(rg), 1))(*[v for r in rg for v in r])
    mode = 1 if bed is not None else (2 if (rg or n_unmapped) else 0)
    out = C.c_uint64()
    rc = L.view_count_oracle(os.fsencode(path), num_filter[0], num_filter[1], 0 if subsample is None else 1, 0 if subsample is None else threshold(subsample),
                             seed, mode, flat, len(rg), n_unmapped, C.byref(out))
    if rc:
        raise RuntimeError(L.view_count_oracle_error().decode())
    return out.value


def oracle_hash(name, seed):
    return _L().view_count_oracle_hash(name, len(name), seed)


def oracle_cli(args):
    r = subprocess.run([ORACLE_EXE, "view"] + list(args), capture_output=True)
    return r.returncode, r.stdout, r.stderr


def fnv1a(name, seed):
    """SubsampleFilter.simpleHash (filtering.d:350-358), restated in Python."""
    h = 14695981039346656037
    for b in bytes(name) + int(seed).to_bytes(8, "little"):
        h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


REFS = [("c1", 10000), ("c2", 5000)]
INS, MATCH = 1, 0


def edge_reads():
    """(ref, pos, mapq, flag, cigar, seq, name), coordinate-sorted; the comments give the read's [pos, pos + basesCovered)."""
    def rd(ref, pos, flag, cigar, name, seq_len=10):
        return (ref, pos, 60, flag, cigar, "ACGT" * (seq_len // 4) + "ACGT"[:seq_len % 4], name)
    return [
        rd(0, 90, 0, [(10, MATCH)], "ends_at_100"),               # [90, 100)
        rd(0, 90, 0x10, [(11, MATCH)], "reaches_100"),            # [90, 101)
        rd(0, 100, 0, [(10, INS)], "zero_at_100"),                # zero-length at a region start
        rd(0, 100, 0x4, [(10, MATCH)], "unmapped_at_100"),        # unmapped: basesCovered 0
        rd(0, 150, 0x40, [(10, INS)], "zero_at_150"),             # zero-length inside a region
        rd(0, 150, 0x4 | 0x1, [(10, MATCH)], "unmapped_at_150"),
        rd(0, 250, 0x1 | 0x80, [(300, MATCH)], "two_regions", 300),   # [250, 550): reaches [100, 300) and [500, 600)
        rd(0, 600, 0x400, [(10, MATCH)], "at_600"),               # [600, 610)
        rd(1, 40, 0, [(5, MATCH), (100, 3), (5, MATCH)], "spliced"),   # [40, 150) on c2
        rd(-1, -1, 0x4, [], "tail_a"),
        rd(-1, -1, 0x4 | 0x1, [], "tail_b"),
    ]


def write_edge_bam(path, sorted_file=True):
    reads = edge_reads()
    if sorted_file:
        return helpers.write_bam(path, REFS, reads, bins="auto")
    recs = []
    for ref, pos, mapq, flag, cigar, seq, name in reads:
        rec = fc.record(ref, pos, mapq, flag, -1, -1, name=name, seq=seq)
        if cigar != [(len(seq), 0)]:                      # fc.record writes a plain match CIGAR: rebuild with the read's own
            import struct
            bs, = struct.unpack_from("<i", rec, 0)
            body = bytearray(rec[4:])
            l_name = body[8]
            n_old = struct.unpack_from("<I", body, 12)[0] & 0xFFFF
            cg = b"".join(struct.pack("<I", (l << 4) | op) for l, op in cigar)
            body[12:16] = struct.pack("<I", (flag << 16) | len(cigar))
            body = body[:32 + l_name] + cg + body[32 + l_name + 4 * n_old:]
            rec = struct.pack("<i", len(body)) + bytes(body)
        recs.append(rec)
    placed, tail = recs[:-2], recs[-2:]
    random.Random(7).shuffle(placed)
    return helpers.write_bgzf(path, fc.bam_body(REFS, placed + tail), len(REFS))
