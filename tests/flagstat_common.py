"""Shared pieces of the flagstat tests: the binding of the CPU restatement (tools/flagstat_oracle.c, TEST INFRASTRUCTURE) and a
hand-made BAM whose records reach every category of computeFlagStatistics (sambamba/flagstat.d:31-57) in both QC classes."""
import ctypes as C
import os
import struct
import subprocess

import helpers

FIELDS = ("total", "secondary", "supplementary", "duplicates", "mapped", "paired", "read1", "read2", "proper_pair", "both_mapped",
          "singletons", "mate_diff_chr", "mate_diff_chr_mapq5")
ORACLE_LIB = os.path.join(helpers.ROOT, "tools", "_build", "libflagstat_oracle.so")
ORACLE_EXE = os.path.join(helpers.ROOT, "tools", "_build", "flagstat_oracle")

_lib = None


def oracle_flagstat(path):
    """{category: (QC-passed, QC-failed)} from the C restatement."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(ORACLE_LIB)
        _lib.oracle_flagstat.argtypes = [C.c_char_p, C.POINTER(C.c_uint64)]
        _lib.oracle_flagstat_error.restype = C.c_char_p
    out = (C.c_uint64 * 26)()
    if _lib.oracle_flagstat(os.fsencode(path), out) != 0:
        raise RuntimeError(_lib.oracle_flagstat_error().decode())
    return {n: (out[2 * i], out[2 * i + 1]) for i, n in enumerate(FIELDS)}


def oracle_cli(args):
    r = subprocess.run([ORACLE_EXE, "flagstat"] + list(args), capture_output=True)
    return r.returncode, r.stdout, r.stderr


def record(ref, pos, mapq, flag, next_ref, next_pos=0, name="r", seq="ACGTACGTAC"):
    """One BAM record (block_size included) with real mate fields; a 10M CIGAR when the read has a position."""
    nm = name.encode() + b"\0"
    cigar = [(len(seq), 0)] if pos >= 0 else []
    code = {c: i for i, c in enumerate("=ACMGRSVTWYHKDBN")}
    packed = bytes((code[seq[i]] << 4) | (code[seq[i + 1]] if i + 1 < len(seq) else 0) for i in range(0, len(seq), 2))
    tlen = 0 if next_ref != ref or ref < 0 else next_pos - pos
    body = struct.pack("<iiIIiiii", ref, pos, (4680 << 16) | (mapq << 8) | len(nm), (flag << 16) | len(cigar), len(seq), next_ref, next_pos, tlen)
    body += nm + b"".join(struct.pack("<I", (l << 4) | op) for l, op in cigar) + packed + bytes([30] * len(seq))
    return struct.pack("<i", len(body)) + body


def bam_body(refs, records, sorted_header=False):
    text = ("@HD\tVN:1.6\tSO:coordinate\n" if sorted_header else "@HD\tVN:1.6\tSO:unsorted\n") + "".join(f"@SQ\tSN:{n}\tLN:{l}\n" for n, l in refs)
    out = b"BAM\1" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for n, l in refs:
        out += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l)
    return out + b"".join(records)


HAND_REFS = [("chrA", 100000), ("chrB", 50000)]


def hand_records():
    """Every category in both QC classes: each line below is written once as QC-passed and, for all but the last few, once more with
    flag 0x200 -- so the two classes differ.  Not coordinate-sorted; the unplaced reads (refID -1) come last."""
    P, PROPER, UNM, MUNM, REV, R1, R2, SEC, QCF, DUP, SUP = 0x1, 0x2, 0x4, 0x8, 0x10, 0x40, 0x80, 0x100, 0x200, 0x400, 0x800
    base = [
        (0, 500, 60, P | PROPER | R1, 0, 700),                  # a proper pair on one reference
        (0, 700, 60, P | PROPER | R2 | REV, 0, 500),
        (0, 900, 60, P | R1 | DUP, 0, 950),                     # duplicate
        (0, 100, 60, P | R1 | SEC, 1, 300),                     # paired + secondary: counted as secondary, never on the pair lines
        (0, 200, 60, P | R2 | SUP, 1, 300),                     # paired + supplementary: the same
        (0, 300, 60, P | SEC | SUP, 0, 10),                     # both: secondary wins (if / else if)
        (0, 1200, 60, P | PROPER | UNM | R1, 0, 1300),          # proper_pair on an unmapped read: not properly paired; its mate mapped: no singleton
        (0, 1300, 60, P | R2, 0, 1200),                         # mapped with a mapped mate
        (0, 1500, 60, P | MUNM | R1, 0, 1500),                  # singleton: mapped, mate unmapped
        (0, 1500, 0, P | UNM | R2, 0, 1500),                    # its mate: unmapped, mate mapped
        (0, 2000, 4, P | R1, 1, 4000),                          # mate on another reference, MAPQ 4
        (0, 2100, 5, P | R2, 1, 4100),                          # ... MAPQ 5
        (1, 4000, 60, P | R1 | REV, 0, 2000),                   # ... from the other side, MAPQ 60
        (1, 6000, 30, P | R1, -1, -1),                          # mate "mapped" by its flag but without a reference: ref_id != mate_ref_id as written
        (1, 7000, 60, 0, -1, -1),                               # single-end, mapped
        (1, 7100, 60, DUP, -1, -1),                             # single-end duplicate
        (1, 7200, 60, SUP, -1, -1),                             # single-end supplementary
        (-1, -1, 0, P | UNM | MUNM | R1, -1, -1),               # the unplaced tail: a pair with both reads unmapped
        (-1, -1, 0, P | UNM | MUNM | R2, -1, -1),
        (-1, -1, 0, UNM, -1, -1),
    ]
    extra = [(1, 8000, 60, P | PROPER | R1, 1, 8200), (1, 8200, 60, P | PROPER | R2, 1, 8000), (-1, -1, 0, UNM, -1, -1)]
    rows = [(r, q, m, f, nr, np_) for r, q, m, f, nr, np_ in base] + [(r, q, m, f | QCF, nr, np_) for r, q, m, f, nr, np_ in base[:-1]] + extra
    placed = [x for x in rows if x[0] >= 0]
    tail = [x for x in rows if x[0] < 0]
    return [record(r, q, m, f, nr, np_, name=f"h{i}") for i, (r, q, m, f, nr, np_) in enumerate(placed + tail)]


def write_hand_bam(path, block=0xFF00):
    return helpers.write_bgzf(path, bam_body(HAND_REFS, hand_records()), len(HAND_REFS), block=block)


def write_mapped_share(path, a, b):
    """b reads of which a are mapped (the rest unplaced and unmapped): the `mapped` line prints percent(a, b)."""
    recs = [record(0, 10 * i, 60, 0, -1, -1, name=f"m{i}") for i in range(a)] + [record(-1, -1, 0, 0x4, -1, -1, name=f"u{i}") for i in range(b - a)]
    return helpers.write_bgzf(path, bam_body([("c1", 100000)], recs), 1)
