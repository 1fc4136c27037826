"""The BGZF compressor of `view -f bam` (bgzf_deflate.cuh) and its member cut (kernels.cuh) compiled for the host against the CUDA-on-CPU
emulation (tests/emul/emul_bgzf.cpp): every member (random ones and the golden files' payloads) inflates under zlib to its input with zlib's CRC32, dynamic code lengths stay within 15 / 7
bits, level 0 is zlib's level 0 byte for byte, the compressed size stays within 1.10x of zlib level 6, and the cut agrees with the CPU
restatement (tools/view_count_oracle.c) with the state carried across sub-batch splits."""
import ctypes as C
import gzip
import os
import random
import struct
import zlib

import pytest

import helpers
import test_oracle_view_bam as tov
import view_bam_common as vb

LIB = os.path.join(helpers.ROOT, "tests", "emul", "libemul_bgzf.so")
L = 0xFF00
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
        _lib.emul_bgzf_compress.argtypes = [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_uint32, C.c_int, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32)]
        _lib.emul_bam_cut.argtypes = [C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint32)]
        _lib.emul_bam_cut.restype = C.c_uint32
    return _lib


def compress(mems, level, grid=8):
    n = len(mems)
    body = b"".join(mems)
    offs, o = [], 0
    for m in mems:
        offs.append(o)
        o += len(m)
    out, ol = C.create_string_buffer(n * 65536), (C.c_uint32 * n)()
    _L().emul_bgzf_compress(body, (C.c_uint64 * n)(*offs), (C.c_uint32 * n)(*[len(m) for m in mems]), n, level, grid, out, ol)
    raw = out.raw
    return [raw[i * 65536:i * 65536 + ol[i]] for i in range(n)]


def code_lengths(d):
    """(block type, max lit/len length, max distance length, max code-length-code length) of the one DEFLATE block in d."""
    bits = int.from_bytes(d, "little")
    pos = [0]

    def get(n):
        v = (bits >> pos[0]) & ((1 << n) - 1)
        pos[0] += n
        return v
    assert get(1) == 1
    t = get(2)
    if t != 2:
        return t, 0, 0, 0
    hlit, hdist, hclen = get(5) + 257, get(5) + 1, get(4) + 4
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    cl = [0] * 19
    for i in range(hclen):
        cl[order[i]] = get(3)
    codes, nxt, c = {}, {}, 0
    bl = [cl.count(n) if n else 0 for n in range(8)]
    for b in range(1, 8):
        c = (c + bl[b - 1]) << 1
        nxt[b] = c
    for s in range(19):
        if cl[s]:
            codes[(cl[s], nxt[cl[s]])] = s
            nxt[cl[s]] += 1
    lens = []
    while len(lens) < hlit + hdist:
        code, n = 0, 0
        while (n, code) not in codes:
            code = (code << 1) | get(1)
            n += 1
        s = codes[(n, code)]
        if s < 16:
            lens.append(s)
        elif s == 16:
            lens += [lens[-1]] * (3 + get(2))
        elif s == 17:
            lens += [0] * (3 + get(3))
        else:
            lens += [0] * (11 + get(7))
    return t, max(lens[:hlit]), max(lens[hlit:]), max(cl)


def check(mems, level):
    out = compress(mems, level)
    for m, r in zip(mems, out):
        assert r[:16] == vb.HEADER_START and struct.unpack_from("<H", r, 16)[0] == len(r) - 1
        d = r[18:-8]
        u = zlib.decompressobj(-15)
        assert u.decompress(d) == m and u.eof and not u.unused_data
        assert struct.unpack("<II", r[-8:]) == (zlib.crc32(m), len(m))
        if level == 0:
            assert d == zlib.compress(m, 0, -15)      # (one deflate call with Z_FINISH, as bgzfCompress makes it)
        else:
            t, mll, md, mcl = code_lengths(d)
            assert mll <= 15 and md <= 15 and mcl <= 7
    return out


def random_member(rnd):
    k = rnd.randrange(6)
    n = rnd.choice([1, 2, 3, 17, 255, 256, 257, 1000, rnd.randrange(1, 4000)])
    if k == 0:
        return bytes(rnd.randrange(256) for _ in range(n))
    if k == 1:
        return bytes([rnd.randrange(256)]) * n
    if k == 2:
        p = bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 20)))
        return (p * (n // len(p) + 1))[:n]
    if k == 3:
        a = bytes(rnd.choice(b"ACGT") for _ in range(rnd.randrange(1, 600)))
        return (a * (n // len(a) + 2))[rnd.randrange(len(a)):][:n]
    if k == 4:
        return bytes(rnd.choice(b"!#%&+-05:?AFK") for _ in range(n))
    return bytes(rnd.randrange(4) + 60 for _ in range(n))


def _check_slice(args):
    seed, n, level = args
    rnd = random.Random(seed)
    check([random_member(rnd) for _ in range(n)], level)
    return n


def test_round_trip_random_small():
    """25,000 seeded random members (random bytes, runs, short and long repeats, quality-like text) at level -1 and 2,000 at level 0, spread
    over the host's cores: every CTA under the emulation switches its 256 fibers at each barrier, about 30 ms a member."""
    import multiprocessing as mp
    jobs = [(s, 500, -1) for s in range(50)] + [(1000 + s, 500, 0) for s in range(4)]
    with mp.get_context("fork").Pool(max(1, min(len(jobs), os.cpu_count() or 1))) as pool:
        assert sum(pool.map(_check_slice, jobs, chunksize=1)) == 27000


def golden_members():
    mems = []
    for name in ("issue_204.bam", "mate_overlaps_1_3M_4M.bam", "issue225.bam"):
        u = gzip.open(os.path.join(helpers.GOLDEN, name)).read()
        mems += [u[i:i + L] for i in range(0, len(u), L)]
    return mems


def test_round_trip_large_and_ratio(tmp_path):
    rnd = random.Random(7)
    mems = golden_members()
    g = helpers.gen_bam(str(tmp_path / "g.bam"), "-r", "chrA:400000", "-n", 8000, "-s", 3, "-t", 2)
    u = gzip.open(g).read()
    mems += [u[i:i + L] for i in range(0, min(len(u), 8 * L), L)]
    mems += [bytes(rnd.randrange(256) for _ in range(L)), b"\0" * L, bytes(rnd.choice(b"ACGT") for _ in range(L))]
    out = check(mems, -1)
    ours = sum(len(r) for r in out)
    ref = 0
    for m in mems:
        ref += len(zlib.compress(m, 6, -15)) + 26
    print("compressed %d bytes, zlib level 6 %d: %.4fx" % (ours, ref, ours / ref))
    assert ours <= 1.10 * ref, (ours, ref, ours / ref)
    check(mems[-6:], 0)


def cut(batches, sizes):
    """The members of sizes split into sub-batches at the given cut points, with the state carried; plus the final open member."""
    P, cur = C.c_uint32(0), C.c_ulonglong(0)
    ms, i = [], 0
    for j in list(batches) + [len(sizes)]:
        part = sizes[i:j]
        mo, ml = (C.c_ulonglong * (3 * (P.value + sum(part)) // L + 8))(), (C.c_uint32 * (3 * (P.value + sum(part)) // L + 8))()
        n = _L().emul_bam_cut((C.c_uint32 * max(len(part), 1))(*part), len(part), C.byref(P), C.byref(cur), mo, ml)
        ms += [ml[k] for k in range(n)]
        i = j
    if P.value:
        ms.append(P.value)
    return ms


@pytest.mark.parametrize("sizes", [
    [L // 2, L // 2, 100], [L // 2, L // 2 + 1, 64], [L, 100], [100, L + 500, 64, 64], [3 * L + 70, 64], [100, 100, L - 150, 64],
    [1000] * 300, [L // 3] * 40, [L // 2 + 1] * 30, [5000, 0, 0, 70000, 0, 64, 64, 0, L, 0, 0, 200],
])
def test_cut_against_oracle(tmp_path, sizes):
    recs = [tov.sized(n, "r%d" % i) for i, n in enumerate(sizes) if n]
    raw, want, _ = tov.run(tmp_path, recs)
    want = want[1:]      # (the header member)
    rnd = random.Random(len(sizes))
    for splits in ([], [len(sizes) // 2], sorted(rnd.sample(range(1, len(sizes)), min(len(sizes) - 1, 5))), list(range(1, len(sizes)))):
        assert cut(splits, sizes) == want, splits
