"""Region queries stage only the BAI chunks of the regions (SURVEY 8a row a17: getGroupChunks,
randomaccessmanager.d:247-294 -> only those BGZF blocks are copied, inflated and scanned).  Results must equal the
whole-file oracle on every region, and narrow queries must touch a small part of the file."""
import os
import random

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    d = tmp_path_factory.mktemp("sparse")
    return helpers.gen_bam(str(d / "big.bam"), "-r", "chrA:3000000", "-r", "chrB:500", "-r", "chrC:1000000", "-r", "chrD:800000", "-n", 400000, "-s", 9, "-t", 8)


LIN0 = {0: 0, 1: 3000000, 2: 3000500, 3: 4000500}


def test_base_counts_of_narrow_windows(big):
    import sambamba_b200 as sb
    with sb.BDepth(big) as b:
        b.run_base(collect=False)
        total_blocks = b.stats()["n_blocks"]
    rnd = random.Random(2)
    windows = [(1000, 3000), (2_999_000, 3_000_700), (3_000_500 + 400_000, 3_000_500 + 420_000), (4_000_500 + 790_000, 4_000_500 + 800_000)]
    windows += [(s, s + rnd.randrange(50, 30000)) for s in (rnd.randrange(0, 4_700_000) for _ in range(6))]
    for wa, wb in windows:
        want, _ = helpers.oracle_counts(big, window=(wa, wb))
        with sb.BDepth(big) as b:
            got = b.run_base(window=(wa, wb))
            st = b.stats()
        assert np.array_equal(got, want), (wa, wb)
        assert st["n_blocks"] < 0.2 * total_blocks, (wa, wb, st["n_blocks"], total_blocks)       # sparse staging engaged
    # many scattered regions in one query (exome-like): several chunks, several segments per sub-batch
    with sb.BDepth(big) as b:
        regs = sorted({(0, s, s + 300) for s in (rnd.randrange(0, 2_990_000) for _ in range(60))} | {(3, s, s + 500) for s in (rnd.randrange(0, 790_000) for _ in range(20))})
        b.set_regions(regs)
        b.set_tuning(chunk_blocks=7)
        got = b.run_base()
        st = b.stats()
        b.set_regions([])
    full, _ = helpers.oracle_counts(big)
    mask = np.zeros(full.shape[1], bool)
    for r, s, e in regs:
        mask[LIN0[r] + s:LIN0[r] + e] = True
    assert np.array_equal(got[:, mask], full[:, mask])
    assert st["n_blocks"] < total_blocks


def test_cli_region_and_base_with_L_match_oracle(big, tmp_path):
    bed = tmp_path / "q.bed"
    rnd = random.Random(3)
    rows = sorted((c, s, s + rnd.randrange(20, 4000)) for c, s in ((rnd.choice(["chrA", "chrC", "chrD"]), rnd.randrange(0, 780_000)) for _ in range(40)))
    bed.write_text("".join(f"{c}\t{s}\t{e}\n" for c, s, e in rows) + "chrB\t0\t500\n")
    for args in (["region", "-L", "chrC:500000-501000", "-T", "5", "-T", "20", big], ["region", "-L", str(bed), "-T", "10", big],
                 ["base", "-L", "chrA:1,500,000-1,500,400", big], ["base", "-L", str(bed), "-c", "0", big], ["base", "-L", "chrD", "-q", "20", big]):
        rc1, out1, err1 = helpers.run_cli(args)
        rc2, out2, err2 = helpers.oracle_cli(args)
        assert rc1 == rc2 == 0, (args, err1, err2)
        assert out1 == out2, (args, out1[:300], out2[:300])


def test_foreign_index_falls_back_to_the_whole_file(big, tmp_path):
    # an index that does not describe the file must not change results (the reference only checks that one exists)
    import shutil
    import sambamba_b200 as sb
    other = helpers.gen_bam(str(tmp_path / "other.bam"), "-r", "chrA:3000000", "-r", "chrB:500", "-r", "chrC:1000000", "-r", "chrD:800000", "-n", 50000, "-s", 4, "-t", 2)
    p = str(tmp_path / "copy.bam")
    shutil.copy(big, p)
    shutil.copy(other + ".bai", p + ".bai")
    wa, wb = 1_200_000, 1_203_000
    want, _ = helpers.oracle_counts(big, window=(wa, wb))
    with sb.BDepth(p) as b:
        got = b.run_base(window=(wa, wb))
    assert np.array_equal(got, want)


def test_foreign_index_restarts_before_the_last_batch(tmp_path):
    # The index of the file's first ten reads bounds the counter window far too tightly: a read of the first sub-batch falls outside it and
    # the run starts over with the whole genome as its window, while later batches and sub-batches of the first run are still ahead.
    import sambamba_b200 as sb
    reads = [(0, 20 * i, 30, 0, [(40, 0)], "ACGTA" * 8, "r%d" % i) for i in range(4000)]
    p = helpers.write_bam(str(tmp_path / "f.bam"), [("r0", 90000)], reads, block=4096, bins="auto", index=False)
    head = helpers.write_bam(str(tmp_path / "head.bam"), [("r0", 90000)], reads[:10], block=4096, bins="auto", index=False)
    with sb.BDepth(head) as b:
        open(p + ".bai", "wb").write(b.build_index())
    want, _ = helpers.oracle_counts(p)
    with sb.BDepth(p) as b:
        b.set_tuning(1 << 16, 2)
        got = b.run_base()
        st = b.stats()
    assert np.array_equal(got, want) and st["n_batches"] > 1 and st["n_records"] == 4000, st


def test_lazy_open_frames_only_what_a_region_query_needs(big, tmp_path):
    """bdepth_open_lazy: a region query must not depend on BGZF members outside its BAI chunks.  A copy of the file whose
    LAST data member is damaged cannot be opened eagerly, but answers a query on its first reference when opened lazily --
    and reports the damage as soon as a run needs the whole file."""
    import sambamba_b200 as sb
    raw = bytearray(open(big, "rb").read())
    # walk the members to the last data block and break its magic
    off, last = 0, None
    while off + 18 <= len(raw):
        bsize = (raw[off + 16] | (raw[off + 17] << 8)) + 1
        isize = int.from_bytes(raw[off + bsize - 4:off + bsize], "little")
        if isize == 0:
            break
        last = off
        off += bsize
    raw[last] = 0x00
    bad = str(tmp_path / "bad.bam")
    open(bad, "wb").write(raw)
    open(bad + ".bai", "wb").write(open(big + ".bai", "rb").read())
    with pytest.raises(sb.BDepthError) as ei:
        sb.BDepth(bad)
    assert "wrong BGZF magic" in str(ei.value)
    want, _ = helpers.oracle_counts(big, window=(1000, 40000))
    with sb.BDepth(bad, lazy=True) as b:
        assert np.array_equal(b.run_base(window=(1000, 40000)), want)
        rows = b.run_regions([(0, 5000, 9000), (0, 200000, 201000)], [1, 10])
        with pytest.raises(sb.BDepthError) as ei:
            b.run_base(collect=False)              # the whole file: the rest is framed now
        assert "wrong BGZF magic" in str(ei.value)
    with sb.BDepth(big, lazy=True) as b, sb.BDepth(big) as e:
        assert b.run_regions([(0, 5000, 9000), (0, 200000, 201000)], [1, 10]) == rows == e.run_regions([(0, 5000, 9000), (0, 200000, 201000)], [1, 10])
        got = b.run_base(collect=False)            # lazily opened handles do whole-file runs too
        assert b.stats()["n_blocks"] == e.stats()["n_blocks"] or e.run_base(collect=False) is None and b.stats()["n_blocks"] == e.stats()["n_blocks"]
