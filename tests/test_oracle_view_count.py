"""The CPU restatement of `sambamba view -c` (tools/view_count_oracle.c) pinned against hand-written expectations: the state machine on merged
regions, positional regions with repeats, '*', BedFilter on an unsorted file, the flag bits and the subsampling hash."""
import pytest

import helpers
import view_count_common as vc

pytestmark = pytest.mark.timeout(300)


@pytest.fixture(scope="module")
def edge(tmp_path_factory):
    d = tmp_path_factory.mktemp("vco")
    return {"sorted": vc.write_edge_bam(str(d / "s.bam")), "unsorted": vc.write_edge_bam(str(d / "u.bam"), sorted_file=False), "dir": d}


BED = [(0, 500, 600), (0, 200, 300), (0, 100, 200)]      # any order; [100, 200) and [200, 300) touch: one merged region


def test_whole_file_and_flag_bits(edge):
    for k in ("sorted", "unsorted"):
        p = edge[k]
        assert vc.oracle_count(p) == 11
        assert vc.oracle_count(p, num_filter=(0, 4)) == 7               # not unmapped
        assert vc.oracle_count(p, num_filter=(1, 0)) == 3               # paired
        assert vc.oracle_count(p, num_filter=(1, 4)) == 1
        assert vc.oracle_count(p, num_filter=(0x410, 0)) == 0


def test_merged_regions_state_machine(edge):
    """reaches_100, zero_at_150 (strictly inside), unmapped_at_150 and two_regions (once, although it reaches both merged regions);
    not ends_at_100, zero_at_100 (at the start), unmapped_at_100, at_600."""
    p = edge["sorted"]
    assert vc.oracle_count(p, bed=BED) == 4
    assert vc.oracle_count(p, bed=BED + [(1, 149, 150)]) == 5            # spliced [40, 150) reaches 149
    assert vc.oracle_count(p, bed=BED + [(1, 150, 151)]) == 4
    assert vc.oracle_count(p, bed=[(0, 100, 101)]) == 1                  # only reaches_100: zero_at_100 and unmapped_at_100 sit at the start
    assert vc.oracle_count(p, bed=[]) == 0


def test_bedfilter_on_unsorted_file(edge):
    p = edge["unsorted"]
    assert vc.oracle_count(p, bed=BED) == 4
    assert vc.oracle_count(p, bed=list(reversed(BED + [(1, 149, 150)]))) == 5
    with pytest.raises(RuntimeError):
        vc.oracle_count(p, bed=[])


def test_positional_regions_repeats_and_star(edge):
    p = edge["sorted"]
    a, b = (0, 100, 200), (0, 150, 300)
    assert vc.oracle_count(p, regions=[a]) == 3
    assert vc.oracle_count(p, regions=[b]) == 1
    assert vc.oracle_count(p, regions=[a, b, a]) == 7                    # a read in k of the regions counts k times
    assert vc.oracle_count(p, regions=[a, b, a], n_unmapped=1) == 9
    assert vc.oracle_count(p, n_unmapped=2) == 4
    assert vc.oracle_count(p, regions=[(0, 0, 10000)]) == 8
    assert vc.oracle_count(p, regions=[(1, 40, 41)]) == 1
    with pytest.raises(RuntimeError, match="start must be less than end"):
        vc.oracle_count(p, regions=[(0, 5, 5)])


def test_fnv1a_hash_and_subsample(edge):
    assert vc.fnv1a(b"", 0) == vc.oracle_hash(b"", 0)
    assert vc.oracle_hash(b"read1", 42) == vc.fnv1a(b"read1", 42) == 0x73B4A4D270E26536
    assert vc.oracle_hash(b"SRR062634.1234", 0x0123456789ABCDEF) == vc.fnv1a(b"SRR062634.1234", 0x0123456789ABCDEF)
    u = helpers.oracle_inflate(edge["sorted"])
    import test_emul_filter as tef
    _, recs = tef.parse_all(u)
    for frac in (0.0, 0.25, 0.5, 0.9, 1.0, 2.0):
        for seed in (0, 1, 12345678901234567):
            want = sum(1 for r in recs if vc.fnv1a(r.name, seed) & 0xFFFFFFFF < vc.threshold(frac))
            assert vc.oracle_count(edge["sorted"], subsample=frac, seed=seed) == want
    assert vc.oracle_count(edge["sorted"], subsample=1.0, seed=3) == 11 and vc.oracle_count(edge["sorted"], subsample=0.0, seed=3) == 0


def test_subsample_threshold_conversion():
    """(0x100000000 * frac).to!ulong: a negative product (and NaN, which fails the same test) is 'Conversion negative overflow', one past
    ulong.max 'Conversion positive overflow'; -0.0 is 0."""
    assert vc.threshold(0.5) == 1 << 31 and vc.threshold(-0.0) == 0 and vc.threshold(1e-12) == 0
    with pytest.raises(ValueError, match="negative overflow"):
        vc.threshold(-1e-300)
    with pytest.raises(ValueError, match="negative overflow"):
        vc.threshold(float("nan"))
    with pytest.raises(ValueError, match="positive overflow"):
        vc.threshold(float("inf"))


def test_oracle_cli(edge):
    p = edge["sorted"]
    d = edge["dir"]
    bed = d / "t.bed"
    bed.write_text("c1\t500\t600\nnochr\t1\t5\nc1 200 300\nc1\t100\t200\n")
    assert vc.oracle_cli(["-c", "-L", str(bed), p]) == (0, b"4\n", b"")
    assert vc.oracle_cli(["-c", "-L", str(bed), str(edge["unsorted"])]) == (0, b"4\n", b"")
    assert vc.oracle_cli(["-c", p, "c1:101-200", "c1:151-300", "c1:101-200", "*"]) == (0, b"9\n", b"")
    assert vc.oracle_cli(["-c", "--num-filter=/4", p]) == (0, b"7\n", b"")
    assert vc.oracle_cli(["-c", "-L", str(bed), p, "c1"]) == (1, b"", b"sambamba-view: specifying both region and BED filename is disallowed\n")
    assert vc.oracle_cli(["-c", p, "c9:1-5"]) == (1, b"", b"sambamba-view: Reference with name c9 does not exist\n")
    assert vc.oracle_cli(["-c", p, "c1:10-5"]) == (1, b"", b"sambamba-view: start must be less than end\n")
    assert vc.oracle_cli(["-c", "-s", "-0.5", p]) == (1, b"", b"sambamba-view: Conversion negative overflow\n")
    assert vc.oracle_cli(["-c", "--num-filter=x", p]) == (1, b"", b"sambamba-view: Unexpected 'x' when converting from type string to type ushort\n")
