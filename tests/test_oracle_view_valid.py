"""The CPU restatement of BioD's isValid (tools/view_count_oracle.c, TEST INFRASTRUCTURE) pinned on hand-written records, each rule's
boundary from both sides (tests/view_valid_common.py), and its place in view_main's filter chain on a small file."""
import pytest

import helpers
import view_count_common as vc
import view_text_common as vt
import view_valid_common as vv

CASES = vv.cases()


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_rule(i):
    what, rec, want = CASES[i]
    got, why = vv.oracle_valid(rec)
    assert got == want, what
    if want == vv.REFUSED:
        assert why in vv.REFUSAL_CODE


def _file(tmp_path, recs, sorted_file=True):
    if sorted_file:
        return vt.write_records(str(tmp_path / "v.bam"), vt.EDGE_REFS, recs)
    import flagstat_common as fc
    return helpers.write_bgzf(str(tmp_path / "u.bam"), fc.bam_body(vt.EDGE_REFS, recs), len(vt.EDGE_REFS))


def test_chain_order(tmp_path):
    """-s before the validator, --num-filter and -L / regions after it (on a sorted file, reads outside the regions never reach it)."""
    good = [vv.rec(name="g%d" % i, pos=10 + i) for i in range(5)]
    bad = vv.rec(name="a@", pos=100)
    broken = vv.rec(b"XXq\x01", name="brk", pos=200, flag=0x10)
    p = _file(tmp_path, good + [bad, broken])
    with vv.valid_oracle():
        with pytest.raises(RuntimeError, match="unknown tag type"):
            vc.oracle_count(p)
        with pytest.raises(RuntimeError, match="unknown tag type"):
            vc.oracle_count(p, num_filter=(0, 0x10))                    # --num-filter comes after the validator
        h = vc.fnv1a(b"brk", 0) & 0xFFFFFFFF
        frac = (h - 1) / 4294967296.0                                    # -s drops "brk": never validated
        assert vc.oracle_count(p, subsample=frac) == sum(1 for r in good + [bad] if (vc.fnv1a(r[36:36 + r[12] - 1], 0) & 0xFFFFFFFF) < vc.threshold(frac)) - (1 if (vc.fnv1a(b"a@", 0) & 0xFFFFFFFF) < vc.threshold(frac) else 0)
        assert vc.oracle_count(p, bed=[(0, 0, 150)]) == 5                # sorted: "brk" is outside the region
        assert vc.oracle_count(p, regions=[(0, 0, 150), (0, 0, 20)]) == 5 + 5
        with pytest.raises(RuntimeError):
            vc.oracle_count(p, regions=[(0, 150, 250)])
        assert vt.oracle_text(p, bed=[(0, 0, 150)]).count(b"\n") == 5
    assert vc.oracle_count(p) == 7 and vc.oracle_count(p, bed=[(0, 0, 150)]) == 6
    q = _file(tmp_path, good + [broken, bad], sorted_file=False)
    with vv.valid_oracle():
        with pytest.raises(RuntimeError):
            vc.oracle_count(q, bed=[(0, 0, 150)])                        # unsorted: BedFilter comes after the validator


def test_cli():
    import subprocess
    p = helpers.GOLDEN + "/issue_204.bam"
    a = subprocess.run([vc.ORACLE_EXE, "view", "-c", p], capture_output=True, text=True)
    b = subprocess.run([vc.ORACLE_EXE, "view", "-c", "-v", p], capture_output=True, text=True)
    assert a.returncode == 0 and b.returncode == 0 and int(b.stdout) <= int(a.stdout)
