"""SINTAX without a GPU: the reference CLI's --tabbedout equals vsg_sintax_rows fed with the reference's own
per-bootstrap winners (vsref_sintax), byte for byte, which pins the vote, the formatting and the strand rule; and the
options vsg_sintax_rows refuses."""
import numpy as np
import pytest

import sintax_cases as sc
from vsearch_b200 import lib

needs_ref = pytest.mark.skipif(not sc.reference_available(), reason="oracle/_ref (reference CLI + sintax shim) not built")


@needs_ref
@pytest.mark.parametrize("case", [c for c in sc.CASES if not sc.CASES[c][5]])
def test_rows_match_reference_cli(case, tmp_path):
    want = sc.run_cli(case, str(tmp_path))
    boots = sc.ref_bootstraps(case)
    heads, _ = sc.database()
    _, _, both, cutoff, _, _ = sc.CASES[case]
    got = lib.sintax_rows(sc.to_results(boots), sc.data()["q_heads"], heads, cutoff=cutoff, strand_both=both)
    assert got == want
    rows = want.decode().splitlines()
    assert any(r.split("\t")[1] == "" for r in rows) and any(r.split("\t")[1] != "" for r in rows)
    # the stored digests the GPU tests compare against are these very results
    assert sc.reference("cli", case, lambda: want) == sc.checkers.digest(want)
    if case in sc.PER_BOOTSTRAP:
        assert sc.reference("boots", case, lambda: boots) == sc.checkers.digest(boots)


def test_rows_reject_bad_options():
    r = np.zeros(1, dtype=lib.SINTAX_DT)
    with pytest.raises(lib.VsgError, match="sintax_random"):
        lib.sintax_rows(r, ["q"], ["t;tax=d:A"], random_ties=1)
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(lib.VsgError, match="cutoff"):
            lib.sintax_rows(r, ["q"], ["t;tax=d:A"], cutoff=bad)


def test_rows_unclassified_and_header_variants():
    """fewer than 50 successful bootstraps: an empty row; the tax= parsing quirks of tax_parse / tax_split"""
    heads = ["t0 xtax=d:Fake;tax=D:Dom,p:Phy,s:Sp", "t1;tax=d:Dom,p:Phy,s:Sp;note=a,b"]
    r = np.zeros(3, dtype=lib.SINTAX_DT)
    r["seqno"] = -1
    r["nboot"][1, 0] = 49
    r["seqno"][1, 0, :49] = 0
    r["nboot"][2, 0] = 60
    r["seqno"][2, 0, :40] = 0
    r["seqno"][2, 0, 40:60] = 1
    got = lib.sintax_rows(r, ["a", "b", "c"], heads, cutoff=0.5).decode().split("\n")
    assert got[0] == "a\t\t\t" and got[1] == "b\t\t\t"
    # t1's species name runs to the next ',' of the whole header, as tax_split reads it
    assert got[2] == "c\td:Dom(1.00),p:Phy(1.00),s:Sp(0.67)\t+\td:Dom,p:Phy,s:Sp"
    assert lib.sintax_rows(r[:0], [], heads) == b""
