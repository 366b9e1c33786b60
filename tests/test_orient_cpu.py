"""--orient without a GPU: a numpy restatement of the vote (distinct query k-mers, the 8x rule per k-mer, the 4x rule per
read) reproduces the reference CLI's --tabbedout rows for every option set, which pins the fixture and the rules the GPU
tests check; and the new entry points are declared and exported."""
import numpy as np
import pytest

import orient_cases as oc
from vsearch_b200 import lib


@pytest.mark.parametrize("case", list(oc.CASES))
def test_restatement_matches_reference_rows(case, tmp_path):
    c = oc.CASES[case]
    rec = oc.reference(case)
    if c["udb"]:
        udb = lib.Udb(oc.udb_path(str(tmp_path)))
        assert udb.info.wordlength == 8 and udb.n == oc.UDB_SEQS
        kc, _ = udb.words()
        udb.close()
        words = np.nonzero(kc)[0].astype(np.int64)
        counts = kc[words].astype(np.int64)
    else:
        seqs, skip_lower = oc.database_as_indexed(case, rec.get("dust"))
        words, counts = oc.word_counts(seqs, c["k"], skip_lower)
    rows = oc.orient_rows(oc.data()["q_seqs"], c["k"], c["qmask"] != "none", words, counts)
    assert rows == rec["rows"]
    s = np.array(rows)[:, 0]
    assert [int((s == v).sum()) for v in range(3)] == rec["summary"]


@pytest.mark.parametrize("k", [3, 4, 5, 6])
@pytest.mark.parametrize("mask", ["none", "soft"])
def test_restatement_matches_reference_votes_at_short_wordlengths(k, mask, tmp_path):
    """on the strand-biased fixture reads are oriented both ways even at k = 3..6, and the restatement's rows equal the
    reference CLI's there too"""
    d = oc.biased_data()
    want = oc.biased_reference(k, mask, lambda: oc.run_biased_cli(k, mask, str(tmp_path)))
    skip = mask == "soft"
    assert oc.orient_rows(d["q_seqs"], k, skip, *oc.word_counts(d["db_seqs"], k, skip)) == want
    r = np.array(want)
    assert set(r[:, 0]) == {0, 1, 2} and (r[:, 1] > 0).sum() > 20 and (r[:, 2] > 0).sum() > 20, (k, mask)


def test_fixture_covers_the_rules():
    """every case has reads of all three outcomes; the joins fall on both sides of the 4x rule; short reads get 0/0"""
    d = oc.data()
    rows = np.array(oc.reference("a_defaults")["rows"])
    assert set(rows[:, 0]) == {0, 1, 2}
    for i in d["meta"]["short_queries"]:
        assert list(rows[i]) == [2, 0, 0]
    joins = [i for i, h in enumerate(d["q_heads"]) if h.startswith("o") and h[1:].split()[0].isdigit()
             and int(h[1:].split()[0]) % 9 in (5, 6)]
    both = rows[joins]
    decided = both[(both[:, 1] > 0) & (both[:, 2] > 0)]
    assert (decided[:, 0] != 2).any() and (decided[:, 0] == 2).any()
    lq = d["meta"]["long_query"]
    assert len(d["q_seqs"][lq]) > 100_000 and rows[lq, 1] > 10_000
    # the UDB case runs at the file's word length 8, not the default 12
    assert oc.reference("f_udb8")["rows"] != oc.reference("a_defaults")["rows"]


def test_symbols_declared_and_exported():
    syms = lib.declared_symbols()
    assert "vsg_orient" in syms and "vsg_orient_stream" in syms
    exported = lib.load()
    assert hasattr(exported, "vsg_orient") and hasattr(exported, "vsg_orient_stream")
