"""--uchime_ref without a GPU: the case generator reproduces the inputs behind tests/golden/uchime_reference.json, and
where oracle/_ref/vsearch is built a fresh reference run reproduces the recorded digests and counts."""
import os

import pytest

import uchime_cases as U

GOLD = U.golden()


@pytest.mark.parametrize("name", sorted(U.CASES))
def test_case_inputs_match_goldens(tmp_path, name):
    q, r = U.CASES[name][0](str(tmp_path))
    assert U.sha(q) == GOLD[name]["query_sha256"]
    assert (U.sha(r) if r else None) == GOLD[name]["db_sha256"]


@pytest.mark.skipif(not os.path.exists(U.STOCK), reason="oracle/_ref/vsearch not built")
def test_api_example_reproduces_expected_tsv(tmp_path):
    """the api_examples fixtures: the reference's --uchimeout holds the rows of expected_chimera.tsv (which the library
    example writes in thread order, so the rows are compared sorted)"""
    _, paths = U.run_reference("api_example", str(tmp_path))
    with open(os.path.join(U.FIXTURES, "expected_chimera.tsv")) as f:
        expected = sorted(f.read().splitlines())
    with open(paths["uchimeout"]) as f:
        assert sorted(f.read().splitlines()) == expected


@pytest.mark.skipif(not os.path.exists(U.STOCK), reason="oracle/_ref/vsearch not built")
@pytest.mark.parametrize("name", sorted(U.CASES))
def test_reference_cli_reproduces_goldens(tmp_path, name):
    rec, _ = U.run_reference(name, str(tmp_path))
    assert rec == GOLD[name]
