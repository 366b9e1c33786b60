"""--chimeras_denovo on the GPU: every output file of every case of tests/chimeras_denovo_cases.py byte for byte against
the reference CLI's digests (and against a fresh reference run where oracle/_ref/vsearch is built), the summary counts,
bands capped at 1 and 7 sequences, the serial pass's recomputations, --fasta_score, and the refusals."""
import os

import pytest

import chimeras_denovo_cases as D
from vsearch_b200 import lib as vlib

pytestmark = pytest.mark.gpu

GOLD = D.golden()


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def _run(ctx, d, name, **extra):
    q = D.CASES[name][0](d)
    paths = {k: os.path.join(d, "mine." + k) for k in D.OUTPUTS}
    st = ctx.uchime(q, None, command=D.C, **paths, **D.api_opts(D.CASES[name][1]), **extra)
    return st, paths


def _check(st, paths, want):
    assert {k: D.U.sha(p) for k, p in paths.items()} == want["files"]
    assert {k: st[k] for k in want["counts"]} == want["counts"]


@pytest.mark.parametrize("name", sorted(D.CASES))
def test_chimeras_denovo_equals_reference_cli(ctx, tmp_path, name):
    st, paths = _run(ctx, str(tmp_path), name)
    _check(st, paths, GOLD[name])
    if os.path.exists(D.STOCK):
        ref = tmp_path / "ref"
        ref.mkdir()
        rec, _ = D.run_reference(name, str(ref))
        assert rec["files"] == GOLD[name]["files"]


@pytest.mark.parametrize("cap", [1, 7])
@pytest.mark.parametrize("name", ["cd_default", "cd_abskew2", "cd_equal", "cd_parts100", "cd_collision"])
def test_chimeras_denovo_band_caps(ctx, tmp_path, name, cap):
    """the files do not depend on how the sorted input is cut into bands"""
    st, paths = _run(ctx, str(tmp_path), name, band_cap=cap)
    _check(st, paths, GOLD[name])
    if cap == 1:
        assert st["bands"] == st["queries"] and st["recomputed"] == 0


def test_chimeras_denovo_collision_recomputes(ctx, tmp_path):
    """many reads of one abundance at --abskew 1: a band's earlier members are taken as parents of its later ones; where
    one of them turns out chimeric, the serial pass rebuilds the later heaps, aligns what the speculative cut left out,
    and finishes those queries again"""
    st, paths = _run(ctx, str(tmp_path), "cd_collision")
    _check(st, paths, GOLD["cd_collision"])
    assert st["bands"] < st["queries"]
    assert st["recomputed"] > 0


def test_chimeras_denovo_fasta_score(ctx, tmp_path):
    """--fasta_score appends ;uchime_denovo= with the uchime score, which --chimeras_denovo never sets"""
    d = str(tmp_path)
    st, paths = _run(ctx, d, "cd_default", fasta_score=1, fasta_width=0)
    plain = os.path.join(d, "plain")
    os.mkdir(plain)
    _, p0 = _run(ctx, plain, "cd_default", fasta_width=0)
    for k in ("chimeras", "nonchimeras"):
        with open(paths[k]) as f, open(p0[k]) as g:
            a, b = f.read().splitlines(), g.read().splitlines()
        assert [x for x in a if not x.startswith(">")] == [x for x in b if not x.startswith(">")]
        assert [x for x in a if x.startswith(">")] == [x + ";uchime_denovo=0.0000" for x in b if x.startswith(">")]
    assert st["chimeras"] > 0


def _refused(ctx, d, q, match, outputs=("chimeras",), **kw):
    paths = {k: os.path.join(d, "bad." + k) for k in outputs}
    with pytest.raises(vlib.VsgError, match=match) as e:
        ctx.uchime(q, None, **paths, **kw)
    assert "failed (-3)" in str(e.value)
    for p in paths.values():
        assert not os.path.exists(p)


def test_chimeras_denovo_refusals(ctx, tmp_path):
    d = str(tmp_path)
    q = D.CASES["cd_default"][0](d)
    c = {"command": D.C}
    _refused(ctx, d, q, "chimeras_parts", chimeras_parts=1, **c)
    _refused(ctx, d, q, "chimeras_parts", chimeras_parts=101, **c)
    _refused(ctx, d, q, "chimeras_parents_max", chimeras_parents_max=1, **c)
    _refused(ctx, d, q, "chimeras_parents_max", chimeras_parents_max=21, **c)
    _refused(ctx, d, q, "chimeras_length_min", chimeras_length_min=0, **c)
    _refused(ctx, d, q, "chimeras_diff_pct", chimeras_diff_pct=-0.1, **c)
    _refused(ctx, d, q, "chimeras_diff_pct", chimeras_diff_pct=50.5, **c)
    _refused(ctx, d, q, "borderline", outputs=("chimeras", "borderline"), **c)
    for cmd in ("uchime_denovo", "uchime2_denovo", "uchime3_denovo"):
        for field, v in (("chimeras_parts", 7), ("chimeras_parents_max", 5), ("chimeras_length_min", 20), ("chimeras_diff_pct", 0.3)):
            _refused(ctx, d, q, "belong to --chimeras_denovo", command=cmd, **{field: v})
    _refused(ctx, d, q, "no output file", outputs=(), **c)
    _refused(ctx, d, q, "strand plus", strand_both=1, **c)
    _refused(ctx, d, q, "hardmask", qmask="dust", hardmask=1, **c)
    _refused(ctx, d, os.path.join(d, "missing.fasta"), "cannot open", **c)
    import gzip
    gz = os.path.join(d, "q.fasta.gz")
    with open(q, "rb") as fi, gzip.open(gz, "wb") as fo:
        fo.write(fi.read())
    _refused(ctx, d, gz, "gzip", **c)
    with pytest.raises(vlib.VsgError, match="read by --uchime_ref only"):
        ctx.uchime(q, q, chimeras=os.path.join(d, "bad.chimeras"), **c)
