"""Chimera detection on the GPU: every output file of every case of tests/uchime_cases.py (--uchime_ref and the three de
novo commands) byte for byte against the reference CLI's digests (and against a fresh reference run where
oracle/_ref/vsearch is built), the summary counts, a UDB database, several batches, abundance bands capped at 1 and 7
sequences, the serial pass's recomputations, and the refusals."""
import os

import pytest

import uchime_cases as U
from vsearch_b200 import lib as vlib

pytestmark = pytest.mark.gpu

GOLD = U.golden()


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def _run(ctx, d, name, db=None, **extra):
    q, r = U.CASES[name][0](d)
    opts = dict(U.CASES[name][1])
    paths = {k: os.path.join(d, "mine." + k) for k in U.OUTPUTS}
    st = ctx.uchime(q, db or r, **paths, **opts, **extra)
    assert st["bands"] == 0 or "command" in opts
    return st, paths


def _check(st, paths, want):
    assert {k: U.sha(p) for k, p in paths.items()} == want["files"]
    assert {k: st[k] for k in want["counts"]} == want["counts"]


@pytest.mark.parametrize("name", sorted(U.CASES))
def test_uchime_ref_equals_reference_cli(ctx, tmp_path, name):
    st, paths = _run(ctx, str(tmp_path), name)
    _check(st, paths, GOLD[name])
    if os.path.exists(U.STOCK):
        ref = tmp_path / "ref"
        ref.mkdir()
        rec, _ = U.run_reference(name, str(ref))
        assert rec["files"] == GOLD[name]["files"]


@pytest.mark.parametrize("name", ["a_default", "iupac_short", "long_refs"])
def test_uchime_ref_in_small_batches(ctx, tmp_path, name):
    st, paths = _run(ctx, str(tmp_path), name, batch_queries=7)
    _check(st, paths, GOLD[name])


@pytest.mark.parametrize("cap", [1, 7])
@pytest.mark.parametrize("name", U.DENOVO)
def test_uchime_denovo_band_caps(ctx, tmp_path, name, cap):
    """the files do not depend on how the sorted input is cut into bands"""
    st, paths = _run(ctx, str(tmp_path), name, band_cap=cap)
    _check(st, paths, GOLD[name])
    if cap == 1:
        assert st["bands"] == st["queries"] and st["recomputed"] == 0


def test_uchime_denovo_band_collision_recomputes(ctx, tmp_path):
    """many near-identical sequences of one abundance: earlier non-chimeras of the band change later candidate lists,
    and the serial pass finishes those queries again"""
    st, paths = _run(ctx, str(tmp_path), "dn_collision")
    _check(st, paths, GOLD["dn_collision"])
    assert st["bands"] < st["queries"]
    assert st["recomputed"] > 0


def test_uchime_ref_udb_database(ctx, tmp_path):
    """the UDB file --makeudb_usearch makes of a case's database (dbmask dust) gives the FASTA database's files"""
    d = str(tmp_path)
    _, r = U.CASES["a_default"][0](d)
    udb = os.path.join(d, "db.udb")
    ctx.makeudb_usearch(r, udb)
    st, paths = _run(ctx, d, "a_default", db=udb)
    _check(st, paths, GOLD["a_default"])


def test_uchime_ref_api_example_rows(ctx, tmp_path):
    st, paths = _run(ctx, str(tmp_path), "api_example")
    with open(os.path.join(U.FIXTURES, "expected_chimera.tsv")) as f:
        expected = sorted(f.read().splitlines())
    with open(paths["uchimeout"]) as f:
        assert sorted(f.read().splitlines()) == expected


def _refused(ctx, d, q, db, match, outputs=("uchimeout",), **kw):
    paths = {k: os.path.join(d, "bad." + k) for k in outputs}
    with pytest.raises(vlib.VsgError, match=match) as e:
        ctx.uchime(q, db, **paths, **kw)
    assert "failed (-3)" in str(e.value)
    for p in paths.values():
        assert not os.path.exists(p)


def test_uchime_ref_refusals(ctx, tmp_path):
    d = str(tmp_path)
    q, r = U.CASES["a_default"][0](d)
    _refused(ctx, d, q, r, "no output file", outputs=())
    _refused(ctx, d, q, r, "strand plus", strand_both=1)
    _refused(ctx, d, q, r, "hardmask", qmask="dust", dbmask="soft", hardmask=1)
    _refused(ctx, d, q, r, "hardmask", qmask="soft", dbmask="dust", hardmask=1)
    _refused(ctx, d, q, os.path.join(d, "missing.fasta"), "cannot open")
    _refused(ctx, d, os.path.join(d, "missing.fasta"), r, "cannot open")
    _refused(ctx, d, q, None, "database")
    _refused(ctx, d, q, r, "read by --uchime_ref only", command=1)
    _refused(ctx, d, q, None, "hardmask", command=3, qmask="dust", hardmask=1)
    _refused(ctx, d, q, None, "strand plus", command=2, strand_both=1)
    fq = os.path.join(d, "q.fastq")
    with open(fq, "w") as f:
        f.write("@a\nACGTACGTACGT\n+\nIIIIIIIIIIII\n")
    _refused(ctx, d, fq, r, "FASTQ")
    import gzip
    gz = os.path.join(d, "q.fasta.gz")
    with open(q, "rb") as fi, gzip.open(gz, "wb") as fo:
        fo.write(fi.read())
    _refused(ctx, d, gz, r, "gzip")


def test_uchime_ref_refuses_deferred_pairs(ctx, tmp_path):
    """a query whose alignment with a candidate passes the 16-bit aligner's cell bound is refused, naming the query"""
    import numpy as np
    rng = np.random.default_rng(3)
    ref = bytes(rng.choice(list(b"ACGT"), size=30000).astype(np.uint8).tobytes())
    d = str(tmp_path)
    r = os.path.join(d, "db.fasta")
    q = os.path.join(d, "q.fasta")
    with open(r, "w") as f:
        f.write(">long\n" + ref.decode() + "\n")
    with open(q, "w") as f:
        f.write(">longquery\n" + ref[:1200].decode() + "\n")
    _refused(ctx, d, q, r, "longquery", maxseqlength=100000)
