"""--orient on the GPU against the reference: vsg_orient_stream's output files equal `vsearch --orient ... --threads 1`
byte for byte for the option sets (a)-(g) and its strand counts equal the CLI's summary; vsg_orient's rows equal the
CLI's --tabbedout rows (the 105 kb read included) for whole calls, slices, small memory budgets, small batches and
device groups; and the errors come back with their codes."""
import bz2
import gzip
import os
import re

import numpy as np
import pytest

import checkers
import orient_cases as oc
from vsearch_b200 import lib, synth

pytestmark = pytest.mark.gpu


def _db_masking(case):
    """(database sequences, mask_lower, dust_db) as the caller maps --dbmask / --hardmask"""
    c = oc.CASES[case]
    seqs = oc.data()["db_seqs"]
    if c["hardmask"]:
        return [re.sub(rb"[a-z]", b"N", s) for s in seqs], 1, 0
    return seqs, int(c["dbmask"] != "none"), int(c["dbmask"] == "dust")


def _group(case, tmp, devices=(0,)):
    if oc.CASES[case]["udb"]:
        udb = lib.Udb(oc.udb_path(tmp))
        g = lib.Group.from_udb(list(devices), udb)
        udb.close()
        return g
    seqs, ml, dust = _db_masking(case)
    return lib.Group(list(devices), synth.SeqSet(seqs), wordlength=oc.CASES[case]["k"], mask_lower=ml, dust_db=dust)


def _stream(case, tmp, devices=(0,), batch_queries=65536):
    c = oc.CASES[case]
    _, qa, qq = oc.write_inputs(tmp)
    outs = {o: os.path.join(tmp, f"{case}.gpu.{o}") for o in c["outs"]}
    g = _group(case, tmp, devices)
    st, ns = g.orient_stream(qq if c["fastq"] else qa, query_mask_lower=int(c["qmask"] != "none"), notrunclabels=int(c["notrunc"]),
                             fasta_width=c["width"], batch_queries=batch_queries, **outs)
    g.close()
    return {o: open(p, "rb").read() for o, p in outs.items()}, st, ns


@pytest.mark.parametrize("case", list(oc.CASES))
def test_stream_matches_reference_cli(case, tmp_path):
    rec = oc.reference(case)
    got, st, ns = _stream(case, str(tmp_path))
    assert {o: checkers.digest(b) for o, b in got.items()} == rec["files"]
    assert oc.parse_rows(got["tabbedout"]) == rec["rows"]
    assert list(ns) == rec["summary"]
    nq = len(oc.data()["q_seqs"])
    assert st["queries"] == st["rows"] == nq and st["matched"] == ns[0] + ns[1]
    if case in ("a_defaults", "b_fastq"):
        # many small batches write the same files
        small, st2, _ = _stream(case, str(tmp_path), batch_queries=37)
        assert small == got and st2["batches"] > 5


def _context_rows(case, tmp, ctx):
    c = oc.CASES[case]
    if c["udb"]:
        udb = lib.Udb(oc.udb_path(tmp))
        db, ix, _ = ctx.udb_load(udb)
        udb.close()
    else:
        seqs, ml, dust = _db_masking(case)
        db = ctx.seqset(synth.SeqSet(seqs))
        if dust:
            db.dust()
        ix = ctx.index(db, wordlength=c["k"], mask_lower=ml)
    q = oc.data()["q_seqs"]
    qs = ctx.seqset(synth.SeqSet(q))
    qml = int(c["qmask"] != "none")
    return db, ix, qs, qml


@pytest.mark.parametrize("case", list(oc.CASES))
def test_orient_rows_match_reference(case, tmp_path):
    rows = np.array(oc.reference(case)["rows"], dtype=np.int64)
    ctx = lib.Context(0)
    db, ix, qs, qml = _context_rows(case, str(tmp_path), ctx)
    n = rows.shape[0]
    got = ctx.orient(ix, qs, 0, n, query_mask_lower=qml)
    assert (got == rows).all()
    # slices, and the 105 kb read on its own: the same rows
    lq = oc.data()["meta"]["long_query"]
    for q0, m in ((100, 57), (lq, 1), (n - 1, 1), (0, 1)):
        assert (ctx.orient(ix, qs, q0, m, query_mask_lower=qml) == rows[q0:q0 + m]).all()
    assert ctx.orient(ix, qs, 5, 0, query_mask_lower=qml).shape == (0, 3)
    for h in (qs, ix, db):
        h.close()
    ctx.close()


def test_small_budget_cuts_launches(tmp_path, monkeypatch):
    """VSG_DIR_BUDGET_MB=1: 16 384 windows per launch, so the reads take many launches and the long one goes alone"""
    monkeypatch.setenv("VSG_DIR_BUDGET_MB", "1")
    rows = np.array(oc.reference("a_defaults")["rows"], dtype=np.int64)
    ctx = lib.Context(0)
    db, ix, qs, qml = _context_rows("a_defaults", str(tmp_path), ctx)
    assert (ctx.orient(ix, qs, 0, rows.shape[0], query_mask_lower=qml) == rows).all()
    for h in (qs, ix, db):
        h.close()
    ctx.close()


def test_group_of_two_equals_one(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one, _, n1 = _stream("b_fastq", str(tmp_path))
    two, _, n2 = _stream("b_fastq", str(tmp_path), devices=(0, 1))
    assert one == two and n1 == n2


def test_errors(tmp_path):
    tmp = str(tmp_path)
    _, qa, qq = oc.write_inputs(tmp)
    seqs = oc.data()["db_seqs"][:50]
    g = lib.Group([0], synth.SeqSet(seqs), wordlength=12, mask_lower=1)
    tab = os.path.join(tmp, "o.tsv")
    with pytest.raises(lib.VsgError, match=r"\(-3\).*no output file"):
        g.orient_stream(qa)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*FASTQ output with FASTA input"):
        g.orient_stream(qa, fastqout=os.path.join(tmp, "o.fq"))
    fq = open(qq, "rb").read()
    bad = {
        "truncated.fq": (fq[:fq.index(b"\n@o3\n") + 9], r"FASTQ record 4: the file ends early"),
        "shortqual.fq": (fq[:fq.index(b"\n@o2\n") - 1] + fq[fq.index(b"\n@o2\n"):], r"FASTQ record 2: the quality is not as long"),
        "plus.fq": (fq.replace(b"\n+\n", b"\n+other\n", 1), r"FASTQ record 1: the '\+' line"),
    }
    for name, (text, msg) in bad.items():
        p = os.path.join(tmp, name)
        open(p, "wb").write(text)
        with pytest.raises(lib.VsgError, match=r"\(-3\).*" + msg):
            g.orient_stream(p, tabbedout=tab)
    gz, bzf = os.path.join(tmp, "reads.fa.gz"), os.path.join(tmp, "reads.fa.bz2")
    open(gz, "wb").write(gzip.compress(open(qa, "rb").read()))
    open(bzf, "wb").write(bz2.compress(open(qa, "rb").read()))
    with pytest.raises(lib.VsgError, match=r"\(-3\).*gzip-compressed input is not supported"):
        g.orient_stream(gz, tabbedout=tab)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*bzip2-compressed input is not supported"):
        g.orient_stream(bzf, tabbedout=tab)
    g.close()
    ctx = lib.Context(0)
    db = ctx.seqset(synth.SeqSet(seqs))
    ix = ctx.index(db, wordlength=12, mask_lower=1)
    qs = ctx.seqset(synth.SeqSet(oc.data()["q_seqs"][:10]))
    with pytest.raises(lib.VsgError, match=r"\(-3\).*out of bounds"):
        ctx.orient(ix, qs, 5, 6)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*out of bounds"):
        ctx.orient(ix, qs, -1, 1)
    for h in (qs, ix, db):
        h.close()
    ctx.close()
