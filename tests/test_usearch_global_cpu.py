"""--usearch_global's writer pinned without a GPU: for every case of usearch_global_cases.py with a FASTA database, each
query's rows are rebuilt from the reference's hit list (tests/golden/usearch_global_reference.json: target, strand,
printed identity, CIGAR) with the plain-C aligner (checkers.oracle_nw16, trims_from_cigar, finish_hit), and
vsg_search_write (no device) must write every output file byte for byte as the reference CLI did.  DUST is not restated:
the files that print DUST-masked sequences are left to the GPU test.  A failed write leaves no file."""
import os
import re

import pytest

import checkers
import usearch_global_cases as cases
from vsearch_b200 import lib as vlib


def read_fastx(path, notrunclabels=False):
    labels, seqs = [], []
    text = open(path).read()
    if text.startswith("@"):
        lines = text.splitlines()
        for i in range(0, len(lines), 4):
            labels.append(lines[i][1:])
            seqs.append(lines[i + 1])
    else:
        for rec in text.split(">")[1:]:
            h, _, body = rec.partition("\n")
            labels.append(h)
            seqs.append(body.replace("\n", ""))
    if not notrunclabels:
        labels = [re.split(r"[ \t]", h)[0] for h in labels]
    return labels, [s.encode() for s in seqs]


def size_of(h):
    """header_get_size: (^|;)size=[0-9]+(;|$), else 1"""
    m = re.search(r"(?:^|;)size=([0-9]+)(?=;|$)", h)
    return int(m.group(1)) if m else 1


def hardmask(s: bytes) -> bytes:
    return re.sub(rb"[a-z]", b"N", s)


def rebuild_row(q: bytes, t: bytes, target: int, strand: int):
    """the search row of query q (plus strand) against target t on `strand`, and its CIGAR, from the oracle aligner"""
    qs = cases.revcomp(q) if strand else q
    f = checkers.oracle_row_fields(qs, t)
    _, _, _, _, _, cigar = checkers.oracle_nw16(qs, t)
    r = vlib.SearchResult(target=target, matches=f["matches"], mismatches=f["mismatches"], gaps=f["gaps"],
                          alignment_length=f["aligned"], query_length=len(q), target_length=len(t), accepted=1, strand=strand,
                          nwscore=f["nwscore"], id=f["id"], internal_alignment_length=f["internal_alignment_length"],
                          internal_gaps=f["internal_gaps"])
    return r, cigar


def inputs(name, directory):
    """(query labels, query sequences as printed, database labels, database sequences as printed) of case `name`"""
    inp, cli, kw, outputs, dbkind = cases.CASES[name]
    q, db = cases.input_files(inp, directory)
    notrunc = kw.get("notrunclabels", 0)
    dl, ds = read_fastx(db, notrunc)
    keep = [i for i in range(len(ds)) if kw.get("minseqlength", 32) <= len(ds[i]) <= kw.get("maxseqlength", 50000)]
    dl, ds = [dl[i] for i in keep], [ds[i] for i in keep]
    ql, qs = read_fastx(q, notrunc)
    if kw.get("hardmask"):
        if kw.get("dbmask") == "soft":
            ds = [hardmask(s) for s in ds]
        if kw.get("qmask") == "soft":
            qs = [hardmask(s) for s in qs]
    return q, db, ql, qs, dl, ds


@pytest.mark.parametrize("name", sorted(n for n, c in cases.CASES.items() if c[4] == "fasta"))
def test_search_write_equals_reference(tmp_path, name):
    inp, cli, kw, outputs, dbkind = cases.CASES[name]
    want = cases.golden()[name]
    q, db, ql, qs, dl, ds = inputs(name, str(tmp_path))
    assert cases.sha256(q) == want["query_sha256"] and cases.sha256(db) == want["db_sha256"]
    assert len(want["hits"]) == len(ql)
    hits = []
    for i, hl in enumerate(want["hits"]):
        rows = []
        for target, strand, ident, cigar in hl:
            r, c = rebuild_row(qs[i], ds[target], target, strand)
            assert f"{r.id:.1f}" == ident, (name, i, target)
            assert (c if r.matches != r.alignment_length else "=") == cigar, (name, i, target)
            rows.append((r, c))
        hits.append(rows)
    paths = cases.output_files(str(tmp_path / "mine"), name, outputs)
    os.makedirs(tmp_path / "mine")
    wkw = {k: v for k, v in kw.items() if k in {f for f, _ in vlib.UsearchGlobalOpts._fields_}}
    matched = vlib.search_write(ql, qs, [size_of(h) for h in ql], hits, dl, ds, [size_of(h) for h in dl], **paths, **wkw)
    skip = cases.dusted(name)
    assert {o: h for o, h in cases.output_digests(paths).items() if o not in skip} == \
        {o: h for o, h in want["files"].items() if o not in skip}
    assert matched == want["matched"] and len(ql) == want["queries"]


def test_search_write_failure_leaves_no_file(tmp_path):
    name = "a_default"
    q, db, ql, qs, dl, ds = inputs(name, str(tmp_path))
    hits = [[rebuild_row(qs[i], ds[t], t, s) for t, s, _, _ in hl] for i, hl in enumerate(cases.golden()[name]["hits"])]
    out = tmp_path / "out"
    out.mkdir()
    paths = cases.output_files(str(out), "x", cases.OUTPUTS)
    paths["dbnotmatched"] = str(tmp_path / "no" / "such" / "dir" / "x.dbnotmatched")   # the last file written fails
    with pytest.raises(vlib.VsgError, match="cannot write"):
        vlib.search_write(ql, qs, [size_of(h) for h in ql], hits, dl, ds, [size_of(h) for h in dl], **paths)
    assert os.listdir(out) == []
    # a printed --uc row that needs its CIGAR and has none is refused before any file is made
    bare = [[(r, None) for r, _ in h] for h in hits]
    with pytest.raises(vlib.VsgError, match="needs its CIGAR"):
        vlib.search_write(ql, qs, [size_of(h) for h in ql], bare, dl, ds, [size_of(h) for h in dl], uc=str(out / "x.uc"))
    assert os.listdir(out) == []
    with pytest.raises(vlib.VsgError, match="maxhits"):
        vlib.search_write(ql, qs, [size_of(h) for h in ql], hits, dl, ds, [size_of(h) for h in dl], uc=str(out / "x.uc"), maxhits=-1)
    assert os.listdir(out) == []
