"""vsg_usearch_global_command on the GPU.  Every output file of every case of usearch_global_cases.py equals the reference
CLI's (sha256, tests/golden/usearch_global_reference.json), also in batches of 7 queries; the UDB case searches a file made
by Context.makeudb_usearch, which must equal the reference's UDB file; with oracle/_ref/vsearch present the reference's
files are made afresh too.  Each refusal leaves no file.  At scale (200 000 reads against 20 000 ZOTUs) the OTU table,
--dbmatched and --uc rows equal a Python tabulation of Context.search_hits over the same queries, and every printed CIGAR
agrees with its row's columns, matches and gaps."""
import bz2
import ctypes as C
import gzip
import os
import re

import numpy as np
import pytest

import usearch_global_cases as cases
from vsearch_b200 import lib as vlib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def _database(ctx, tmp_path, name):
    """the case's database path: the FASTA file, or the UDB file Context.makeudb_usearch makes of it"""
    inp, cli, kw, outputs, dbkind = cases.CASES[name]
    q, db = cases.input_files(inp, str(tmp_path))
    if dbkind != "udb":
        return q, db
    udb = str(tmp_path / f"{name}.udb")
    ctx.makeudb_usearch(db, udb)
    assert cases.sha256(udb) == cases.golden()[name]["udb_sha256"]
    return q, udb


def _run_case(ctx, tmp_path, name, **extra):
    inp, cli, kw, outputs, dbkind = cases.CASES[name]
    want = cases.golden()[name]
    q, db = _database(ctx, tmp_path, name)
    assert cases.sha256(q) == want["query_sha256"] and cases.sha256(cases.input_files(inp, str(tmp_path))[1]) == want["db_sha256"]
    mine = tmp_path / "mine"
    mine.mkdir(exist_ok=True)
    paths = cases.output_files(str(mine), name, outputs)
    st = ctx.usearch_global_command(q, db, **paths, **kw, **extra)
    assert cases.output_digests(paths) == want["files"]
    assert (st["matched"], st["queries"]) == (want["matched"], want["queries"])
    assert st["hits"] == sum(len(h) for h in want["hits"])
    return q, db


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_usearch_global_command_equals_reference_cli(ctx, tmp_path, name):
    q, db = _run_case(ctx, tmp_path, name)
    if os.path.exists(cases.STOCK):
        inp, cli, kw, outputs, dbkind = cases.CASES[name]
        ref = tmp_path / "ref"
        ref.mkdir()
        if dbkind == "udb":
            cases.reference_makeudb(cases.input_files(inp, str(tmp_path))[1], str(ref / "db.udb"))
            assert cases.sha256(str(ref / "db.udb")) == cases.golden()[name]["udb_sha256"]
        rpaths = cases.output_files(str(ref), name, outputs)
        counts = cases.reference_run(q, db, cli, rpaths)
        assert cases.output_digests(rpaths) == cases.golden()[name]["files"]
        assert counts == {k: cases.golden()[name][k] for k in counts}


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_usearch_global_command_batches_of_7(ctx, tmp_path, name):
    _run_case(ctx, tmp_path, name, batch_queries=7)


def _refused(ctx, tmp_path, q, db, match, **kw):
    out = tmp_path / "out"
    out.mkdir(exist_ok=True)
    paths = {} if kw.pop("no_outputs", False) else cases.output_files(str(out), "x", cases.OUTPUTS)
    with pytest.raises(vlib.VsgError, match=match) as e:
        ctx.usearch_global_command(q, db, **paths, **kw)
    assert "(-3)" in str(e.value)          # VSG_EINVAL
    assert sorted(os.listdir(out)) == []


def test_usearch_global_command_refusals(ctx, tmp_path):
    q, db = cases.input_files("amplicons", str(tmp_path))
    _refused(ctx, tmp_path, q, db, "No output", no_outputs=True, id=0.97)
    for path, comp, what in ((q, gzip.compress, "gzip"), (q, bz2.compress, "bzip2")):
        z = tmp_path / f"q.{what}"
        z.write_bytes(comp(open(path, "rb").read()))
        _refused(ctx, tmp_path, str(z), db, what, id=0.97)
        _refused(ctx, tmp_path, q, str(z), what, id=0.97)
    _refused(ctx, tmp_path, q, db, "hardmask", hardmask=1, id=0.97)
    _refused(ctx, tmp_path, q, db, "hardmask", hardmask=1, qmask="soft", id=0.97)
    _refused(ctx, tmp_path, q, db, "hardmask", hardmask=1, dbmask="soft", id=0.97)
    _refused(ctx, tmp_path, str(tmp_path / "missing.fa"), db, "cannot open", id=0.97)
    _refused(ctx, tmp_path, q, str(tmp_path / "missing.fa"), "cannot open", id=0.97)
    _refused(ctx, tmp_path, q, db, "maxhits", maxhits=-1, id=0.97)
    one = (C.c_int64 * 1)(1)
    for field in ("query_sizes", "target_sizes", "query_labels", "target_labels"):
        _refused(ctx, tmp_path, q, db, "pass them NULL", id=0.97, **{field: C.cast(one, C.POINTER(C.c_int64))})


def test_usearch_global_command_refuses_deferred_pairs(ctx, tmp_path):
    rng = np.random.default_rng(9)
    t = bytes(rng.choice(list(b"ACGT"), size=6000).astype(np.uint8))
    b = bytearray(t)
    b[3000] = b"ACGT"[(b"ACGT".index(b[3000]) + 1) % 4]
    q = tmp_path / "long.q.fasta"
    q.write_text(f">q\n{bytes(b).decode()}\n")
    db = tmp_path / "long.db.fasta"
    db.write_text(f">t\n{t.decode()}\n")
    # 6 000 x 6 000 cells: beyond the 16-bit aligner, and no fallback callback
    _refused(ctx, tmp_path, str(q), str(db), "failed", id=0.97, qmask="none", dbmask="none")
    # every pair deferred (a gap penalty outside 16 bits): the search goes through the callback, the CIGAR cannot
    s = bytes(rng.choice(list(b"ACGT"), size=200).astype(np.uint8))
    m = bytearray(s)
    m[100] = b"ACGT"[(b"ACGT".index(m[100]) + 1) % 4]
    q2 = tmp_path / "short.q.fasta"
    q2.write_text(f">r1\n{bytes(m).decode()}\n")
    db2 = tmp_path / "short.db.fasta"
    db2.write_text(f">z1\n{s.decode()}\n")
    pen = np.array(vlib.DEFAULT_PEN, dtype=np.int64)
    pen[4] = 2 ** 31 - 1
    c = vlib.Context(0, pen=pen)
    try:
        c.set_fallback(lambda qi, strand, ti: (390, 200, 199, 1, 0, 0, 0, 0, 0))
        out = tmp_path / "ok"
        out.mkdir()
        c.usearch_global_command(str(q2), str(db2), blast6out=str(out / "x.b6"), id=0.97)   # without --uc no CIGAR is needed
        assert open(out / "x.b6").read().startswith("r1\tz1\t99.5\t")
        _refused(c, tmp_path, str(q2), str(db2), "defers the alignment of r1 with z1", id=0.97)
    finally:
        c.close()


# ---- at scale, against Context.search_hits ---------------------------------------------------------------------------

class _Seqs:
    """the arrays Context.seqset uploads"""

    def __init__(self, seqs):
        self.cat = np.frombuffer(b"".join(seqs) + b"\0", dtype=np.uint8)
        self.lens = np.array([len(s) for s in seqs], dtype=np.int32)
        self.offs = np.zeros(len(seqs), dtype=np.int64)
        if len(seqs) > 1:
            self.offs[1:] = np.cumsum(self.lens[:-1], dtype=np.int64)


def _cigar_agrees(cigar, row):
    """a CIGAR's columns, gap runs and match-or-mismatch columns against the row's alignment statistics"""
    ops = re.findall(r"(\d*)([MID])", cigar)
    assert "".join(n + o for n, o in ops) == cigar
    cols = sum(int(n or 1) for n, _ in ops)
    mcols = sum(int(n or 1) for n, o in ops if o == "M")
    gaps = sum(1 for _, o in ops if o != "M")
    assert (cols, gaps, mcols) == (row.alignment_length, row.gaps, row.matches + row.mismatches), (cigar, cols, gaps, mcols)
    assert row.matches < row.alignment_length


def test_usearch_global_command_at_scale(ctx, tmp_path):
    rng = np.random.default_rng(11)
    nz, nr, L = 20_000, 200_000, 250
    alphabet = np.frombuffer(b"ACGT", dtype=np.uint8)
    zot = alphabet[rng.integers(0, 4, size=(nz, L))]
    pick = rng.integers(0, nz, size=nr)
    reads = zot[pick].copy()
    # 0..3 substitutions per read, a share of the reads reverse-complemented, one in ten with an indel
    for k in range(3):
        rows = np.nonzero(rng.random(nr) < 0.35)[0]
        cols = rng.integers(0, L, size=rows.size)
        reads[rows, cols] = alphabet[(np.searchsorted(alphabet, reads[rows, cols]) + 1) % 4]
    seqs = [r.tobytes() for r in reads]
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    for i in np.nonzero(rng.random(nr) < 0.1)[0]:
        p = int(rng.integers(5, L - 5))
        seqs[i] = seqs[i][:p] + seqs[i][p + 1:] if i % 2 else seqs[i][:p] + b"G" + seqs[i][p:]
    for i in np.nonzero(rng.random(nr) < 0.3)[0]:
        seqs[i] = seqs[i].translate(comp)[::-1]
    zseqs = [z.tobytes() for z in zot]
    zlab = [f"Zotu{i + 1}" for i in range(nz)]
    qlab = [f"r{i};sample=S{i % 96}" for i in range(nr)]
    q = tmp_path / "reads.fa"
    db = tmp_path / "zotus.fa"
    q.write_text("".join(f">{h}\n{s.decode()}\n" for h, s in zip(qlab, seqs)))
    db.write_text("".join(f">{h}\n{s.decode()}\n" for h, s in zip(zlab, zseqs)))
    paths = {k: str(tmp_path / f"out.{k}") for k in ("otutabout", "dbmatched", "uc")}
    st = ctx.usearch_global_command(str(q), str(db), **paths, id=0.97, strand_both=1, qmask="none", dbmask="none")
    assert st["queries"] == nr

    dbs = ctx.seqset(_Seqs(zseqs))
    qs = ctx.seqset(_Seqs(seqs))
    ix = ctx.index(dbs, 8, 0)
    try:
        o = vlib.default_search_opts()
        o.id = 0.97
        o.strand_both = 1
        rows, first, _ = ctx.search_hits(ix, dbs, qs, 0, nr, o)
    finally:
        ix.close()
        qs.close()
        dbs.close()
    assert st["hits"] == int(first[-1])
    count, dbm, uc_want, matched = {}, np.zeros(nz, dtype=np.int64), [], 0
    for i in range(nr):
        a, b = int(first[i]), int(first[i + 1])
        sample = f"S{i % 96}"
        if b > a:
            matched += 1
            r = rows[a]
            key = (zlab[r.target], sample)
            count[key] = count.get(key, 0) + 1
            uc_want.append((f"H\t{r.target}\t{len(seqs[i])}\t{r.id:.1f}\t{'-' if r.strand else '+'}\t0\t0", qlab[i], zlab[r.target], r))
            for j in range(a, b):
                dbm[rows[j].target] += 1
        else:
            uc_want.append((None, qlab[i], None, None))
    assert st["matched"] == matched
    samples = sorted({f"S{i % 96}" for i in range(nr)}, key=str.encode)
    otus = sorted(zlab, key=str.encode)
    table = "#OTU ID" + "".join("\t" + s for s in samples) + "\n" + "".join(
        o + "".join(f"\t{count.get((o, s), 0)}" for s in samples) + "\n" for o in otus)
    assert open(paths["otutabout"]).read() == table
    assert re.findall(r"^>(\S+)$", open(paths["dbmatched"]).read(), flags=re.M) == [zlab[t] for t in np.nonzero(dbm)[0]]
    uc = open(paths["uc"]).read().splitlines()
    assert len(uc) == nr
    ncigar = 0
    for line, (head, ql, tl, r) in zip(uc, uc_want):
        f = line.split("\t")
        if head is None:
            assert line == f"N\t*\t*\t*\t.\t*\t*\t*\t{ql}\t*"
            continue
        assert "\t".join(f[:7]) == head and f[8:] == [ql, tl]
        if f[7] == "=":
            assert r.matches == r.alignment_length
        else:
            _cigar_agrees(f[7], r)
            ncigar += 1
    assert ncigar > 10_000
