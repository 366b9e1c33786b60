"""vsg_search_exact and vsg_search_exact_command on the GPU.  The command: every output file of every case of
search_exact_cases.py equals the reference CLI's (sha256, tests/golden/search_exact_reference.json), also with batches
of 7 queries and with hashes cut to 6 bits (VSG_EXACT_HASH_BITS, so most candidates are collisions the comparison must
reject); with oracle/_ref/vsearch present the reference's files are made afresh too; each refusal leaves no file.  The
library call: record by record against a dictionary lookup in Python, at 200 000 queries and 100 000 targets of up to
50 000 nt, with a too-small cap, and over 3 000 identical targets."""
import bz2
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

import search_exact_cases as cases
from vsearch_b200 import lib as vlib

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def _run_case(ctx, tmp_path, name, **extra):
    inp, cli, kw, outputs = cases.CASES[name]
    q, db = cases.input_files(inp, str(tmp_path))
    want = cases.golden()[name]
    assert cases.sha256(q) == want["query_sha256"] and cases.sha256(db) == want["db_sha256"]
    mine = tmp_path / "mine"
    mine.mkdir(exist_ok=True)
    paths = cases.output_files(str(mine), name, outputs)
    st = ctx.search_exact_command(q, db, **paths, **kw, **extra)
    assert cases.output_digests(paths) == want["files"]
    assert (st["matched"], st["queries"]) == (want["matched"], want["queries"])
    return q, db, want


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_search_exact_command_equals_reference_cli(ctx, tmp_path, name):
    q, db, want = _run_case(ctx, tmp_path, name)
    if os.path.exists(cases.STOCK):
        inp, cli, kw, outputs = cases.CASES[name]
        ref = tmp_path / "ref"
        ref.mkdir()
        rpaths = cases.output_files(str(ref), name, outputs)
        counts = cases.reference_run(q, db, cli, rpaths)
        assert cases.output_digests(rpaths) == want["files"]
        assert counts == {k: want[k] for k in counts}


@pytest.mark.parametrize("name", ["a_default", "b_strand_both", "c_dups_all", "o_edges", "p_fastq"])
@pytest.mark.parametrize("batch", [7, 65536])
def test_search_exact_command_batches(ctx, tmp_path, name, batch):
    _run_case(ctx, tmp_path, name, batch_queries=batch)


_COLLIDING = """
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import search_exact_cases as cases
from vsearch_b200 import lib as vlib
ctx = vlib.Context(0)
bad = []
for name in {names!r}:
    inp, cli, kw, outputs = cases.CASES[name]
    q, db = cases.input_files(inp, {d!r})
    paths = cases.output_files({d!r}, name, outputs)
    ctx.search_exact_command(q, db, **paths, **kw)
    if cases.output_digests(paths) != cases.golden()[name]["files"]:
        bad.append(name)
ctx.close()
print("BAD", bad)
sys.exit(1 if bad else 0)
"""


def test_search_exact_command_colliding_hashes(tmp_path):
    # the knob is read when an index is made, in a process of its own so no other test sees it
    names = ["a_default", "b_strand_both", "c_dups_all", "e_symbols_none", "g_hardmask"]
    code = _COLLIDING.format(tests=HERE, root=os.path.dirname(HERE), names=names, d=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, VSG_EXACT_HASH_BITS="6"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


def _refused(ctx, tmp_path, q, db, match, **kw):
    out = tmp_path / "out"
    out.mkdir(exist_ok=True)
    paths = {} if kw.pop("no_outputs", False) else cases.output_files(str(out), "x", cases.OUTPUTS)
    with pytest.raises(vlib.VsgError, match=match) as e:
        ctx.search_exact_command(q, db, **paths, **kw)
    assert "(-3)" in str(e.value)          # VSG_EINVAL
    assert sorted(os.listdir(out)) == []


def test_search_exact_command_refusals(ctx, tmp_path):
    q, db = cases.input_files("amplicons", str(tmp_path))
    _refused(ctx, tmp_path, q, db, "No output", no_outputs=True)
    for path, comp, what in ((q, gzip.compress, "gzip"), (q, bz2.compress, "bzip2")):
        z = tmp_path / f"q.{what}"
        z.write_bytes(comp(open(path, "rb").read()))
        _refused(ctx, tmp_path, str(z), db, what)
        _refused(ctx, tmp_path, q, str(z), what)
    udb = tmp_path / "db.udb"
    ctx.udb_make([b"ACGT" * 20, b"GGCA" * 30], ["a", "b"]).write(str(udb))
    _refused(ctx, tmp_path, q, str(udb), "UDB")
    _refused(ctx, tmp_path, q, db, "hardmask", hardmask=1)
    _refused(ctx, tmp_path, q, db, "hardmask", hardmask=1, qmask="soft")
    _refused(ctx, tmp_path, q, db, "hardmask", hardmask=1, dbmask="soft")
    _refused(ctx, tmp_path, str(tmp_path / "missing.fa"), db, "cannot open")
    _refused(ctx, tmp_path, q, str(tmp_path / "missing.fa"), "cannot open")


# ---- the library call against a dictionary lookup ------------------------------------------------------------------

_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def _expected(queries, targets, strand_both, maxhits=0):
    index = {}
    for t, s in enumerate(targets):
        index.setdefault(s, []).append(t)
    out = []
    for q in queries:
        hits = [(t, 0) for t in index.get(q, [])]
        if strand_both:
            hits += [(t, 1) for t in index.get(q.translate(_COMP)[::-1], [])]
        hits.sort(key=lambda h: h[0])
        out.append(hits[:maxhits] if maxhits else hits)
    return out


def _check_rows(rows, first, want, queries, match=2):
    assert int(first[-1]) == sum(len(w) for w in want)
    for i, w in enumerate(want):
        got = rows[int(first[i]):int(first[i + 1])]
        assert [(r.target, r.strand) for r in got] == w, i
        L = len(queries[i])
        for r in got:
            assert (r.matches, r.mismatches, r.gaps, r.alignment_length, r.query_length, r.target_length, r.accepted, r.nwscore,
                    r.id, r.internal_alignment_length, r.internal_gaps) == (L, 0, 0, L, L, L, 1, L * match, 100.0, L, 0)


class _Seqs:
    """the arrays Context.seqset uploads"""

    def __init__(self, seqs):
        self.cat = np.frombuffer(b"".join(seqs) + b"\0", dtype=np.uint8)
        self.lens = np.array([len(s) for s in seqs], dtype=np.int32)
        self.offs = np.zeros(len(seqs), dtype=np.int64)
        if len(seqs) > 1:
            self.offs[1:] = np.cumsum(self.lens[:-1], dtype=np.int64)


def test_search_exact_library_at_scale(ctx):
    rng = np.random.default_rng(7)
    lens = np.concatenate([rng.integers(50, 600, size=99_990), rng.integers(20_000, 50_001, size=10)])
    alphabet = np.frombuffer(b"ACGT", dtype=np.uint8)
    targets = [alphabet[rng.integers(0, 4, size=int(n))].tobytes() for n in lens]
    for k in range(0, 2000, 2):   # some targets repeated under other numbers
        targets[50_000 + k] = targets[k]
    queries = []
    for i in range(200_000):
        t = targets[int(rng.integers(0, len(targets)))]
        u = i % 10
        if u < 5:
            queries.append(t)
        elif u < 7:
            queries.append(t.translate(_COMP)[::-1])
        elif u < 9:
            b = bytearray(t)
            p = int(rng.integers(0, len(b)))
            b[p] = b"CGTA"[b"ACGT".index(b[p])]   # one substitution
            queries.append(bytes(b))
        else:
            queries.append(alphabet[rng.integers(0, 4, size=len(t))].tobytes())
    db = ctx.seqset(_Seqs(targets))
    qs = ctx.seqset(_Seqs(queries))
    ix = ctx.exact_index(db)
    try:
        for strand_both in (0, 1):
            o = vlib.default_search_opts()
            o.strand_both = strand_both
            want = _expected(queries, targets, strand_both)
            rows, first, _ = ctx.search_exact(ix, qs, 0, len(queries), o)
            _check_rows(rows, first, want, queries)
        # maxhits, and a query range inside the set
        o.strand_both = 1
        rows, first, _ = ctx.search_exact(ix, qs, 1000, 5000, o, maxhits=1)
        _check_rows(rows, first, _expected(queries[1000:6000], targets, 1, maxhits=1), queries[1000:6000])
        # a cap too small: VSG_ECAP with the right count and first[]
        n = int(first[-1])
        with pytest.raises(vlib.VsgError, match=r"\(-5\)"):
            ctx.search_exact(ix, qs, 1000, 5000, o, maxhits=1, cap=n - 1)
    finally:
        ix.close()
        qs.close()
        db.close()


def test_search_exact_library_identical_targets(ctx):
    rng = np.random.default_rng(8)
    alphabet = np.frombuffer(b"ACGT", dtype=np.uint8)
    same = alphabet[rng.integers(0, 4, size=250)].tobytes()
    others = [alphabet[rng.integers(0, 4, size=250)].tobytes() for _ in range(500)]
    targets = others[:250] + [same] * 3000 + others[250:]
    queries = [same, same.translate(_COMP)[::-1], others[3], b"", same[:-1]]
    db = ctx.seqset(_Seqs(targets))
    qs = ctx.seqset(_Seqs(queries))
    ix = ctx.exact_index(db)
    try:
        o = vlib.default_search_opts()
        o.strand_both = 1
        rows, first, _ = ctx.search_exact(ix, qs, 0, len(queries), o)
        _check_rows(rows, first, _expected(queries, targets, 1), queries)
        assert int(first[1]) == 3000
        rows, first, _ = ctx.search_exact(ix, qs, 0, len(queries), o, maxhits=5)
        _check_rows(rows, first, _expected(queries, targets, 1, maxhits=5), queries)
    finally:
        ix.close()
        qs.close()
        db.close()
