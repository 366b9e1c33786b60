"""Search limits above the ranker's 1 024 shared-memory slots: --maxaccepts 0 --maxrejects 0 (every target), and any
maxaccepts + maxrejects + 8 > 1024.  The unbounded ranker must give search_topscores' lists element by element, the
search the reference's rows and search16 workload, the streaming driver the reference CLI's bytes and the search_batch
shim the reference library's records.  The reference's results are stored in tests/golden/exhaustive_reference.json
(made from the compiled reference, see _reference), so these tests need only the GPU."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import checkers
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
STOCK = os.path.join(REF, "vsearch")
RESULTS = os.path.join(ROOT, "tests", "golden", "exhaustive_reference.json")


def _reference(name, inputs, compute, available):
    """what the unmodified reference returned for `inputs`, keyed by `name` and a hash of the inputs.  With the compiled
    reference present and VSG_RECORD_REFERENCE=<file>, `compute()` runs it and the result is added to <file>; copying
    that file to RESULTS makes the record the tests use."""
    h = hashlib.sha256()
    checkers._feed(h, inputs)
    key = f"{name}:{h.hexdigest()[:24]}"
    out = os.environ.get("VSG_RECORD_REFERENCE")
    if out and available:
        val = checkers.canon(compute())
        rec = json.load(open(out)) if os.path.exists(out) else {}
        rec[key] = val
        with open(out, "w") as f:
            f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(rec[k], separators=(",", ":"))
                                        for k in sorted(rec)) + "\n}\n")
        return val
    stored = json.load(open(RESULTS))
    if key not in stored:
        raise AssertionError(f"no stored reference result {key} in {RESULTS}")
    return stored[key]


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def _families(n_fam, n_per, length, seed, fam_div=0.08, member_div=0.03):
    """one ancestor, n_fam families at fam_div from it, n_per members at member_div from their family: every member
    shares enough k-mers with every other to be a candidate, and --id 0.9 accepts about its own family only"""
    rng = np.random.default_rng(seed)
    root = synth.random_seqs(rng, 1, length)[0]
    fams = [synth.mutate(rng, root, fam_div) for _ in range(n_fam)]
    seqs = [synth.mutate(rng, fams[i % n_fam], member_div).tobytes() for i in range(n_fam * n_per)]
    return seqs, fams, rng


def _queries(rng, fams, n, length, n_random=0):
    qs = []
    for i in range(n):
        f = synth.mutate(rng, fams[i % len(fams)], 0.03)
        a = int(rng.integers(0, max(1, f.shape[0] - length)))
        qs.append(f[a: a + length].tobytes())
    qs += [synth.random_seqs(rng, 1, length)[0].tobytes() for _ in range(n_random)]
    return qs


# ---- 1. the unbounded ranker against search_topscores (oracle/ranker.c) ----------------------------------------------

def _ranker_db():
    rng = np.random.default_rng(71)
    root = synth.random_seqs(rng, 1, 150)[0]
    seqs = []
    for i in range(6000):                       # thousands tied on count and length
        s = root.copy()
        if i % 3 == 1:
            s[int(rng.integers(0, 150))] = synth.ACGT[int(rng.integers(0, 4))]
        seqs.append(s[: 150 - (i % 5)].tobytes())
    other = synth.random_seqs(rng, 60000, 90)
    seqs += [other[i].tobytes() for i in range(60000)]
    for j in range(60):                         # one family spread over all three shards
        seqs.insert(1100 * j + 7, synth.mutate(rng, root, 0.08).tobytes())
    long_q = b"".join(synth.mutate(rng, root, 0.05).tobytes() for _ in range(18))     # > 2 048 windows
    assert len(long_q) - 7 > 2048
    queries = [root.tobytes(), synth.mutate(rng, root, 0.04).tobytes(), root[:60].tobytes(), long_q,
               other[5].tobytes(), synth.random_seqs(rng, 1, 120)[0].tobytes()]
    # soft-masked stretches: with mask_lower they seed no k-mer
    queries.append(root[:50].tobytes() + root[50:110].tobytes().lower() + root[110:].tobytes())
    return seqs, queries


@pytest.mark.parametrize("k,mask_lower", [(8, 0), (8, 1), (12, 0)])
def test_unbounded_ranker_equals_the_oracle(ctx, k, mask_lower):
    seqs, queries = _ranker_db()
    dbs, qss = synth.SeqSet(seqs), synth.SeqSet(queries)
    n = len(seqs)
    assert n > 2 * 32766
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(dbs, k=k)
    long_seen = False
    for tophits in (1025, 4096, n):
        opts = checkers.search_opts(n, id=0.9, k=k, mask_lower=mask_lower)
        opts.tophits = tophits
        seqno, count, nc = ctx.rank(ix, qs, 0, len(queries), opts.minwordmatches, tophits, mask_lower)
        for i, q in enumerate(queries):
            s_, c_ = od.topscores(q, opts)
            assert nc[i] == len(s_), (tophits, i, nc[i], len(s_))
            assert seqno[i, :nc[i]].tolist() == s_.tolist() and count[i, :nc[i]].tolist() == c_.tolist(), (tophits, i)
            long_seen |= len(q) > 2000 and nc[i] > 0
    # the tied crowd fills the lists beyond 1 024, and cuts fall inside it
    seqno, count, nc = ctx.rank(ix, qs, 0, 1, checkers.MINWORDMATCHES[k], n, mask_lower)
    assert nc[0] > 4096 and count[0, 1024] == count[0, 1025]
    assert long_seen
    od.close(); ix.close(); db.close(); qs.close()


def test_unbounded_ranker_in_chunks_equals_one_chunk(ctx):
    """a device key budget far below the candidates: rank_lists emits, sorts and cuts consecutive query ranges one at a
    time (a single query over the budget alone), and the lists are those of one chunk"""
    seqs, queries = _ranker_db()
    queries = queries + queries[::-1]
    dbs, qss = synth.SeqSet(seqs), synth.SeqSet(queries)
    n = len(seqs)
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, 8, 0)
    want = ctx.rank(ix, qs, 0, len(queries), 12, n)
    old = os.environ.get("VSG_DIR_BUDGET_MB")
    os.environ["VSG_DIR_BUDGET_MB"] = "1"        # 1 MB / 4 / 24 B: about 10 900 keys per chunk
    try:
        small = vlib.Context(0)
    finally:
        if old is None:
            del os.environ["VSG_DIR_BUDGET_MB"]
        else:
            os.environ["VSG_DIR_BUDGET_MB"] = old
    db2 = small.seqset(dbs); qs2 = small.seqset(qss)
    ix2 = small.index(db2, 8, 0)
    for tophits in (n, 3000):
        got = small.rank(ix2, qs2, 0, len(queries), 12, tophits)
        ref = want if tophits == n else ctx.rank(ix, qs, 0, len(queries), 12, tophits)
        assert got[2].tolist() == ref[2].tolist()
        for i in range(len(queries)):
            m = int(ref[2][i])
            assert got[0][i, :m].tolist() == ref[0][i, :m].tolist() and got[1][i, :m].tolist() == ref[1][i, :m].tolist(), (tophits, i)
    assert int(np.sum(want[2])) > 3 * 10900
    ix2.close(); db2.close(); qs2.close(); small.close()
    ix.close(); db.close(); qs.close()


def test_search_cut_into_subbatches_by_candidate_volume(ctx):
    """800 queries with ~6 000 candidates each exceed one sub-batch's 2^22 candidates: the call is cut into several
    sub-batches, and its rows and work are those of the two halves searched on their own"""
    seqs, _ = _ranker_db()
    rng = np.random.default_rng(3)
    root = np.frombuffer(seqs[0], dtype=np.uint8)
    queries = [synth.mutate(rng, root, 0.03).tobytes() for _ in range(800)]
    dbs, qss = synth.SeqSet(seqs), synth.SeqSet(queries)
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, 8, 0)
    _, _, nc = ctx.rank(ix, qs, 0, len(queries), 12, len(seqs))
    assert int(nc.sum()) > (1 << 22) + 100000
    o = vlib.default_search_opts(); o.id = 0.97; o.maxaccepts = 0; o.maxrejects = 0
    hits, first, work = ctx.search_hits(ix, db, qs, 0, len(queries), o)
    parts = [ctx.search_hits(ix, db, qs, a, 400, o) for a in (0, 400)]
    assert first[-1] > 800
    assert np.diff(first).tolist() == np.diff(parts[0][1]).tolist() + np.diff(parts[1][1]).tolist()
    assert bytes(hits) == bytes(parts[0][0]) + bytes(parts[1][0])
    assert work[:2].tolist() == (parts[0][2][:2] + parts[1][2][:2]).tolist()
    assert int(work[0]) == int(nc.sum())      # nothing pre-rejected, no limit: every candidate is aligned
    ix.close(); db.close(); qs.close()


# ---- 2. the search against the compiled reference --------------------------------------------------------------------

def _search_data():
    seqs, fams, rng = _families(30, 100, 300, seed=5)
    queries = _queries(rng, fams, 150, 200)
    return synth.SeqSet(seqs), synth.SeqSet(queries)


def _ref_rows(name, dbs, qss, maxaccepts, maxrejects, strand_both):
    """the reference library's records (multi-threaded search_batch, every record) and its search16 pairs and cells.  The
    library takes the limits as given, so they arrive clamped to the database as the CLI would clamp them."""
    n = len(dbs)
    ma, mr = (maxaccepts or n), (maxrejects or n)

    def compute():
        r = checkers.RefDb(dbs, k=8, id=0.9, maxaccepts=ma, maxrejects=mr, strand_both=strand_both)
        checkers.ref().vsref_work_reset()
        counts, a = r.search_rows(qss, max_results=r.tophits * 2)
        pairs, cells, calls = (checkers.C.c_longlong() for _ in range(3))
        checkers.ref().vsref_work_get(checkers.C.byref(pairs), checkers.C.byref(cells), checkers.C.byref(calls))
        m = r.tophits * 2
        r.close()
        rows = [[[int(a["target"][q * m + j]), float(a["id"][q * m + j]), int(a["matches"][q * m + j]),
                  int(a["mismatches"][q * m + j]), int(a["gaps"][q * m + j]), int(a["alnlen"][q * m + j]),
                  int(a["accepted"][q * m + j]), int(a["strand"][q * m + j])] for j in range(int(counts[q]))]
                for q in range(len(qss))]
        return [checkers.digest(rows), [len(x) for x in rows], int(pairs.value), int(cells.value)]
    return _reference(name, (dbs, qss, ma, mr, strand_both), compute, checkers.ref() is not None)


def _rows(res, counts, stride):
    return [[[r.target, r.id, r.matches, r.mismatches, r.gaps, r.alignment_length, r.accepted, r.strand]
             for r in (res[q * stride + j] for j in range(int(counts[q])))] for q in range(len(counts))]


@pytest.mark.parametrize("maxaccepts,maxrejects,strand_both,lazy",
                         [(0, 0, 0, 0), (0, 0, 0, 1), (10, 0, 1, 0), (0, 32, 0, 0), (1500, 2500, 0, 0), (1500, 2500, 0, 1)])
def test_search_above_1024_candidates_equals_the_reference(ctx, maxaccepts, maxrejects, strand_both, lazy):
    dbs, qss = _search_data()
    digest, nrows, pairs, cells = _ref_rows("exhaustive_search", dbs, qss, maxaccepts, maxrejects, strand_both)
    n = len(dbs)
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, 8, 0)
    o = vlib.default_search_opts(); o.id = 0.9; o.maxaccepts = maxaccepts; o.maxrejects = maxrejects
    o.strand_both = strand_both; o.lazy = lazy
    # the queries have more candidates than the shared-memory ranker holds
    _, _, nc = ctx.rank(ix, qs, 0, len(qss), 12, n)
    assert np.median(nc) > 1024
    stride = 2 * n
    res, counts, work = ctx.search(ix, db, qs, 0, len(qss), o, stride)
    got = _rows(res, counts, stride)
    assert [len(x) for x in got] == nrows
    assert checkers.digest(got) == digest
    assert (int(work[0]), int(work[1])) == (pairs, cells)
    if not strand_both:
        checkers.check_search_rows(res, counts, stride, qss, dbs)
    # vsg_search_hits: the same rows back to back
    hits, first, work2 = ctx.search_hits(ix, db, qs, 0, len(qss), o)
    assert first[-1] == sum(nrows) and np.diff(first).tolist() == nrows
    flat = [x for q in got for x in q]
    assert [[h.target, h.id, h.matches, h.mismatches, h.gaps, h.alignment_length, h.accepted, h.strand] for h in hits[:first[-1]]] == flat
    assert bytes(hits)[: first[-1] * vlib.C.sizeof(vlib.SearchResult)] == b"".join(bytes(res[q * stride + j]) for q in range(len(qss)) for j in range(int(counts[q])))
    assert (int(work2[0]), int(work2[1])) == (pairs, cells)
    # a short buffer: VSG_ECAP and the number of rows needed
    nh = vlib.C.c_int64()
    short = (vlib.SearchResult * 4)()
    f2 = np.zeros(len(qss) + 1, dtype=np.int64)
    rc = vlib.load().vsg_search_hits(ctx.h, ix.h, db.h, qs.h, vlib.C.c_int64(0), vlib.C.c_int64(len(qss)), vlib.C.byref(o),
                                     vlib.C.c_int64(0), short, vlib.C.c_int64(4), vlib._ptr(f2, vlib.C.c_int64), vlib.C.byref(nh), None)
    assert rc == -5 and nh.value == first[-1] and f2.tolist() == first.tolist()
    # maxhits cuts every list
    hits3, first3, _ = ctx.search_hits(ix, db, qs, 0, len(qss), o, maxhits=3)
    assert np.diff(first3).tolist() == [min(3, x) for x in nrows]
    ix.close(); db.close(); qs.close()


# ---- 3. the streaming driver against the reference CLI ---------------------------------------------------------------

def _stream_files(tmp_path, n_db, n_q):
    seqs, fams, rng = _families(max(1, n_db // 100), min(100, n_db), 300, seed=17)
    seqs = seqs[:n_db]
    qs = _queries(rng, fams, n_q, 200, n_random=4)
    dbs = synth.SeqSet(seqs)
    dbf = str(tmp_path / "db.fasta"); qf = str(tmp_path / "q.fasta")
    synth.write_fasta(dbf, dbs, "d")
    synth.write_fasta(qf, synth.SeqSet(qs), "q")
    return dbs, dbf, qf, [f"d{i}" for i in range(len(dbs))]


@pytest.mark.parametrize("mode,n_db", [("exhaustive", 3000), ("ten_both_no_hits", 3000), ("dust_maxhits", 3000),
                                       ("exhaustive", 500)])
def test_stream_without_limits_equals_the_reference_cli(tmp_path, mode, n_db):
    dbs, dbf, qf, labels = _stream_files(tmp_path, n_db, 100)
    ref_out = str(tmp_path / "ref.b6"); got_out = str(tmp_path / "got.b6")
    args = ["--usearch_global", qf, "--db", dbf, "--id", "0.9", "--blast6out", ref_out, "--threads", "1", "--quiet"]
    o = vlib.default_search_opts(); o.id = 0.9
    kw = {}
    dust = 0
    if mode == "exhaustive":
        args += ["--qmask", "none", "--dbmask", "none", "--maxaccepts", "0", "--maxrejects", "0"]
        o.maxaccepts = 0; o.maxrejects = 0
    elif mode == "ten_both_no_hits":
        args += ["--qmask", "none", "--dbmask", "none", "--maxaccepts", "10", "--maxrejects", "0", "--strand", "both",
                 "--output_no_hits"]
        o.maxaccepts = 10; o.maxrejects = 0; o.strand_both = 1
        kw = dict(output_no_hits=1)
    else:
        args += ["--maxaccepts", "0", "--maxrejects", "0", "--maxhits", "5"]      # default masking: dust on both sides
        o.maxaccepts = 0; o.maxrejects = 0; o.mask_lower = 1; o.qmask_dust = 1
        dust = 1
        kw = dict(maxhits=5, qmask_dust=1)
    nwant, want = _reference("exhaustive_stream", (open(qf, "rb").read(), open(dbf, "rb").read(), args[4:6] + args[8:]),
                             lambda: checkers.run_stock(args, [ref_out], lambda t: (len(t), checkers.digest(t))),
                             os.path.exists(STOCK))
    g = vlib.Group([0], dbs, wordlength=8, mask_lower=dust, dust_db=dust)
    st = g.stream(labels, qf, o, got_out, batch_queries=40, **kw)
    g.close()
    got = open(got_out, "rb").read()
    assert st["queries"] == 104
    assert st["rows"] >= 100 * (5 if mode == "dust_maxhits" else 10)
    assert len(got) == nwant and checkers.digest(got) == want


# ---- 4. the search_batch shim (seam 2) with limits above 1 024 -------------------------------------------------------

@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "seam2_driver_gpu")),
                    reason="oracle/_ref (compiled reference + shims) not present")
@pytest.mark.parametrize("case", [
    ["id=0.9", "maxaccepts=2000", "maxrejects=3000", "max_results=64"],
    # the sequence-content filters on the unbounded lists, both strands (flags per strand's list)
    ["id=0.9", "maxaccepts=2000", "maxrejects=3000", "max_results=64", "idprefix=4", "idsuffix=3", "selfid=1", "strand=1"],
])
def test_search_batch_shim_with_large_limits_equals_reference(tmp_path, case):
    seqs, fams, rng = _families(20, 80, 300, seed=29)
    qs = _queries(rng, fams, 60, 300) + seqs[5:8]      # three queries identical to a target (--selfid)
    dbf, qf = str(tmp_path / "db.fasta"), str(tmp_path / "q.fasta")
    synth.write_fasta(dbf, synth.SeqSet(seqs), "d")
    synth.write_fasta(qf, synth.SeqSet(qs), "q")
    outs = []
    for exe in ("seam2_driver_ref", "seam2_driver_gpu"):
        r = subprocess.run([os.path.join(REF, exe), dbf, qf] + case, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (exe, r.stdout[-2000:], r.stderr[-2000:])
        outs.append(r.stdout.splitlines())
    assert len(outs[0]) > 60 * 20
    assert outs[0] == outs[1], [x for x in zip(outs[0], outs[1]) if x[0] != x[1]][:5]
