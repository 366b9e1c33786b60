"""Every --wordlength from 3 to 15 on the device against the oracle: the k-mer index and the ranker (the dense index of
3..10 with its shared-memory bitmaps and the HBM de-duplication of long queries, the sparse index of 11..15), dense
indexes over three shards, whole searches under each word length's default minwordmatches, the reference's cap of
32 767 on a target's k-mer count, the longest query the ranker takes, the orientation vote on one and on three shards,
and clustering at word lengths 5 and 10 against the reference CLI's stored records."""

import numpy as np
import pytest

import checkers
import orient_cases as oc
from test_cluster_gpu import _reads, device_records, reference_records
from test_search_gpu import gpu_opts, rows_of
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu

KS = list(range(3, 16))
KMER_CAP = 2048          # distinct k-mers a query holds in shared memory (rank_steps.cuh); longer queries go through HBM
SHARD = 32766            # targets per static index shard
COUNT_CAP = 32767        # a target's k-mer count saturates here (searchcore.cpp:306-315)
IUPAC = np.frombuffer(b"NRYSWKMBDHV", dtype=np.uint8)


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def rank_opts(k, tophits, mask_lower=0):
    o = checkers.search_opts(1, k=k, mask_lower=mask_lower)
    o.tophits = tophits
    return o


def check_lists(ctx, ix, qs, od, queries, k, tophits, mask_lower=0):
    """the device's candidate lists of every query equal the oracle's, element by element; returns the oracle's"""
    o = rank_opts(k, tophits, mask_lower)
    seqno, count, nc = ctx.rank(ix, qs, 0, len(queries), o.minwordmatches, tophits, mask_lower)
    want = []
    for i, q in enumerate(queries):
        s, c = od.topscores(q, o)
        assert nc[i] == len(s), (k, tophits, mask_lower, i, int(nc[i]), len(s))
        assert seqno[i, :nc[i]].tolist() == s.tolist() and count[i, :nc[i]].tolist() == c.tolist(), (k, tophits, mask_lower, i)
        want.append((s, c))
    return want


def soft_mask(rng, s, n=40):
    b = bytearray(s)
    a = int(rng.integers(0, max(1, len(b) - n)))
    b[a:a + n] = bytes(b[a:a + n]).lower()
    return bytes(b)


def with_iupac(rng, s, n=6):
    a = np.frombuffer(s, dtype=np.uint8).copy()
    a[rng.integers(0, a.shape[0], size=n)] = IUPAC[rng.integers(0, IUPAC.shape[0], size=n)]
    return a.tobytes()


def mixed_case(k):
    """(database, queries, roots) of one shard: families of 2-10 % variants, unrelated sequences, soft-masked stretches
    and IUPAC symbols, an empty target and targets of k - 1 and k nt; queries of family members, a soft-masked and an
    IUPAC one, k - 1 and k nt, 2 047 + k and 2 048 + k nt (the two sides of KMER_CAP) and ~6 000 nt of repeats"""
    rng = np.random.default_rng(500 + k)
    roots = synth.random_seqs(rng, 30, 400)
    seqs = [synth.mutate(rng, roots[i % 30], float(rng.uniform(0.02, 0.1))).tobytes() for i in range(2400)]
    seqs += [r.tobytes() for r in synth.random_seqs(rng, 600, 300)]
    for i in range(0, len(seqs), 13):
        seqs[i] = soft_mask(rng, seqs[i])
    for i in range(5, len(seqs), 17):
        seqs[i] = with_iupac(rng, seqs[i])
    r0 = roots[0].tobytes()
    seqs[100], seqs[1000], seqs[2000] = b"", r0[:k - 1], r0[:k]
    queries = [synth.mutate(rng, roots[i], 0.03).tobytes() for i in range(12)]
    queries += [soft_mask(rng, roots[12].tobytes(), 150), with_iupac(rng, roots[13].tobytes(), 12), r0[:k - 1], r0[:k]]
    flank = synth.random_seqs(rng, 1, 2048 + k)[0].tobytes()
    for n in (2047 + k, 2048 + k):
        queries.append((roots[14].tobytes() + flank)[:n])
    queries.append((roots[15].tobytes() + roots[16].tobytes() + roots[17].tobytes()[:200]) * 6)
    assert [len(q) - k + 1 for q in queries[-3:-1]] == [KMER_CAP, KMER_CAP + 1] and len(queries[-1]) == 6000
    return synth.SeqSet(seqs), queries, roots


@pytest.mark.parametrize("k", KS)
def test_ranker_every_wordlength_vs_oracle(ctx, k):
    dbs, queries, _ = mixed_case(k)
    n = len(dbs)
    db = ctx.seqset(dbs); qs = ctx.seqset(synth.SeqSet(queries))
    for mask_lower in (0, 1):
        ix = ctx.index(db, k, mask_lower)
        od = checkers.OracleDb(dbs, k=k, mask_lower=mask_lower)
        for tophits in (1, 8, 1024, 1025, n):
            want = check_lists(ctx, ix, qs, od, queries, k, tophits, mask_lower)
            if tophits == n:
                full = want
        # the k-nt query finds the k-nt target; family members find their family
        assert 2000 in full[15][0].tolist() and all(len(full[i][0]) >= 60 for i in range(12)), k
        if k == 3:
            # nearly every target holds every 3-mer: far more than 1 024 targets tie at the 1 024-th count
            ties = [int((c == c[1023]).sum()) for s, c in full if len(c) > 1024]
            assert ties and max(ties) > 1024, ties
        od.close(); ix.close()
    db.close(); qs.close()


@pytest.mark.parametrize("k", [3, 6, 9, 10])
def test_dense_index_over_three_shards_vs_oracle(ctx, k):
    """70 000 short targets, three static shards; one family spread over all of them"""
    rng = np.random.default_rng(600 + k)
    m = synth.random_seqs(rng, 70_000, 100)
    root = synth.random_seqs(rng, 1, 100)[0]
    fam = np.arange(7, 70_000, 500)
    m[fam] = root
    sub = rng.random((fam.shape[0], 100)) < 0.03
    m[fam] = np.where(sub, synth.ACGT[rng.integers(0, 4, size=(fam.shape[0], 100))], m[fam])
    dbs = synth.SeqSet.from_matrix(m)
    queries = [root.tobytes(), synth.mutate(rng, root, 0.03).tobytes(), synth.random_seqs(rng, 1, 100)[0].tobytes(),
               synth.random_seqs(rng, 1, 1250)[0].tobytes() + root.tobytes() + synth.random_seqs(rng, 1, 1250)[0].tobytes(),
               root[:k].tobytes()]
    db = ctx.seqset(dbs); qs = ctx.seqset(synth.SeqSet(queries))
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(dbs, k=k)
    for tophits in (1, 8, 1024, 1025, len(dbs)):
        want = check_lists(ctx, ix, qs, od, queries, k, tophits)
    s = want[0][0]
    assert len(dbs) > 2 * SHARD and {int(t) // SHARD for t in s if t % 500 == 7} == {0, 1, 2}
    od.close(); ix.close(); db.close(); qs.close()


def search_case(k):
    """families of 2-10 % variants and unrelated targets with soft-masked and IUPAC symbols; queries of family members
    and short random reads (at k = 3 their targets' counts spread around minwordmatches 18)"""
    rng = np.random.default_rng(700 + k)
    roots = [synth.random_seqs(rng, 1, int(rng.integers(150, 400)))[0] for _ in range(40)]
    seqs = [synth.mutate(rng, roots[i % 40], float(rng.uniform(0.02, 0.1))).tobytes() for i in range(320)]
    seqs += [synth.random_seqs(rng, 1, int(rng.integers(60, 300)))[0].tobytes() for _ in range(80)]
    for i in range(0, len(seqs), 11):
        seqs[i] = soft_mask(rng, seqs[i])
    for i in range(3, len(seqs), 19):
        seqs[i] = with_iupac(rng, seqs[i], 3)
    queries = [synth.mutate(rng, roots[i], 0.03).tobytes() for i in range(40)]
    short = [synth.random_seqs(rng, 1, int(rng.integers(26, 34)))[0].tobytes() for _ in range(8)]
    return synth.SeqSet(seqs), queries, short


def check_search(ctx, ix, db, dbs, queries, k, mask_lower, maxaccepts, maxrejects):
    qss = synth.SeqSet(queries)
    qs = ctx.seqset(qss)
    od = checkers.OracleDb(dbs, k=k, mask_lower=mask_lower)
    opts = checkers.search_opts(len(dbs), id=0.9, maxaccepts=maxaccepts, maxrejects=maxrejects, k=k, mask_lower=mask_lower)
    o = gpu_opts(0.9, maxaccepts, maxrejects, mask_lower=mask_lower, k=k)
    assert o.minwordmatches < 0     # the driver takes minwordmatches_defaults[k]
    res, counts, work = ctx.search(ix, db, qs, 0, len(queries), o, opts.tophits)
    pairs = cells = rows = 0
    for i, q in enumerate(queries):
        hits, p, cl = od.search(q, opts)
        pairs += p; cells += cl
        want = [[h.target, h.id, h.matches, h.mismatches, h.nwgaps, h.nwalignmentlength, h.accepted, h.strand] for h in hits]
        assert rows_of(res, counts, i, opts.tophits) == want, (k, mask_lower, i)
        rows += len(want)
    assert (int(work[0]), int(work[1])) == (pairs, cells), k
    checkers.check_search_rows(res, counts, opts.tophits, qss, dbs)
    od.close(); qs.close()
    return rows


@pytest.mark.parametrize("k", KS)
def test_search_every_wordlength_vs_oracle(ctx, k):
    dbs, queries, short = search_case(k)
    db = ctx.seqset(dbs)
    for mask_lower in (0, 1):
        ix = ctx.index(db, k, mask_lower)
        assert check_search(ctx, ix, db, dbs, queries, k, mask_lower, 2, 16) > 30
        # short reads with a reject budget as large as the database: every candidate is aligned, so one target more or
        # less at the k-mer threshold changes the workload
        check_search(ctx, ix, db, dbs, short, k, mask_lower, 1, len(dbs) - 20)
        ix.close()
    if k == 3:
        od = checkers.OracleDb(dbs, k=3)
        at18 = [len(od.topscores(q, rank_opts(3, len(dbs)))[0]) for q in short]
        o17 = rank_opts(3, len(dbs)); o17.minwordmatches = 17
        at17 = [len(od.topscores(q, o17)[0]) for q in short]
        od.close()
        assert any(a != b for a, b in zip(at17, at18)), (at17, at18)
    db.close()


@pytest.mark.parametrize("k", [9, 10, 12, 15])
def test_count_cap_vs_oracle(ctx, k):
    """a 40 000-nt query with more than 32 767 distinct k-mers against exact copies of itself and copies one and two
    bases longer (all saturate at 32 767, so length then seqno decides), a copy with its second half mutated (below the
    cap) and 1 500 unrelated short targets (tophits = n takes the unbounded ranker)"""
    rng = np.random.default_rng(800 + k)
    q = synth.random_seqs(rng, 1, 40_000)[0]
    nk = checkers.oracle_unique_kmers(q.tobytes(), k).shape[0]
    assert nk > COUNT_CAP, nk
    seqs = [r.tobytes() for r in synth.random_seqs(rng, 1500, 200)]
    half = np.concatenate([q[:20_000], synth.mutate(rng, q[20_000:], 0.3)]).tobytes()
    exact, plus1, plus2, mutated = [40, 700, 1300], [10, 900], [5, 1100], 600
    for i in exact:
        seqs[i] = q.tobytes()
    for i in plus1:
        seqs[i] = q.tobytes() + b"A"
    for i in plus2:
        seqs[i] = b"GT" + q.tobytes()
    seqs[mutated] = half
    dbs = synth.SeqSet(seqs)
    queries = [q.tobytes(), q[:3000].tobytes()]
    db = ctx.seqset(dbs); qs = ctx.seqset(synth.SeqSet(queries))
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(dbs, k=k)
    for tophits in (1, 8, 1024, 1025, len(dbs)):
        s, c = check_lists(ctx, ix, qs, od, queries, k, tophits)[0]
        top = exact + plus1 + plus2
        assert s[:len(top)].tolist() == top[:tophits] and (c[:len(top)] == COUNT_CAP).all(), (tophits, s[:8], c[:8])
        if tophits > len(top):
            assert s[len(top)] == mutated and c[len(top)] < COUNT_CAP, (s[len(top)], c[len(top)])
    od.close(); ix.close(); db.close(); qs.close()


@pytest.mark.parametrize("k", [3, 8, 15])
def test_longest_query_the_ranker_takes(ctx, k):
    """65 535 windows (65 534 + k nt) rank and equal the oracle's list; one window more is refused"""
    rng = np.random.default_rng(900 + k)
    q = synth.random_seqs(rng, 1, 65_535 + k)[0]
    seqs = [r.tobytes() for r in synth.random_seqs(rng, 1100, 400)]
    seqs[17] = q[:40_000].tobytes()
    seqs[500] = synth.mutate(rng, q[1000:1400], 0.02).tobytes()
    dbs = synth.SeqSet(seqs)
    db = ctx.seqset(dbs)
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(dbs, k=k)
    ok = [q[:65_534 + k].tobytes()]
    qs = ctx.seqset(synth.SeqSet(ok))
    for tophits in (8, len(dbs)):
        s, c = check_lists(ctx, ix, qs, od, ok, k, tophits)[0]
        # at k = 3 every target holds all 64 3-mers and the shortest come first
        assert k == 3 or (s[0] == 17 and c[0] == min(COUNT_CAP, checkers.oracle_unique_kmers(seqs[17], k).shape[0])), s[:4]
    qs.close()
    qs = ctx.seqset(synth.SeqSet([b"ACGT" * 100, q.tobytes()]))
    for tophits in (8, len(dbs)):
        with pytest.raises(vlib.VsgError, match=r"\(-3\).*longer than the device ranker supports"):
            ctx.rank(ix, qs, 0, 2, checkers.MINWORDMATCHES[k], tophits)
    od.close(); ix.close(); db.close(); qs.close()


def orient_check(ctx, dbs, k, mask_lower, queries, want):
    db = ctx.seqset(dbs)
    ix = ctx.index(db, k, mask_lower)
    qs = ctx.seqset(synth.SeqSet(queries))
    got = ctx.orient(ix, qs, 0, len(queries), query_mask_lower=mask_lower)
    qs.close(); ix.close(); db.close()
    bad = [i for i in range(len(queries)) if got[i].tolist() != want[i]]
    assert not bad, (k, mask_lower, len(bad), bad[:3], [got[i].tolist() for i in bad[:3]], [want[i] for i in bad[:3]])


@pytest.mark.parametrize("k", KS)
def test_orient_every_wordlength(ctx, k):
    """the orient fixture, on which reads are oriented from k = 7 on, and the strand-biased one, on which they are at
    every k, both ways"""
    d, b = oc.data(), oc.biased_data()
    for mask_lower in (0, 1):
        want = oc.orient_rows(d["q_seqs"], k, mask_lower, *oc.word_counts(d["db_seqs"], k, mask_lower))
        if k >= 7:
            assert {r[0] for r in want} == {0, 1, 2}, (k, mask_lower)
        orient_check(ctx, synth.SeqSet(d["db_seqs"]), k, mask_lower, d["q_seqs"], want)
        want = oc.orient_rows(b["q_seqs"], k, mask_lower, *oc.word_counts(b["db_seqs"], k, mask_lower))
        r = np.array(want)
        assert set(r[:, 0]) == {0, 1, 2} and (r[:, 1] > 0).sum() > 20 and (r[:, 2] > 0).sum() > 20, (k, mask_lower)
        orient_check(ctx, synth.SeqSet(b["db_seqs"]), k, mask_lower, b["q_seqs"], want)


_COMP = np.arange(256, dtype=np.uint8)
_COMP[np.frombuffer(b"ACGTacgt", dtype=np.uint8)] = np.frombuffer(b"TGCAtgca", dtype=np.uint8)


def matrix_word_counts(m, k, skip_lower):
    """oc.word_counts of the rows of an (n, L) ASCII matrix, vectorised: (sorted k-mers, rows holding each)"""
    code = oc._CODE[m]
    bad = code < 0
    if skip_lower:
        bad |= (m >= ord("a")) & (m <= ord("z"))
    w = m.shape[1] - k + 1
    v = np.zeros((m.shape[0], w), dtype=np.int64)
    nbad = np.zeros((m.shape[0], w), dtype=np.int64)
    for j in range(k):
        v = (v << 2) | np.maximum(code[:, j:j + w], 0)
        nbad += bad[:, j:j + w]
    v = np.where(nbad == 0, v, -1)
    v.sort(axis=1)
    keep = v >= 0
    keep[:, 1:] &= v[:, 1:] != v[:, :-1]
    return np.unique(v[keep], return_counts=True)


def three_shard_orient_db():
    """the strand-biased fixture's 300 targets repeated to 70 000 with 1 % substitutions.  Copies of every 25th target
    are reverse-complemented in shard 1 and of every 5th in shard 2: the reads of those targets lose their votes only
    with the later shards counted, and at small k, where a k-mer's counts come from the whole composition, some k-mer
    ratios cross the 8x rule only then"""
    rng = np.random.default_rng(95)
    src = oc.biased_data()["db"]
    n = 70_000
    pick = np.arange(n) % src.shape[0]
    m = src[pick]
    sub = rng.random(m.shape) < 0.01
    m = np.where(sub, synth.ACGT[rng.integers(0, 4, size=m.shape)], m)
    shard = np.arange(n) // SHARD
    flip = ((pick % 25 == 0) & (shard == 1)) | ((pick % 5 == 0) & (shard == 2))
    m[flip] = _COMP[m[flip]][:, ::-1]
    return m


@pytest.mark.parametrize("k", [5, 10, 11, 15])
def test_orient_three_shards(ctx, k):
    m = three_shard_orient_db()
    assert m.shape[0] > 2 * SHARD
    q = oc.biased_data()["q_seqs"]
    for mask_lower in (0, 1):
        want = oc.orient_rows(q, k, mask_lower, *matrix_word_counts(m, k, mask_lower))
        r = np.array(want)
        assert (r[:, 1] > 0).sum() > 20 and (r[:, 2] > 0).sum() > 20, (k, mask_lower)
        # some rows hold only with the second and with the third shard counted
        assert oc.orient_rows(q, k, mask_lower, *matrix_word_counts(m[:SHARD], k, mask_lower)) != want
        assert oc.orient_rows(q, k, mask_lower, *matrix_word_counts(m[:2 * SHARD], k, mask_lower)) != want
        orient_check(ctx, synth.SeqSet.from_matrix(np.ascontiguousarray(m)), k, mask_lower, q, want)


def cluster_reference(k, tmp):
    """the reads, their labels and `vsearch --cluster_fast --wordlength k --threads 8` (stored): (clusters, digest of
    the S/H records)"""
    seqs = _reads(1500, 40, seed=300 + k)
    labels = [f"w{i:05d}" for i in range(len(seqs))]
    want = reference_records(tmp, "cluster_fast_wordlength", (seqs, labels, 0.97, 8, k), seqs, labels,
                             ["--id", "0.97", "--threads", "8", "--wordlength", str(k)])
    return seqs, labels, want


@pytest.mark.parametrize("k", [5, 10])
def test_cluster_fast_wordlength_equals_reference_cli(tmp_path, k):
    seqs, labels, (nclusters, want) = cluster_reference(k, str(tmp_path))
    ncl, got, work = device_records(seqs, labels, 0.97, 8, wordlength=k)
    assert ncl == nclusters and 1 < ncl < len(seqs)
    assert got == want
