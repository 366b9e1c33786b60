"""The ranker's short-query instance (rank_kernel<RankShort>, three CTAs per SM) against its full instance and the
oracle.  vsg_rank takes the short instance when tophits <= 64 and every query of the call has np2 + nwin + 1 <= 512
(nwin: its windows, np2: nwin rounded up to a power of two).  Every case ranks its queries alone, and again with one
3 000-nt query appended, which sends the whole call to the full instance; each query's row (targets, counts, length)
must be the same in both calls and equal to the oracle's search_topscores."""

import numpy as np
import pytest

import checkers
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu

SHORT_SLOTS = 512       # RankShort::KCAP (rank.cu)
SHORT_TOPHITS = 64      # RankShort::TOPHITS
SHORT_CAND = 256        # RankShort::CAND: more ties than this take the sort-and-cut scan
IUPAC = np.frombuffer(b"NRYSWKMBDHV", dtype=np.uint8)


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def fits_short(qlen, k):
    nwin = max(1, qlen - k + 1)
    np2 = 1
    while np2 < nwin:
        np2 *= 2
    return np2 + nwin + 1 <= SHORT_SLOTS


def longest_short(k):
    """the longest query the short instance takes at word length k (255 windows)"""
    n = max(n for n in range(k, 700) if fits_short(n, k))
    assert n - k + 1 == 255
    return n


def long_query(seed=1):
    return synth.random_seqs(np.random.default_rng(seed), 1, 3000)[0].tobytes()


def rank_opts(k, tophits, mask_lower=0):
    o = checkers.search_opts(1, k=k, mask_lower=mask_lower)
    o.tophits = tophits
    return o


def check_short_and_full(ctx, ix, od, k, queries, tophits, mask_lower=0):
    """ranks `queries` alone and with a 3 000-nt query appended; both equal the oracle, query by query"""
    o = rank_opts(k, tophits, mask_lower)
    n = len(queries)
    alone = ctx.seqset(synth.SeqSet(queries))
    plus = ctx.seqset(synth.SeqSet(queries + [long_query()]))
    a = ctx.rank(ix, alone, 0, n, o.minwordmatches, tophits, mask_lower)
    b = ctx.rank(ix, plus, 0, n + 1, o.minwordmatches, tophits, mask_lower)
    alone.close(); plus.close()
    for i, q in enumerate(queries):
        s, c = od.topscores(q, o)
        for name, (seqno, count, nc) in (("alone", a), ("with a long query", b)):
            where = (name, k, tophits, mask_lower, i, len(q))
            assert nc[i] == len(s), where + (int(nc[i]), len(s))
            assert seqno[i, :nc[i]].tolist() == s.tolist() and count[i, :nc[i]].tolist() == c.tolist(), where


def soft_mask(rng, s, n=40):
    b = bytearray(s)
    a = int(rng.integers(0, max(1, len(b) - n)))
    b[a:a + n] = bytes(b[a:a + n]).lower()
    return bytes(b)


def with_iupac(rng, s, n=6):
    a = np.frombuffer(s, dtype=np.uint8).copy()
    a[rng.integers(0, a.shape[0], size=n)] = IUPAC[rng.integers(0, IUPAC.shape[0], size=n)]
    return a.tobytes()


def family_case(k):
    """one shard: 40 families of 2-10 % variants of 500-nt roots, unrelated targets, soft-masked and IUPAC targets;
    queries of family members from 150 nt up to the longest the short instance takes, soft-masked and IUPAC ones,
    one of fewer windows than minwordmatches, k - 1 and k nt"""
    rng = np.random.default_rng(900 + k)
    roots = synth.random_seqs(rng, 40, 500)
    seqs = [synth.mutate(rng, roots[i % 40], float(rng.uniform(0.02, 0.1))).tobytes() for i in range(2000)]
    seqs += [r.tobytes() for r in synth.random_seqs(rng, 500, 350)]
    for i in range(0, len(seqs), 13):
        seqs[i] = soft_mask(rng, seqs[i])
    for i in range(5, len(seqs), 17):
        seqs[i] = with_iupac(rng, seqs[i])
    top = longest_short(k)
    queries = [synth.mutate(rng, roots[i][:int(rng.integers(150, top))], 0.03).tobytes()[:top] for i in range(10)]
    queries += [roots[10][:top].tobytes(), roots[11][:top - 1].tobytes()]
    queries += [soft_mask(rng, roots[12][:top].tobytes(), 120), with_iupac(rng, roots[13][:top].tobytes(), 10)]
    few = checkers.MINWORDMATCHES[k] + k - 2          # one window fewer than minwordmatches
    queries += [roots[14][:few].tobytes(), roots[15][:k - 1].tobytes(), roots[15][:k].tobytes()]
    assert all(fits_short(len(q), k) for q in queries)
    return synth.SeqSet(seqs), queries, roots


@pytest.mark.parametrize("k", [3, 8, 10, 12])
def test_short_instance_equals_full_and_oracle(ctx, k):
    dbs, queries, roots = family_case(k)
    db = ctx.seqset(dbs)
    top = longest_short(k)
    for mask_lower in (0, 1):
        ix = ctx.index(db, k, mask_lower)
        od = checkers.OracleDb(dbs, k=k, mask_lower=mask_lower)
        for tophits in (1, 41, SHORT_TOPHITS):
            check_short_and_full(ctx, ix, od, k, queries, tophits, mask_lower)
        # the other side of the rule: one window more, or tophits 65, runs the full instance alone too
        check_short_and_full(ctx, ix, od, k, queries + [roots[16][:top + 1].tobytes()], SHORT_TOPHITS, mask_lower)
        check_short_and_full(ctx, ix, od, k, queries, SHORT_TOPHITS + 1, mask_lower)
        od.close(); ix.close()
    db.close()


def test_ties_beyond_the_candidate_buffer(ctx):
    """3 000 copies of one sequence, cut to 40 different lengths: every copy ties on the count, far more than the short
    instance's 256 candidate keys, so its sort-and-cut scan orders them by length and number"""
    k = 8
    rng = np.random.default_rng(77)
    root = synth.random_seqs(rng, 1, 600)[0]
    seqs = [root[:560 + (i * 7) % 40].tobytes() for i in range(3000)]
    seqs += [r.tobytes() for r in synth.random_seqs(rng, 1000, 600)]
    dbs = synth.SeqSet(seqs)
    queries = [root[a:a + 250].tobytes() for a in (0, 100, 300)] + [synth.mutate(rng, root[:262], 0.05).tobytes()[:262]]
    db = ctx.seqset(dbs)
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(dbs, k=k)
    s, c = od.topscores(queries[0], rank_opts(k, len(seqs)))
    assert int((c == c[0]).sum()) >= 3000 > SHORT_CAND
    for tophits in (1, 8, SHORT_TOPHITS):
        check_short_and_full(ctx, ix, od, k, queries, tophits)
    od.close(); ix.close(); db.close()


def test_running_threshold_over_two_shards(ctx):
    """40 000 targets, two static shards, one family spread over both: the short instance carries its running threshold
    from shard to shard as the full one does"""
    k = 8
    rng = np.random.default_rng(78)
    m = synth.random_seqs(rng, 40_000, 300)
    root = synth.random_seqs(rng, 1, 300)[0]
    fam = np.arange(11, 40_000, 97)
    m[fam] = root
    sub = rng.random((fam.shape[0], 300)) < 0.04
    m[fam] = np.where(sub, synth.ACGT[rng.integers(0, 4, size=(fam.shape[0], 300))], m[fam])
    dbs = synth.SeqSet.from_matrix(m)
    queries = [synth.mutate(rng, root[a:a + 250], 0.03).tobytes() for a in (0, 25, 50)] + [root[:262].tobytes()]
    db = ctx.seqset(dbs)
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(dbs, k=k)
    s, _ = od.topscores(queries[3], rank_opts(k, SHORT_TOPHITS))
    assert {int(t) // 32766 for t in s} == {0, 1}
    for tophits in (1, 41, SHORT_TOPHITS):
        check_short_and_full(ctx, ix, od, k, queries, tophits)
    od.close(); ix.close(); db.close()
