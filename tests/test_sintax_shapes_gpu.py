"""vsg_sintax against the SINTAX oracle (oracle/sintax.c, pinned to the reference in test_sintax_oracle_cpu.py),
whole result rows and on a mismatch bootstrap by bootstrap: every word length from 3 to 15 on one index shard and on
three, with ties planted across the shards; the query edges of the k-mer and draw kernels (31-33 and power-of-two
distinct counts, both sides of KMER_CAP, the longest query the ranker takes, empty, ambiguous and lower-case queries);
a call cut into many chunks by a small scratch budget; extreme seeds and query numbers, and slices of a call."""
import contextlib
import os

import numpy as np
import pytest

import checkers
import sintax_cases as sc
from vsearch_b200 import lib, synth

pytestmark = pytest.mark.gpu

KS = list(range(3, 16))
KMER_CAP = 2048          # distinct k-mers a query keeps in shared memory; longer queries build their table in HBM
BOOTS = 100
MAX_WINDOWS = 65_535     # the ranker's longest query: 65 534 + k nt


@pytest.fixture(scope="module")
def ctx():
    c = lib.Context(0)
    yield c
    c.close()


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def device_rows(ctx, ix, qs, q0, nq, seed, both, qnum0):
    return sc.as_array(ctx.sintax(ix, qs, q0, nq, seed, strand_both=both, query_number0=qnum0))


def oracle_rows(od, queries, qnum0, seed, both):
    return np.stack([od.sintax(q, qnum0 + i, seed, both) for i, q in enumerate(queries)])


def first_difference(got, want, od, queries, qnum0, seed, both):
    """the first query, strand and bootstrap where the device and the oracle differ, with both winners, their counts
    on that bootstrap's sample and their lengths"""
    i = int(np.nonzero((got != want).any(axis=1))[0][0])
    _, tr = od.sintax(queries[i], qnum0 + i, seed, both, trace=True)
    lens = od.ss.lens
    msg = [f"query {i} (query number {qnum0 + i}, {len(queries[i])} nt) of {len(queries)}: "
           f"device strand {got[i, 0]} nboot {got[i, 1:3].tolist()} best {got[i, 3:5].tolist()}, "
           f"oracle strand {want[i, 0]} nboot {want[i, 1:3].tolist()} best {want[i, 3:5].tolist()}"]
    for s in range(2):
        g, w = got[i, 5 + BOOTS * s:5 + BOOTS * (s + 1)], want[i, 5 + BOOTS * s:5 + BOOTS * (s + 1)]
        diff = np.nonzero(g != w)[0]
        if diff.shape[0] == 0:
            continue
        j = int(diff[0])
        won = [b for b in range(BOOTS) if tr[BOOTS * s + b].winner >= 0]
        b = won[j] if j < len(won) else None
        if b is None:
            msg.append(f"strand {s}: winner #{j}: device {g[j]}, the oracle has only {len(won)} successful bootstraps")
            break
        r = tr[BOOTS * s + b]
        samp = set(r.samp[:r.nsamp])

        def count(t):
            if t < 0:
                return None
            return len(samp & set(checkers.oracle_unique_kmers(od.ss.seq(int(t)), od.k, od.mask_lower).tolist()))

        msg.append(f"strand {s}, winner #{j} = bootstrap {b} ({r.nsamp} sampled k-mers, {r.ntied} targets tie at the "
                   f"top count {r.count}, numbers {r.tied_lo}..{r.tied_hi}): device target {g[j]} count {count(g[j])} "
                   f"length {lens[g[j]] if g[j] >= 0 else None}; oracle target {w[j]} count {r.count} length {lens[w[j]]}")
        break
    return "; ".join(msg)


def check(got, want, od, queries, qnum0, seed, both, what):
    if not np.array_equal(got, want):
        nbad = int((got != want).any(axis=1).sum())
        raise AssertionError(f"{what}: {nbad} of {len(queries)} rows differ from the oracle; first: "
                             + first_difference(got, want, od, queries, qnum0, seed, both))


# ---- a. every word length on one shard ------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS)
def test_every_wordlength_one_shard(ctx, k):
    d = sc.data()
    _, seqs = sc.database()
    ss = synth.SeqSet(seqs)
    q = d["q_seqs"]
    db = ctx.seqset(ss); qs = ctx.seqset(synth.SeqSet(q))
    long_q, short_q = d["meta"]["long_queries"], d["meta"]["short_queries"]
    assert all(len(q[i]) - k + 1 > KMER_CAP for i in long_q)
    for mask_lower in (0, 1):
        ix = ctx.index(db, k, mask_lower)
        od = checkers.OracleDb(ss, k=k, mask_lower=mask_lower)
        for seed, both in ((42, 0), (2 ** 33 + 5, 1)):
            got = device_rows(ctx, ix, qs, 0, len(q), seed, both, 0)
            check(got, oracle_rows(od, q, 0, seed, both), od, q, 0, seed, both, f"k={k} mask_lower={mask_lower} both={both}")
            # the HBM first-occurrence table ran: the long queries (the second one reverse-complemented) took bootstraps
            assert got[long_q[0], 1] > 0 and (not both or got[long_q[1], 2] > 0)
            assert (got[short_q, 1:3] == 0).all()                 # fewer than 32 distinct k-mers: no bootstraps
        od.close(); ix.close()
    db.close(); qs.close()


# ---- b. three shards with planted cross-shard ties -----------------------------------------------------------------
@pytest.fixture(scope="module")
def three_shards(ctx):
    d = sc.three_shard_data()
    ss = synth.SeqSet(d["db_seqs"])
    db = ctx.seqset(ss); qs = ctx.seqset(synth.SeqSet(d["q_seqs"]))
    yield d, ss, db, qs
    db.close(); qs.close()


@pytest.mark.parametrize("k", KS)
def test_three_shards_cross_shard_ties(ctx, three_shards, k):
    d, ss, db, qs = three_shards
    q = d["q_seqs"]
    n = len(ss)
    assert n > 2 * sc.SHARD and (n - 2 * sc.SHARD) % 2 == 1      # the last shard is partial and has an odd count
    ix = ctx.index(db, k, 0)
    od = checkers.OracleDb(ss, k=k)
    seed = 9
    got = device_rows(ctx, ix, qs, 0, len(q), seed, 1, 0)
    want, ties_across = [], 0
    for i, s in enumerate(q):
        row, tr = od.sintax(s, i, seed, 1, trace=True)
        want.append(row)
        ties_across += sum(1 for r in tr if r.winner >= 0 and r.tied_lo // sc.SHARD != r.tied_hi // sc.SHARD)
    want = np.stack(want)
    check(got, want, od, q, 0, seed, 1, f"three shards k={k}")
    # the combine decides: top counts shared across shards, winners from every shard, the planted losers never win
    winners = want[:, 5:]
    assert ties_across > 0
    assert {int(t) // sc.SHARD for t in winners[winners >= 0]} == {0, 1, 2}
    assert not np.isin(winners, d["meta"]["never"]).any()
    if k >= 4:   # at k = 3 nearly every target holds every sampled 3-mer, and the shortest background targets win
        assert np.isin(d["meta"]["wins"], winners).all()
    od.close(); ix.close()


# ---- c. query edges ---------------------------------------------------------------------------------------------------
def distinct(s, k):
    return checkers.oracle_unique_kmers(s, k).shape[0]


def with_distinct(src, k, want):
    """the shortest prefix of src with exactly `want` distinct k-mers"""
    lo, hi = k, len(src)
    assert distinct(src, k) >= want
    while lo < hi:
        mid = (lo + hi) // 2
        if distinct(src[:mid], k) >= want:
            hi = mid
        else:
            lo = mid + 1
    assert distinct(src[:lo], k) == want
    return src[:lo]


def edge_case(k):
    """(database, queries, names): queries at the edges of the k-mer and draw kernels; the database holds every query
    in 300-nt pieces, each once as it is in upper case and once mutated or in lower case, among random targets, so
    bootstraps find winners"""
    rng = np.random.default_rng(1200 + k)

    def rnd(n):
        return synth.random_seqs(rng, 1, n)[0].tobytes()

    def sprinkled(valid):
        # two random stretches with an IUPAC symbol between them: k + `valid` windows, `valid` of them unambiguous
        a, b = rnd(k - 1 + 20), rnd(k - 1 + valid - 20)
        return a + b"R" + b
    qs = {}
    for dcount in (31, 32, 33, 64, 2047, 2048, 2049):
        qs[f"distinct{dcount}"] = with_distinct(rnd(3 * dcount + 4 * k), k, dcount)
    flank = rnd(2048 + k)
    qs["win2047"] = flank[:2047 + k]
    qs["win2048"] = flank[:2048 + k]
    qs["longest"] = rnd(MAX_WINDOWS - 1 + k)
    qs["empty"] = b""
    qs["k_minus_1"] = flank[:k - 1]
    qs["all_n"] = b"N" * 300
    qs["iupac31"] = sprinkled(31)
    qs["iupac32"] = sprinkled(32)
    iupac = np.frombuffer(rnd(400), dtype=np.uint8).copy()
    iupac[rng.integers(0, 400, size=12)] = np.frombuffer(b"NRYKMSWBDHVN", dtype=np.uint8)
    qs["iupac_mixed"] = iupac.tobytes()
    qs["lower"] = rnd(300).lower()
    seqs = [rnd(int(rng.integers(150, 400))) for _ in range(400)]
    for s in qs.values():
        for t, p in enumerate(range(0, len(s), 300)):
            piece = s[p:p + 300].upper()
            other = piece.lower() if t % 2 else synth.mutate(rng, np.frombuffer(piece, dtype=np.uint8), 0.03).tobytes()
            for x in (piece, other):
                seqs.insert(int(rng.integers(0, len(seqs) + 1)), x)
    return synth.SeqSet(seqs), list(qs.values()), list(qs)


@pytest.mark.parametrize("k", [8, 12])
def test_query_edges(ctx, k):
    dbs, q, names = edge_case(k)
    at = {nm: i for i, nm in enumerate(names)}
    for dcount in (31, 32, 33, 64, 2047, 2048, 2049):
        assert distinct(q[at[f"distinct{dcount}"]], k) == dcount
    assert [len(q[at[nm]]) - k + 1 for nm in ("win2047", "win2048", "longest")] == [KMER_CAP, KMER_CAP + 1, MAX_WINDOWS]
    assert distinct(q[at["longest"]], k) > (60_000 if k == 12 else 40_000)
    for nm, want in (("iupac31", 31), ("iupac32", 32)):
        s = q[at[nm]]
        assert len(s) - k + 1 > 32 and distinct(s, k) == want
    db = ctx.seqset(dbs); qs = ctx.seqset(synth.SeqSet(q))
    for mask_lower in (0, 1):
        ix = ctx.index(db, k, mask_lower)
        od = checkers.OracleDb(dbs, k=k, mask_lower=mask_lower)
        for seed, both in ((5, 0), (2 ** 63 + 11, 1)):
            got = device_rows(ctx, ix, qs, 0, len(q), seed, both, 77)
            check(got, oracle_rows(od, q, 77, seed, both), od, q, 77, seed, both, f"edges k={k} mask_lower={mask_lower} both={both}")
            nb = {nm: int(got[at[nm], 1]) for nm in names}
            for nm in ("distinct31", "empty", "k_minus_1", "all_n", "iupac31"):
                assert nb[nm] == 0 and got[at[nm], 2] == 0, nm
            # bootstraps succeed on the plus strand of the rest (lower-case query symbols count: queries are not masked)
            for nm in names:
                if nm not in ("distinct31", "empty", "k_minus_1", "all_n", "iupac31"):
                    assert nb[nm] > 0, (nm, mask_lower, both)
        od.close(); ix.close()
    qs.close()
    # one window more than the ranker takes is refused
    over = ctx.seqset(synth.SeqSet([q[at["win2047"]], q[at["longest"]] + b"A"]))
    ix = ctx.index(db, k, 0)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*longer than the device ranker supports"):
        ctx.sintax(ix, over, 0, 2, 1, strand_both=1)
    assert ctx.sintax(ix, over, 0, 1, 1)["nboot"].shape == (1, 2)   # the query before it alone is fine
    ix.close(); over.close(); db.close()


# ---- d. the chunk loop ------------------------------------------------------------------------------------------------
def chunk_queries():
    """the fixture's queries with long ones among them: two ~65 000-nt queries side by side (each over a chunk's budget
    alone), and 40 000, 12 000 and 3 000 nt ones, so the HBM first-occurrence scratch changes size between chunks"""
    rng = np.random.default_rng(1300)
    _, seqs = sc.database()
    q = list(sc.data()["q_seqs"])

    def long_query(n):
        parts, total = [], 0
        while total < n:
            s = seqs[int(rng.integers(0, len(seqs)))].upper() if rng.random() < 0.7 else synth.random_seqs(rng, 1, 1000)[0].tobytes()
            parts.append(s); total += len(s)
        return b"".join(parts)[:n]
    for pos, n in ((10, 65_000), (11, 64_000), (100, 40_000), (180, 3_000), (250, 12_000), (len(q) + 5, 65_000)):
        q.insert(pos, long_query(n))
    return q


def test_chunk_loop_equals_one_call(ctx):
    _, seqs = sc.database()
    ss = synth.SeqSet(seqs)
    q = chunk_queries()
    k, seed = 8, 2 ** 64 - 1
    with env(VSG_DIR_BUDGET_MB="1"):
        small = lib.Context(0)
    try:
        want = {}
        for c in (ctx, small):
            db = c.seqset(ss); qs = c.seqset(synth.SeqSet(q)); ix = c.index(db, k, 1)
            before = lib.launch_count()
            want[c is small] = device_rows(c, ix, qs, 0, len(q), seed, 1, 3)
            launches = lib.launch_count() - before
            if c is small:
                # per chunk: revcomp + the four SINTAX kernels
                assert launches % 5 == 0 and launches >= 5 * 10, launches
            else:
                assert launches == 5, launches
            ix.close(); qs.close(); db.close()
    finally:
        small.close()
    assert want[True].tobytes() == want[False].tobytes()
    od = checkers.OracleDb(ss, k=k, mask_lower=1)
    check(want[True], oracle_rows(od, q, 3, seed, 1), od, q, 3, seed, 1, "small budget")
    assert (want[True][[10, 11, 100], 1:3].max(axis=1) > 0).all()
    od.close()


# ---- e. seeds and substreams ------------------------------------------------------------------------------------------
def test_seeds_and_query_numbers(ctx):
    _, seqs = sc.database()
    ss = synth.SeqSet(seqs)
    q = sc.data()["q_seqs"]
    db = ctx.seqset(ss); qs = ctx.seqset(synth.SeqSet(q)); ix = ctx.index(db, 8, 1)
    od = checkers.OracleDb(ss, k=8, mask_lower=1)
    rows = set()
    for seed in (0, 1, 2 ** 63, 2 ** 64 - 1):
        for qn0 in (2 ** 32 - 3, 2 ** 40 + 7):
            whole = device_rows(ctx, ix, qs, 0, len(q), seed, 1, qn0)
            check(whole, oracle_rows(od, q, qn0, seed, 1), od, q, qn0, seed, 1, f"seed={seed} query_number0={qn0}")
            for q0, nq in ((0, 1), (1, 50), (57, 100), (len(q) - 7, 7)):
                part = device_rows(ctx, ix, qs, q0, nq, seed, 1, qn0 + q0)
                assert part.tobytes() == whole[q0:q0 + nq].tobytes(), (seed, qn0, q0, nq)
            rows.add(whole.tobytes())
    assert len(rows) == 8          # every seed and every numbering draws differently
    od.close(); ix.close(); qs.close(); db.close()
