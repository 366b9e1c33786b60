"""The cluster driver's incremental k-mer index (vsg_cluster_index_*) over three shards of 32 768 centroids, against the
oracle, list by list: every word length from 3 to 10, non-contiguous appends (dense number != sequence number), append
schedules that straddle and that end exactly on the shard boundaries, checkpoints on both sides of each boundary, every
ranker path (running threshold, shared memory, HBM, unbounded lists) and tie crowds across shards.  Then clustering of
70 000 centroids past two shard boundaries against the reference CLI's stored records."""
import os

import numpy as np
import pytest

import checkers
from test_cluster_gpu import STOCK, device_records, reference_records
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu

SHARD = 32768                       # targets per incremental shard
NSEQ = 82_000
SKIP = lambda s: s % 7 == 3         # sequences never appended: dense number != sequence number
IUPAC = np.frombuffer(b"NRYSWKMBDHV", dtype=np.uint8)
MOTIF = b"GATTACACCGTTAGCAGGCTTACGATCCGA"   # planted in every 41st sequence: a tie crowd across all shards
SHORT0 = 100                        # sequences SHORT0 + 7 j hold j nt (j = 0 .. 11): empty, k - 1 and k nt at every k
ALL = NSEQ                          # tophits "all": above 1 024, the unbounded lists


def boundary_dense(n):
    return [0, 32765, 32766, 32767, 32768, 32769, 65533, 65534, 65535, 65536, 65537, n - 1]


def checkpoints(n):
    return [1, 32765, 32766, 32767, 32768, 32769, 65535, 65536, 65537, n]


def make_set():
    """82 000 sequences of 60-300 nt: families of 2-10 % variants, unrelated sequences, soft-masked stretches, IUPAC
    symbols, the motif, and 0..11-nt sequences; the targets at the boundary dense numbers are unrelated"""
    rng = np.random.default_rng(4242)
    lens = rng.integers(60, 301, size=NSEQ)
    m = synth.random_seqs(rng, NSEQ, 300)
    roots = synth.random_seqs(rng, 1500, 300)
    seqs = []
    for i in range(NSEQ):
        if i % 5 == 0:
            s = synth.mutate(rng, roots[(i // 5) % 1500], float(rng.uniform(0.02, 0.1)))[:lens[i]]
        else:
            s = m[i, :lens[i]]
        seqs.append(bytearray(s.tobytes()))
    for i in range(7, NSEQ, 41):
        seqs[i][10:10 + len(MOTIF)] = MOTIF
    for i in range(0, NSEQ, 13):
        a = int(rng.integers(0, len(seqs[i]) - 40))
        seqs[i][a:a + 40] = bytes(seqs[i][a:a + 40]).lower()
    for i in range(5, NSEQ, 17):
        a = np.frombuffer(bytes(seqs[i]), dtype=np.uint8).copy()
        a[rng.integers(0, a.shape[0], size=6)] = IUPAC[rng.integers(0, IUPAC.shape[0], size=6)]
        seqs[i] = bytearray(a.tobytes())
    subset = np.array([s for s in range(NSEQ) if not SKIP(s)], dtype=np.uint32)
    for d in boundary_dense(subset.shape[0]):
        seqs[int(subset[d])] = bytearray(synth.random_seqs(rng, 1, int(rng.integers(200, 301)))[0].tobytes())
    for j in range(12):
        assert not SKIP(SHORT0 + 7 * j)
        seqs[SHORT0 + 7 * j] = bytearray(roots[0][:j].tobytes())
    return [bytes(s) for s in seqs], subset


def make_queries(seqs, subset, k):
    """(names, queries): 1-3 % mutants of the boundary targets, short reads (running threshold), ~1 500 nt (shared
    memory without it), 2 047 + k and 2 048 + k nt, ~6 000 nt (HBM), empty, k - 1 nt and low-complexity reads"""
    rng = np.random.default_rng(900 + k)
    n = subset.shape[0]
    names, qs = [], []
    for d in boundary_dense(n):
        t = np.frombuffer(seqs[int(subset[d])], dtype=np.uint8)
        names.append(f"mutant of dense {d}"); qs.append(synth.mutate(rng, t, float(rng.uniform(0.01, 0.03))).tobytes())
    for i in (35, 1000, 40000, 70000):
        t = np.frombuffer(seqs[int(subset[i])], dtype=np.uint8)
        names.append(f"70-nt piece of dense {i}"); qs.append(t[20:90].tobytes())
    long = b"".join(seqs[int(subset[d])] for d in range(500, 30000, 2900))
    names.append("~1 500 nt"); qs.append(long[:1500])
    for w in (2047, 2048):
        names.append(f"{w} + k nt"); qs.append((long * 2)[:w + k])
    names.append("~6 000 nt"); qs.append((long * 4)[:6000])
    names.append("empty"); qs.append(b"")
    names.append("k - 1 nt"); qs.append(seqs[SHORT0 + 7 * (k - 1)])
    names.append("motif"); qs.append(MOTIF)
    names.append("motif + poly-A"); qs.append(MOTIF + b"A" * 40)
    names.append("AC repeat"); qs.append(b"AC" * 60)
    names.append("AACG repeat"); qs.append(b"AACG" * 25)
    return names, qs


@pytest.fixture(scope="module")
def data():
    return make_set()


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def append_calls(schedule, n, prev=0):
    """the vsg_cluster_index_append calls (as dense ranges) that take an index from prev to n centroids"""
    if schedule == "per_checkpoint":
        return [(prev, n)]
    if schedule == "by_1000":                  # one call straddles 32 768 and one 65 536
        cuts = list(range(1000, n, 1000))
    elif schedule == "on_boundaries":          # calls end exactly on 32 768 and 65 536
        cuts = list(range(4096, n, 4096))
    else:                                      # single_at_boundaries: one call per centroid around each boundary
        singles = [b + j for b in (SHARD, 2 * SHARD) for j in range(-4, 5)]
        cuts = sorted(set(list(range(4000, n, 4000)) + [c for c in singles if 0 < c < n]))
    ends = [c for c in cuts if prev < c < n] + [n]
    out, a = [], prev
    for e in ends:
        out.append((a, e)); a = e
    return out


_oracle_cache = {}


def oracle_lists(k, mask_lower, seqs, subset, n, queries):
    """the oracle's full best-first lists (tophits = all) of every query against the first n appended targets, in append
    order (its target numbers are the dense numbers); a list cut to tophits is its prefix"""
    key = (k, mask_lower, n)
    if key not in _oracle_cache:
        if _oracle_cache and next(iter(_oracle_cache))[0] != k:
            _oracle_cache.clear()
        dbs = synth.SeqSet([seqs[int(s)] for s in subset[:n]])
        od = checkers.OracleDb(dbs, k=k, mask_lower=mask_lower)
        o = checkers.search_opts(1, k=k, mask_lower=mask_lower)
        o.tophits = n
        _oracle_cache[key] = ([od.topscores(q, o) for q in queries], dbs.lens.copy())
        od.close()
    return _oracle_cache[key]


def check_rank(cix, qs, queries, names, want, lens, k, schedule, mask_lower, n, tophits):
    cand, count, nc = cix.rank(qs, 0, len(queries), checkers.MINWORDMATCHES[k], tophits)
    for i in range(len(queries)):
        s, c = want[i][0][:tophits], want[i][1][:tophits]
        gs, gc = cand[i, :nc[i]], count[i, :nc[i]]
        if gs.tolist() == s.tolist() and gc.tolist() == c.tolist():
            continue
        r = next((j for j in range(min(len(s), len(gs))) if gs[j] != s[j] or gc[j] != c[j]), min(len(s), len(gs)))

        def at(lst, cnt, j):
            if j >= len(lst):
                return "none"
            d = int(lst[j])
            return f"dense {d} (shard {d // SHARD}, slot {d % SHARD}, count {int(cnt[j])}, length {int(lens[d]) if d < len(lens) else '?'})"
        pytest.fail(f"k={k} schedule={schedule} mask_lower={mask_lower} checkpoint={n} tophits={tophits} query {i} "
                    f"({names[i]}, {len(queries[i])} nt): {int(nc[i])} candidates, oracle {len(s)}; first difference "
                    f"at rank {r}: device {at(gs, gc, r)}, oracle {at(s, c, r)}")
    return cand, count, nc


SCHEDULES = ["per_checkpoint", "by_1000", "on_boundaries", "single_at_boundaries"]
CASES = [(8, s) for s in SCHEDULES] + [(k, s) for k in (3, 4, 5, 6, 7, 9, 10) for s in SCHEDULES[:2]]


@pytest.mark.parametrize("k,schedule", CASES)
def test_cluster_index_vs_oracle(ctx, data, k, schedule):
    seqs, subset = data
    nfinal = subset.shape[0]
    assert 2 * SHARD < nfinal < 3 * SHARD
    names, queries = make_queries(seqs, subset, k)
    ss = ctx.seqset(synth.SeqSet(seqs))
    qs = ctx.seqset(synth.SeqSet(queries))
    for mask_lower in (0, 1):
        cix, have = None, 0
        for n in checkpoints(nfinal):
            if schedule != "per_checkpoint" or cix is None:
                if cix is not None:
                    cix.close()
                cix, have = ctx.cluster_index(ss, k, mask_lower), 0
            for a, b in append_calls(schedule, n, have):
                cix.append(subset[a:b])
            have = n
            assert cix.count == n
            want, lens = oracle_lists(k, mask_lower, seqs, subset, n, queries)
            for tophits in (1, 17, 1024, 1025, ALL):
                cand, count, nc = check_rank(cix, qs, queries, names, want, lens, k, schedule, mask_lower, n, tophits)
            if n == nfinal:
                # the unbounded lists hold every boundary target: the boundary slots are exercised
                for j, d in enumerate(boundary_dense(nfinal)):
                    assert d in cand[j, :nc[j]].tolist(), (k, mask_lower, names[j])
                    if k >= 8:
                        assert cand[j, 0] == d, (k, mask_lower, names[j], cand[j, :4], count[j, :4])
                # the motif's tie crowd spans all three shards and is longer than the bounded lists
                im = names.index("motif")
                top = count[im, 0]
                crowd = cand[im, :nc[im]][count[im, :nc[im]] == top]
                assert k < 8 or (crowd.shape[0] > 1024 and {int(d) // SHARD for d in crowd} == {0, 1, 2}), crowd.shape
        cix.close()
    qs.close(); ss.close()


def test_cluster_index_append_refuses_bad_seqnos(ctx):
    ss = ctx.seqset(synth.SeqSet([b"ACGTACGTAC" * 5] * 10))
    cix = ctx.cluster_index(ss, 8, 0)
    for bad in ([3, 3], [5, 4], [10], [2, 2 ** 31]):
        with pytest.raises(vlib.VsgError, match=r"\(-3\)"):
            cix.append(np.array(bad, dtype=np.uint64).astype(np.uint32))
    assert cix.count == 0
    cix.append([2, 5])
    for bad in ([5], [4], [1, 7]):
        with pytest.raises(vlib.VsgError, match=r"\(-3\)"):
            cix.append(bad)
    cix.append([6, 9])
    assert cix.count == 4
    cix.close(); ss.close()


# ---- end to end: clustering past two shard boundaries ----

NROOTS = 70_000
EDGES = [32766, 32767, 65534, 65535]


def substitute(rng, s, n):
    """s with n bases replaced by other bases"""
    m = s.copy()
    for p in rng.choice(m.shape[0], size=n, replace=False):
        m[p] = synth.ACGT[(int(np.flatnonzero(synth.ACGT == m[p])[0]) + int(rng.integers(1, 4))) % 4]
    return m


def e2e_reads(rc_members=False):
    """70 000 unrelated 200-nt roots, processed first and in label order, so a root's dense number is its position;
    roots j, j + 32 768 and j + 65 536 of some j are 5-8 % variants of each other; ~3 000 190-nt members at 1 %, among
    them members of every root within 3 of the boundary centroids and of the last root"""
    rng = np.random.default_rng(77)
    roots = synth.random_seqs(rng, NROOTS, 200)
    variants = list(range(0, NROOTS - 2 * SHARD, 97))
    for j in variants:
        for t in (j + SHARD, j + 2 * SHARD):
            roots[t] = substitute(rng, roots[j], int(rng.integers(10, 17)))        # 5-8 %
    owners = sorted(set(int(x) for x in rng.integers(0, NROOTS, size=2900)) |
                    {e + d for e in EDGES for d in range(-3, 4)} | {NROOTS - 1} | set(variants))
    seqs = [r.tobytes() for r in roots]
    labels = [f"r{i:06d}" for i in range(NROOTS)]
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    for i, j in enumerate(owners):
        a = int(rng.integers(0, 11))
        s = substitute(rng, roots[j][a:a + 190], 2).tobytes()                    # 1 %
        if rc_members and i % 3 == 1:
            s = s.translate(comp)[::-1]
        seqs.append(s)
        labels.append(f"s{i:06d}_{j:06d}")
    return seqs, labels, owners


def check_members(records, owners):
    """exactly NROOTS clusters, every member an H record to its own root"""
    assert sum(1 for v in records.values() if v[0] == "S") == NROOTS
    for i, j in enumerate(owners):
        v = records[f"s{i:06d}_{j:06d}"]
        assert v[0] == "H" and v[3] == f"r{j:06d}", (i, j, v)


def device_cluster(seqs, labels, threads, **opts):
    """vsg_cluster_fast on the reads sorted as the reference sorts them, with its --cluster_fast defaults and `opts`:
    (results, the S/H records the reference would write, keyed by label: type, cluster, identity, strand, centroid,
    CIGAR)"""
    n = len(seqs)
    order = sorted(range(n), key=lambda i: (-len(seqs[i]), labels[i]))
    ctx = vlib.Context(0)
    ss = ctx.seqset(synth.SeqSet([seqs[i] for i in order]))
    ss.dust()
    o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxrejects = 8
    for k, v in opts.items():
        setattr(o, k, v)
    res, ncl, _ = vlib.cluster_fast(ctx, ss, o, threads)
    rc = ctx.revcomp(ss)
    cig = {}
    for strand, qs in ((0, ss), (1, rc)):
        hq = [k for k in range(n) if res["centroid"][k] >= 0 and res["strand"][k] == strand]
        if hq:
            al = ctx.align_pairs(qs, ss, np.array(hq, dtype=np.uint32), res["centroid"][hq].astype(np.uint32), cigar=True)
            cig.update(zip(hq, al.cigars))
    got = {}
    for k in range(n):
        lab = labels[order[k]]
        if res["centroid"][k] < 0:
            got[lab] = ("S", int(res["cluster"][k]), "*", "*", "*", "*")
        else:
            internal = checkers.finish_hit(1, 1, int(res["alignment_length"][k]), int(res["matches"][k]), int(res["mismatches"][k]),
                                           int(res["gaps"][k]), checkers.trims_from_cigar(cig[k]), o.iddef)[0]
            got[lab] = ("H", int(res["cluster"][k]), f"{res['id'][k]:.1f}", labels[order[int(res["centroid"][k])]],
                        "-" if res["strand"][k] else "+", "=" if res["matches"][k] == internal else cig[k])
    rc.close(); ss.close(); ctx.close()
    return res, ncl, got


def reference_uc(tmp, name, key, seqs, labels, args):
    """`vsearch --cluster_fast <reads> <args> --uc` (stored under `name` and `key`): (clusters, digest of the S/H records
    as device_cluster keys them)"""
    fa = os.path.join(tmp, "reads.fasta")
    with open(fa, "wb") as f:
        for l, s in zip(labels, seqs):
            f.write(b">" + l.encode() + b"\n" + s + b"\n")
    uc = os.path.join(tmp, "ref.uc")

    def reduce(text):
        rec = {}
        for line in text.decode().splitlines():
            f = line.split("\t")
            if f[0] == "S":
                rec[f[8]] = ("S", int(f[1]), "*", "*", "*", "*")
            elif f[0] == "H":
                rec[f[8]] = ("H", int(f[1]), f[3], f[9], f[4], f[7])
        return sum(1 for v in rec.values() if v[0] == "S"), checkers.digest(sorted(rec.items()))
    return checkers.reference(name, key, lambda: checkers.run_stock(["--cluster_fast", fa] + args + ["--uc", uc, "--quiet"],
                                                                    [uc], reduce), os.path.exists(STOCK))


E2E_CASES = {"exhaustive": (["--maxaccepts", "0", "--maxrejects", "0"], {"maxaccepts": 0, "maxrejects": 0}),
             "strand_both": (["--strand", "both"], {"strand_both": 1})}


def e2e_reference(tmp, case, threads):
    """the reads of a case ("plain" or a key of E2E_CASES) and the reference CLI's stored (clusters, digest) for them"""
    seqs, labels, owners = e2e_reads(rc_members=case == "strand_both")
    if case == "plain":
        want = reference_records(tmp, "cluster_fast_three_shards", (seqs, labels, threads), seqs, labels,
                                 ["--id", "0.97", "--threads", str(threads)])
    else:
        args = E2E_CASES[case][0]
        want = reference_uc(tmp, f"cluster_fast_three_shards_{case}", (seqs, labels, args, threads), seqs, labels,
                            ["--id", "0.97", "--threads", str(threads)] + args)
    return seqs, labels, owners, want


@pytest.mark.parametrize("threads", [64, 100])
def test_cluster_fast_past_two_shards_equals_reference_cli(tmp_path, threads):
    """--threads 64: 32 768 = 512 rounds of 64, so a round's appends exactly fill shard 0; --threads 100: one round's
    appends straddle each boundary"""
    seqs, labels, owners, (nclusters, want) = e2e_reference(str(tmp_path), "plain", threads)
    ncl, got, _ = device_records(seqs, labels, 0.97, threads)
    assert ncl == nclusters == NROOTS
    assert got == want
    _, _, rec = device_cluster(seqs, labels, threads)
    check_members(rec, owners)


@pytest.mark.parametrize("case", sorted(E2E_CASES))
def test_cluster_fast_past_two_shards_other_paths_equal_reference_cli(tmp_path, case):
    """--maxaccepts 0 --maxrejects 0 (the driver's unbounded lists), and --strand both with a third of the members
    reverse-complemented"""
    seqs, labels, owners, (nclusters, want) = e2e_reference(str(tmp_path), case, 64)
    _, ncl, got = device_cluster(seqs, labels, 64, **E2E_CASES[case][1])
    assert ncl == nclusters == NROOTS
    assert checkers.digest(sorted(got.items())) == want
    check_members(got, owners)
    if case == "strand_both":
        assert sum(1 for v in got.values() if v[0] == "H" and v[4] == "-") >= len(owners) // 3 - 5


def test_session_ranges_ending_on_shard_boundaries_equal_cluster_fast():
    """a cluster session fed [0, 32 768), [32 768, 65 536) and the rest: the ranges end exactly at 32 768 and 65 536
    centroids"""
    seqs, labels, _ = e2e_reads()
    order = sorted(range(len(seqs)), key=lambda i: (-len(seqs[i]), labels[i]))
    ctx = vlib.Context(0)
    ss = ctx.seqset(synth.SeqSet([seqs[i] for i in order]))
    ss.dust()
    o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxrejects = 8
    want, ncl, _ = vlib.cluster_fast(ctx, ss, o, 64)
    s = vlib.ClusterSession(ctx, ss, o)
    parts = []
    for a, b in ((0, SHARD), (SHARD, 2 * SHARD), (2 * SHARD, ss.n)):
        parts.append(s.assign(a, b - a, 64))
        assert s.clusters == min(b, NROOTS)
    got = np.concatenate(parts)
    assert s.clusters == ncl == NROOTS
    s.close()
    assert got.tobytes() == want.tobytes()
    ss.close(); ctx.close()
