"""GPU parity tests of the batched aligner (vsg_align_pairs) against the oracle.
Bit-exact on score, alignment statistics and CIGAR (integer/byte work: no tolerance)."""
import os

import numpy as np
import pytest

import checkers
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu

IUPAC = b"ACGTUacgtuNnRYSWKMBDHVryswkmbdhvXx-"


def rand_seq(rng, n, alphabet=b"ACGT"):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, a.shape[0], size=n)].tobytes()


trims_from_cigar = checkers.trims_from_cigar


def check(ctx, qseqs, tseqs, pairs, pen=None, n_mismatch=0, expect_kernel=None):
    qs = ctx.seqset(synth.SeqSet(qseqs))
    ts = ctx.seqset(synth.SeqSet(tseqs))
    qi = np.array([p[0] for p in pairs], dtype=np.uint32)
    ti = np.array([p[1] for p in pairs], dtype=np.uint32)
    res = ctx.align_pairs(qs, ts, qi, ti, cigar=True)
    res2 = ctx.align_pairs(qs, ts, qi, ti, cigar=False)
    bad = []
    for k, (a, b) in enumerate(pairs):
        o = checkers.oracle_nw16(qseqs[a], tseqs[b], pen, n_mismatch)
        g = (int(res.score[k]), int(res.aligned[k]), int(res.matches[k]), int(res.mismatches[k]),
             int(res.gaps[k]), res.cigars[k])
        g2 = (int(res2.score[k]), int(res2.aligned[k]), int(res2.matches[k]), int(res2.mismatches[k]),
              int(res2.gaps[k]))
        want_trims = trims_from_cigar(o[5])
        if o != g or g2 != g[:5] or tuple(res.trims[k]) != want_trims or tuple(res2.trims[k]) != want_trims:
            bad.append((k, a, b, len(qseqs[a]), len(tseqs[b]), o, g, g2, tuple(res.trims[k])))
    assert not bad, f"{len(bad)} of {len(pairs)} pairs differ; first: {bad[:3]}"
    if expect_kernel == "fast":
        assert res.exact_pairs == 0 and res.fast_pairs > 0
    if expect_kernel == "exact":
        assert res.fast_pairs == 0 and res.exact_pairs > 0
    qs.close(); ts.close()
    return res


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


def test_config1_shape_allpairs(ctx):
    reads = synth.config1_allpairs(n_reads=96, n_roots=6, length=200)
    seqs = [reads.seq(i) for i in range(len(reads))]
    pairs = [(i, j) for i in range(len(seqs)) for j in range(i + 1, len(seqs))]
    check(ctx, seqs, seqs, pairs, expect_kernel="fast")


def test_every_rows_per_lane_class(ctx):
    """query lengths chosen so that every R = 1..16 instantiation and the multi-strip path run"""
    rng = np.random.default_rng(11)
    qlens = [1, 2, 31, 32, 33, 64, 65, 96, 97, 128, 150, 160, 161, 200, 224, 225, 250, 256, 257,
             288, 300, 320, 333, 352, 384, 400, 416, 448, 470, 480, 500, 512, 513, 700, 1025, 1500]
    qseqs, tseqs, pairs = [], [], []
    for L in qlens:
        root = np.frombuffer(rand_seq(rng, L), dtype=np.uint8)
        qseqs.append(synth.mutate(rng, root, 0.05).tobytes() if L > 3 else root.tobytes())
        qi = len(qseqs) - 1
        for _ in range(5):
            tseqs.append(synth.mutate(rng, root, float(rng.uniform(0, 0.3))).tobytes() or b"A")
            pairs.append((qi, len(tseqs) - 1))
        for dl in (1, 7, 90, 333, 1500):
            tseqs.append(rand_seq(rng, dl))
            pairs.append((qi, len(tseqs) - 1))
    check(ctx, qseqs, tseqs, pairs, expect_kernel="fast")


def test_search_shape_250_vs_1500(ctx):
    rng = np.random.default_rng(12)
    db = synth.random_seqs(rng, 40, 1500)
    qseqs, pairs = [], []
    for i in range(24):
        src = int(rng.integers(0, 40)); st = int(rng.integers(0, 1250))
        qseqs.append(synth.mutate(rng, db[src, st:st + 250], 0.05).tobytes())
        cands = [src] + [int(x) for x in rng.integers(0, 40, size=7)]
        pairs += [(i, c) for c in cands]
    check(ctx, qseqs, [db[i].tobytes() for i in range(40)], pairs, expect_kernel="fast")


def test_iupac_lowercase_n(ctx):
    rng = np.random.default_rng(13)
    for nm in (0, 1):
        c2 = vlib.Context(0, n_mismatch=nm)
        qseqs = [rand_seq(rng, int(rng.integers(1, 300)), IUPAC) for _ in range(12)]
        tseqs = [rand_seq(rng, int(rng.integers(1, 300)), IUPAC) for _ in range(10)]
        tseqs += [rand_seq(rng, 200), rand_seq(rng, 100)]  # pure ACGT targets against IUPAC queries
        qseqs += [rand_seq(rng, 150)]                        # pure ACGT query against IUPAC targets
        pairs = [(i, j) for i in range(len(qseqs)) for j in range(len(tseqs))]
        check(c2, qseqs, tseqs, pairs, n_mismatch=nm)
        c2.close()


def test_edge_cases_host_resolved(ctx):
    rng = np.random.default_rng(14)
    qseqs = [b"", b"A", rand_seq(rng, 50), rand_seq(rng, 5001)]
    tseqs = [b"", b"C", rand_seq(rng, 77), rand_seq(rng, 5000), rand_seq(rng, 4999), b"A" * 40]
    pairs = [(i, j) for i in range(len(qseqs)) for j in range(len(tseqs))]
    check(ctx, qseqs, tseqs, pairs)


def test_non_default_penalties_fast_and_exact(ctx):
    rng = np.random.default_rng(15)
    for _ in range(6):
        pen = np.array([int(rng.integers(1, 6)), -int(rng.integers(1, 8))]
                       + [int(rng.integers(0, 25)) for _ in range(6)]
                       + [int(rng.integers(0, 5)) for _ in range(6)], dtype=np.int64)
        c2 = vlib.Context(0, pen=pen)
        L = int(rng.integers(20, 400))
        root = np.frombuffer(rand_seq(rng, L), dtype=np.uint8)
        qseqs = [synth.mutate(rng, root, 0.1).tobytes() for _ in range(3)]
        tseqs = [synth.mutate(rng, root, 0.2).tobytes() for _ in range(9)] + [rand_seq(rng, 300)]
        pairs = [(i, j) for i in range(3) for j in range(10)]
        check(c2, qseqs, tseqs, pairs, pen=pen)
        c2.close()


def test_exact_kernel_overflow_semantics():
    """huge penalties: saturation and the h_min/h_max overflow flag decide the outcome"""
    rng = np.random.default_rng(16)
    pen = np.array([2, -4, 3000, 3000, 5000, 5000, 3000, 3000, 600, 600, 900, 900, 600, 600], dtype=np.int64)
    c2 = vlib.Context(0, pen=pen)
    qseqs = [rand_seq(rng, L) for L in (10, 20, 30, 40, 60)]
    tseqs = [rand_seq(rng, int(rng.integers(1, 90))) for _ in range(16)]
    pairs = [(i, j) for i in range(5) for j in range(16)]
    res = check(c2, qseqs, tseqs, pairs, pen=pen, expect_kernel="exact")
    assert (res.score == 32767).any() and (res.score != 32767).any()
    c2.close()
    pen2 = np.array([3000, -3000, 1, 1, 18, 18, 1, 1, 1, 1, 2, 2, 1, 1], dtype=np.int64)
    c3 = vlib.Context(0, pen=pen2)
    q = rand_seq(rng, 40)
    check(c3, [q], [q, q[:20], rand_seq(rng, 40), q + q], [(0, j) for j in range(4)], pen=pen2)
    c3.close()
    pen3 = pen2.copy(); pen3[4] = 2 ** 31 - 1   # does not fit a cell: everything deferred
    c4 = vlib.Context(0, pen=pen3)
    check(c4, [q], [q, b"A"], [(0, 0), (0, 1)], pen=pen3)
    c4.close()


def test_exact_kernel_equals_fast_kernel():
    """the same default-penalty workload forced through the exact kernel"""
    os.environ["VSG_DISABLE_FAST"] = "1"
    try:
        c2 = vlib.Context(0)
    finally:
        del os.environ["VSG_DISABLE_FAST"]
    rng = np.random.default_rng(17)
    root = np.frombuffer(rand_seq(rng, 300), dtype=np.uint8)
    qseqs = [synth.mutate(rng, root, 0.1).tobytes() for _ in range(4)] + [rand_seq(rng, 300, IUPAC)]
    tseqs = [synth.mutate(rng, root, 0.2).tobytes() for _ in range(12)] + [rand_seq(rng, 6000)]
    pairs = [(i, j) for i in range(5) for j in range(13)]
    check(c2, qseqs, tseqs, pairs, expect_kernel="exact")
    c2.close()


def test_small_direction_budget_chunks():
    """many chunks: VSG_DIR_BUDGET_MB forces the chunk loop"""
    os.environ["VSG_DIR_BUDGET_MB"] = "1"
    try:
        c2 = vlib.Context(0)
    finally:
        del os.environ["VSG_DIR_BUDGET_MB"]
    reads = synth.config1_allpairs(n_reads=40, n_roots=3, length=200, seed=99)
    seqs = [reads.seq(i) for i in range(len(reads))]
    pairs = [(i, j) for i in range(len(seqs)) for j in range(i + 1, len(seqs))]
    check(c2, seqs, seqs, pairs)
    c2.close()


def test_long_pairs_stay_on_the_fast_kernel(ctx):
    """q+d up to ~16 000 under default penalties: values reach beyond +-16 000 but not the 16-bit limits"""
    rng = np.random.default_rng(18)
    root = np.frombuffer(rand_seq(rng, 4100), dtype=np.uint8)
    qseqs = [synth.mutate(rng, root, 0.03).tobytes()[:4000], rand_seq(rng, 2500)]
    tseqs = [synth.mutate(rng, root, 0.05).tobytes() + rand_seq(rng, 1900), rand_seq(rng, 6000),
             root.tobytes(), rand_seq(rng, 9000)]
    pairs = [(0, 0), (0, 1), (0, 2), (1, 3), (1, 0)]
    res = check(ctx, qseqs, tseqs, pairs, expect_kernel="fast")
    assert int(res.score.min()) < -4000 and int(res.score.max()) > 6000
