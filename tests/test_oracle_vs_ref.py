"""Pins the oracle (oracle/*.c) against the UNMODIFIED reference compiled into
oracle/_ref/libvsref.so, through the reference's stored results (checkers.reference).  CPU only."""
import ctypes as C
import re

import numpy as np
import pytest

import checkers as _libs
from vsearch_b200 import synth

IUPAC = b"ACGTUacgtuNnRYSWKMBDHVryswkmbdhvXx-*."


def rand_seq(rng, n, alphabet=b"ACGT"):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, a.shape[0], size=n)].tobytes()


class Pairs:
    """collects (query, targets, penalties, n_mismatch) cases; check() compares the oracle's alignments of all of them
    with the reference's search16"""

    def __init__(self, name):
        self.name, self.cases = name, []

    def __call__(self, q, targets, pen=None, n_mismatch=0):
        self.cases.append((q, targets, pen, n_mismatch))

    def check(self):
        want = _libs.reference(self.name, self.cases, lambda: _libs.digest([_libs.ref_search16(*c) for c in self.cases]),
                               _libs.ref() is not None)
        got = [[_libs.oracle_nw16(q, t, pen, nm) for t in targets] for q, targets, pen, nm in self.cases]
        assert _libs.digest(got) == want


def test_nw16_random_acgt_related():
    check_pairs = Pairs("nw16_random_acgt_related")
    rng = np.random.default_rng(1)
    for _ in range(60):
        L = int(rng.integers(1, 260))
        root = np.frombuffer(rand_seq(rng, L), dtype=np.uint8)
        q = synth.mutate(rng, root, 0.1).tobytes()
        targets = [synth.mutate(rng, root, float(rng.uniform(0, 0.4))).tobytes() for _ in range(11)]
        targets += [rand_seq(rng, int(rng.integers(1, 300))) for _ in range(5)]
        check_pairs(q, targets)
    check_pairs.check()


def test_nw16_iupac_case_n_and_odd_bytes():
    check_pairs = Pairs("nw16_iupac_case_n_and_odd_bytes")
    rng = np.random.default_rng(2)
    for nm in (0, 1):
        for _ in range(40):
            q = rand_seq(rng, int(rng.integers(1, 120)), IUPAC)
            targets = [rand_seq(rng, int(rng.integers(1, 120)), IUPAC) for _ in range(9)]
            check_pairs(q, targets, n_mismatch=nm)
    check_pairs.check()


def test_nw16_all_byte_values_map():
    # every byte 1..255 appears in a sequence; the aligner sees them through map_4bit
    check_pairs = Pairs("nw16_all_byte_values_map")
    q = bytes(range(1, 256))
    t = bytes(reversed(range(1, 256)))
    check_pairs(q, [t, q, b"ACGT"])
    check_pairs.check()


def test_nw16_edge_lengths_and_empty():
    check_pairs = Pairs("nw16_edge_lengths_and_empty")
    rng = np.random.default_rng(3)
    q = rand_seq(rng, 37)
    targets = [b"", b"A", b"AC", b"ACG", b"ACGT", b"ACGTA", rand_seq(rng, 1), rand_seq(rng, 500), b""]
    check_pairs(q, targets)
    check_pairs(b"", [b"", b"A", rand_seq(rng, 77)])
    check_pairs(b"G", [b"G", b"A", b"", rand_seq(rng, 9)])
    # homopolymers / repeats (tie-breaking stress)
    check_pairs(b"A" * 50, [b"A" * 40, b"A" * 60, b"AT" * 25, b"T" * 50])
    check_pairs(b"ACAC" * 20, [b"CACA" * 20, b"AC" * 33, b"ACC" * 20])
    check_pairs.check()


def test_nw16_non_default_penalties():
    check_pairs = Pairs("nw16_non_default_penalties")
    rng = np.random.default_rng(4)
    for _ in range(30):
        pen = np.array([int(rng.integers(1, 6)), -int(rng.integers(1, 8))]
                       + [int(rng.integers(0, 25)) for _ in range(6)]
                       + [int(rng.integers(0, 5)) for _ in range(6)], dtype=np.int64)
        L = int(rng.integers(5, 150))
        root = np.frombuffer(rand_seq(rng, L), dtype=np.uint8)
        q = synth.mutate(rng, root, 0.15).tobytes()
        targets = [synth.mutate(rng, root, 0.25).tobytes() for _ in range(8)]
        targets.append(rand_seq(rng, int(rng.integers(1, 200))))
        check_pairs(q, targets, pen)
    check_pairs.check()


def test_nw16_overflow_and_limits():
    check_pairs = Pairs("nw16_overflow_and_limits")
    rng = np.random.default_rng(5)
    # big penalties so that 16-bit saturation / the h_min flag fire on short sequences
    pen = np.array([2, -4, 3000, 3000, 5000, 5000, 3000, 3000, 600, 600, 900, 900, 600, 600], dtype=np.int64)
    for L in (10, 30, 60, 120):
        q = rand_seq(rng, L)
        targets = [rand_seq(rng, int(rng.integers(1, 2 * L))) for _ in range(8)]
        check_pairs(q, targets, pen)
    # match score so large that h_max saturates
    pen2 = np.array([3000, -3000, 1, 1, 18, 18, 1, 1, 1, 1, 2, 2, 1, 1], dtype=np.int64)
    q = rand_seq(rng, 40)
    check_pairs(q, [q, q[:20], rand_seq(rng, 40), q + q], pen2)
    # values that do not fit a cell -> every pair deferred (force_scalar_fallback)
    pen3 = pen2.copy(); pen3[4] = 2 ** 31 - 1
    check_pairs(q, [q, b"A"], pen3)
    # long pair under default penalties: top row runs far negative but stays in range
    q = rand_seq(rng, 300)
    check_pairs(q, [rand_seq(rng, 6000), rand_seq(rng, 11)])
    # product limit (q*d > 25e6) and sum limit -> sentinel
    q = rand_seq(rng, 5001)
    check_pairs(q, [rand_seq(rng, 5000), rand_seq(rng, 4999)])
    # saturating boundary row: d long enough that -(go+(j+1)ge) passes -32768 with ge=6 (limit 6553)
    pen4 = np.array([2, -4, 1, 1, 18, 18, 1, 1, 6, 6, 2, 2, 6, 6], dtype=np.int64)
    q = rand_seq(rng, 50)
    check_pairs(q, [rand_seq(rng, 6000), rand_seq(rng, 5400), rand_seq(rng, 5461), rand_seq(rng, 5463)], pen4)
    check_pairs.check()


def test_unique_kmers():
    rng = np.random.default_rng(6)
    cases = [(rand_seq(rng, int(rng.integers(0, 400)), b"ACGTACGTACGTacgtNnRU"), k, ml)
             for k in (3, 8, 9, 10, 12) for ml in (0, 1) for _ in range(20)]
    want = _libs.reference("unique_kmers", cases, lambda: _libs.digest([_libs.ref_unique_kmers(*c) for c in cases]),
                           _libs.ref() is not None)
    assert _libs.digest([_libs.oracle_unique_kmers(*c) for c in cases]) == want


def _family_db(rng, n_roots=12, per=8, L=300):
    roots = synth.random_seqs(rng, n_roots, L)
    seqs = []
    for r in range(n_roots):
        for _ in range(per):
            seqs.append(synth.mutate(rng, roots[r], float(rng.uniform(0.0, 0.2))).tobytes())
    # some junk: short, ambiguous, duplicates
    seqs += [b"ACGT", b"N" * 50, seqs[0], seqs[1][:100], b"ACGTNNNNACGT" * 10]
    return synth.SeqSet(seqs), roots


def _reference_search(db, qs, kw):
    """the reference's tophits, and digests of its candidate lists (search_topscores) and rows for every query"""
    def run_reference():
        r = _libs.RefDb(db, **kw)
        tops = [r.topscores(q) for q in qs]
        rows = r.search(synth.SeqSet(qs), max_results=r.tophits)
        th = r.tophits
        r.close()
        return th, _libs.digest(tops), _libs.digest(rows)
    return _libs.reference("topscores_and_search", (db, qs, kw), run_reference, _libs.ref() is not None)


def _check_oracle(o, opts, qs, tops, rows):
    assert _libs.digest([o.topscores(q, opts) for q in qs]) == tops
    got = [[(h.target, h.id, h.matches, h.mismatches, h.nwgaps, h.nwalignmentlength, h.accepted, h.strand)
            for h in o.search(q, opts)[0]] for q in qs]
    assert _libs.digest(got) == rows


def test_topscores_and_search_match_reference():
    rng = np.random.default_rng(7)
    db, roots = _family_db(rng)
    for (idv, ma, mr) in ((0.9, 1, 32), (0.5, 3, 16), (0.97, 2, 4), (0.8, 100, 100)):
        o = _libs.OracleDb(db)
        opts = _libs.search_opts(len(db), id=idv, maxaccepts=ma, maxrejects=mr)
        qs = [synth.mutate(rng, roots[i % roots.shape[0]], 0.08).tobytes()[: int(rng.integers(60, 300))]
              for i in range(40)]
        qs += [b"ACGTACGTAC", synth.random_seqs(rng, 1, 200)[0].tobytes()]
        th, tops, rows = _reference_search(db, qs, dict(id=idv, maxaccepts=ma, maxrejects=mr))
        assert opts.tophits == th
        _check_oracle(o, opts, qs, tops, rows)
        o.close()


@pytest.mark.parametrize("k", [10, 11, 13, 14])
def test_large_wordlengths_match_reference(k):
    """k >= 10 is the reference's hash variant of unique_count (unique.cpp:243-334); from 13 on the oracle keeps its
    index as sorted (k-mer, target) pairs instead of 4^k list heads: candidate lists and whole searches still equal
    the reference's, soft-masked and IUPAC symbols included"""
    rng = np.random.default_rng(100 + k)
    db, roots = _family_db(rng)
    o = _libs.OracleDb(db, k=k)
    opts = _libs.search_opts(len(db), id=0.9, maxaccepts=2, maxrejects=16, k=k)
    qs = [synth.mutate(rng, roots[i % roots.shape[0]], 0.05).tobytes()[: int(rng.integers(60, 300))] for i in range(30)]
    qs += [b"ACGTACGTAC", synth.random_seqs(rng, 1, 200)[0].tobytes(), roots[0].tobytes()[:120] + b"NNRY" + roots[0].tobytes()[124:200]]
    th, tops, rows = _reference_search(db, qs, dict(k=k, id=0.9, maxaccepts=2, maxrejects=16))
    assert opts.tophits == th
    want = _libs.reference("unique_kmers_large_k", (qs, k), lambda: _libs.digest(
        [_libs.ref_unique_kmers(q, k, m) for q in qs for m in (0, 1)]), _libs.ref() is not None)
    assert _libs.digest([_libs.oracle_unique_kmers(q, k, m) for q in qs for m in (0, 1)]) == want, k
    _check_oracle(o, opts, qs, tops, rows)
    assert sum(len(o.topscores(q, opts)[0]) > 0 for q in qs) >= 25
    o.close()


@pytest.mark.parametrize("k", [3, 4, 5, 6, 7, 9, 12])
def test_other_wordlengths_match_reference(k):
    """the word lengths the device tests trust the oracle at: with few targets the reference keeps most k-mers of small
    k as bitmaps and counts them with its saturating SIMD path, the oracle with plain lists; candidate lists, whole
    searches and the distinct k-mers of soft-masked and IUPAC queries still equal the reference's"""
    rng = np.random.default_rng(200 + k)
    db, roots = _family_db(rng)
    o = _libs.OracleDb(db, k=k)
    opts = _libs.search_opts(len(db), id=0.9, maxaccepts=2, maxrejects=16, k=k)
    qs = [synth.mutate(rng, roots[i % roots.shape[0]], 0.05).tobytes()[: int(rng.integers(60, 300))] for i in range(30)]
    qs += [b"ACGTACGTAC", synth.random_seqs(rng, 1, 200)[0].tobytes(), roots[0].tobytes()[:120] + b"NNRY" + roots[0].tobytes()[124:200],
           roots[1].tobytes()[:100] + roots[1].tobytes()[100:200].lower(), roots[2].tobytes()[:k]]
    th, tops, rows = _reference_search(db, qs, dict(k=k, id=0.9, maxaccepts=2, maxrejects=16))
    assert opts.tophits == th
    want = _libs.reference("unique_kmers_wordlength", (qs, k), lambda: _libs.digest(
        [_libs.ref_unique_kmers(q, k, m) for q in qs for m in (0, 1)]), _libs.ref() is not None)
    assert _libs.digest([_libs.oracle_unique_kmers(q, k, m) for q in qs for m in (0, 1)]) == want, k
    _check_oracle(o, opts, qs, tops, rows)
    assert sum(len(o.topscores(q, opts)[0]) > 0 for q in qs) >= 25
    o.close()
    # mask_lower = 1: the reference soft-masks its database by DUST (--dbmask dust, which upper-cases a sequence before
    # lower-casing its low-complexity stretches) and leaves lower case out of the index and of the queries' k-mers.  Its
    # search_topscores takes a query as given (the soft-masked one included); its search DUST-masks the query first.  The
    # oracle gets the same sequences
    masked = _libs.reference("dust_masked", ([db.seq(i) for i in range(len(db))], qs), lambda: [
        [[m.start(), m.end()] for m in re.finditer(rb"[a-z]+", _dust(s))] for s in [db.seq(i) for i in range(len(db))] + qs],
        _libs.ref() is not None)
    dusted = [_apply_mask(s, iv) for s, iv in zip([db.seq(i) for i in range(len(db))] + qs, masked)]
    assert sum(bool(iv) for iv in masked[:len(db)]) >= 2   # the low-complexity junk targets
    dbm, qsm = synth.SeqSet(dusted[:len(db)]), dusted[len(db):]
    th, tops, rows = _reference_search(db, qs, dict(k=k, id=0.9, maxaccepts=2, maxrejects=16, dust=1))
    o = _libs.OracleDb(dbm, k=k, mask_lower=1)
    opts = _libs.search_opts(len(db), id=0.9, maxaccepts=2, maxrejects=16, k=k, mask_lower=1)
    assert _libs.digest([o.topscores(q, opts) for q in qs]) == tops
    got = [[(h.target, h.id, h.matches, h.mismatches, h.nwgaps, h.nwalignmentlength, h.accepted, h.strand)
            for h in o.search(q, opts)[0]] for q in qsm]
    assert _libs.digest(got) == rows
    o.close()


def _dust(s: bytes) -> bytes:
    """(reference) DUST soft-masking of one sequence"""
    buf = C.create_string_buffer(s, len(s) + 1)
    _libs.ref().vsref_dust(buf, C.c_int(len(s)))
    return buf.raw[:len(s)]


def _apply_mask(s: bytes, intervals) -> bytes:
    """s upper-cased, with the [start, end) intervals lower-cased"""
    b = bytearray(s.upper())
    for a, e in intervals:
        b[a:e] = bytes(b[a:e]).lower()
    return bytes(b)


@pytest.mark.parametrize("k", [10, 12])
def test_count_cap_matches_reference(k):
    """a 40 000-nt query with more than 32 767 distinct k-mers against copies of itself: the reference's counters
    saturate at 32 767 (searchcore.cpp:306-315) and so do the oracle's; length, then seqno, orders the saturated copies"""
    rng = np.random.default_rng(300 + k)
    q = synth.random_seqs(rng, 1, 40_000)[0]
    seqs = [s.tobytes() for s in synth.random_seqs(rng, 60, 200)]
    seqs[7] = seqs[30] = q.tobytes()
    seqs[3] = q.tobytes() + b"A"
    seqs[2] = b"GT" + q.tobytes()
    seqs[40] = np.concatenate([q[:20_000], synth.mutate(rng, q[20_000:], 0.3)]).tobytes()
    db = synth.SeqSet(seqs)
    qs = [q.tobytes(), q[:5000].tobytes()]

    def run_reference():
        r = _libs.RefDb(db, k=k, id=0.9, maxaccepts=2, maxrejects=16)
        tops = [r.topscores(x) for x in qs]
        th = r.tophits
        r.close()
        return th, _libs.digest(tops), _libs.digest([_libs.ref_unique_kmers(x, k) for x in qs])
    th, tops, kmers = _libs.reference("count_cap_topscores", (db, qs, k), run_reference, _libs.ref() is not None)
    opts = _libs.search_opts(len(db), id=0.9, maxaccepts=2, maxrejects=16, k=k)
    assert opts.tophits == th
    assert _libs.digest([_libs.oracle_unique_kmers(x, k) for x in qs]) == kmers
    assert _libs.oracle_unique_kmers(qs[0], k).shape[0] > 32767
    o = _libs.OracleDb(db, k=k)
    got = [o.topscores(x, opts) for x in qs]
    o.close()
    assert _libs.digest(got) == tops
    assert got[0][0][:5].tolist() == [7, 30, 3, 2, 40] and got[0][1][:4].tolist() == [32767] * 4 and got[0][1][4] < 32767
