"""Traceback on demand pair by pair (vsg_align_pairs_gated): every pair of a gated call against the oracle.

A gated call is what the search driver makes: per query a group of candidates, the first the LEADER, the others its
FOLLOWERS.  A checkpoint task holding followers only runs score-only (align_ckpt.cuh, CK_SCOREONLY); once the leaders'
verdicts are in, the ones phase 2 walks are re-run with stores (CK_RERUN).  A follower whose leader was accepted comes
back "not computed".  Checked here, for every kernel class and rows-per-lane the checkpoint kernels have:
  - every pair's score, followers with a skipped walk included (the only value CK_SCOREONLY produces);
  - every statistic of every leader and of every computed follower;
  - the device's verdict, against the identity test restated in float64 (checkers.leader_accepted);
  - the checkpoint task counts, the skipped-walk count, the ungated aligner and the gated call without score-only
    tasks (VSG_CK_SCOREONLY=0)."""
import contextlib
import os

import numpy as np
import pytest

import checkers
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu

NC = 0xFFFF   # aligned = matches = mismatches = 0xffff: a follower whose walk was skipped
PEN_A = [1, -2, 3, 3, 10, 10, 3, 3, 1, 1, 1, 1, 1, 1]          # test_stress_gpu.py's penalty sets
PEN_B = [5, -4, 0, 0, 12, 16, 0, 0, 0, 0, 3, 2, 0, 0]
# interior gap extension 40: a pair of query padding + target length above ~800 leaves the 16-bit fast kernels'
# exact range and goes to the exact kernel, shorter pairs stay on the checkpoint kernels
PEN_WIDE = [2, -4, 1, 1, 18, 18, 1, 1, 1, 1, 40, 40, 1, 1]
GATES = [(-1.0, 2), (1e9, 2)] + [(100.0 * ident + 1e-7, iddef) for ident in (0.9, 0.97) for iddef in range(5)]


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


def rand_seq(rng, n, alphabet=b"ACGT"):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, a.shape[0], size=n)].tobytes()


def sprinkle(rng, s, p, alphabet=b"NRYKMSWacgtn"):
    """IUPAC / lower-case symbols at a share p of the positions, at least one alphabet[0] (an ambiguous symbol: the
    sequence takes the general-alphabet kernels)"""
    a = np.frombuffer(s, dtype=np.uint8).copy()
    hit = rng.random(a.shape[0]) < p
    sym = np.frombuffer(alphabet, dtype=np.uint8)
    a[hit] = sym[rng.integers(0, sym.shape[0], size=int(hit.sum()))]
    if a.shape[0]:
        a[int(rng.integers(0, a.shape[0]))] = sym[0]
    return a.tobytes()


class World:
    """queries, targets and a pair list made of groups (leader first), as vsg_search_batch builds them"""

    def __init__(self, seed, pen=None, n_mismatch=0, budget=None, strict=True):
        self.rng = np.random.default_rng(seed)
        self.q, self.t, self.pairs, self.leader_of = [], [], [], []
        self.pen, self.n_mismatch, self.budget = pen, n_mismatch, budget
        # strict: every leader is on the checkpoint path and the call plans into one chunk, so a follower is skipped
        # exactly when its leader passes the identity test
        self.strict = strict
        self.no_verdict = set()   # leaders the checkpoint walk never sees (host, exact or multi-strip kernels)
        self.sizes = list(self.rng.permutation(np.arange(1, 9)))

    def query(self, s):
        self.q.append(s)
        return len(self.q) - 1

    def group(self, qi, targets, no_verdict=False):
        lead = len(self.pairs)
        for k, s in enumerate(targets):
            self.t.append(s)
            self.pairs.append((qi, len(self.t) - 1))
            self.leader_of.append(-1 if k == 0 else lead)
        if no_verdict:
            self.no_verdict.add(lead)

    def next_size(self):
        """group sizes 1..8, every one of them in turn: odd sizes leave a leader or follower alone in a task"""
        if not self.sizes:
            self.sizes = list(self.rng.permutation(np.arange(1, 9)))
        return int(self.sizes.pop())

    def mutant(self, root, lo=0.0, hi=0.15):
        return synth.mutate(self.rng, np.frombuffer(root, dtype=np.uint8), float(self.rng.uniform(lo, hi))).tobytes() or b"A"

    def candidate(self, root):
        """mostly relatives of the query at 0-15 % divergence (identities on both sides of 90 and 97 %), some unrelated"""
        if self.rng.random() < 0.8:
            return self.mutant(root)
        return rand_seq(self.rng, max(1, len(root) + int(self.rng.integers(-20, 21))))


def world_rows_per_lane(Q, general=False, mixed=False, seed=0):
    """queries of length Q; general: every query carries IUPAC symbols (CK_GEN only); mixed: ACGT queries whose
    candidates are partly IUPAC, so general and plain tasks of one query are planned apart"""
    w = World(1000 + Q + 7 * general + 13 * mixed + seed)
    for _ in range(6):
        root = rand_seq(w.rng, Q)
        qi = w.query(sprinkle(w.rng, root, 0.03) if general else root)
        for _ in range(2):
            cands = [w.candidate(root) for _ in range(w.next_size())]
            if general or mixed:
                cands = [sprinkle(w.rng, c, 0.03) if (general or w.rng.random() < 0.5) else c for c in cands]
            w.group(qi, cands)
    return w


def world_edges():
    """targets shorter than 32, of exactly 32 and several times the query; halves of very different lengths"""
    w = World(2001)
    for Q in (40, 150, 300):
        root = rand_seq(w.rng, Q)
        qi = w.query(root)

        def of_len(L):
            m = w.mutant(root, 0.0, 0.08)
            if L <= len(m):
                s = int(w.rng.integers(0, len(m) - L + 1))
                return m[s:s + L]
            return rand_seq(w.rng, (L - len(m)) // 2) + m + rand_seq(w.rng, L - len(m) - (L - len(m)) // 2)
        for lens in ([1, 3 * Q], [4 * Q + 5, 7], [31, 32, 33], [32, 5 * Q, 20, 1, Q], [3 * Q, 3 * Q + 1, 2],
                     [Q, 31], [20, 3 * Q, 32, 4 * Q, 1, 33, Q, 2 * Q]):
            w.group(qi, [of_len(L) for L in lens])
    return w


def world_penalties(pen=None, n_mismatch=0, seed=0):
    w = World(3000 + seed, pen=pen, n_mismatch=n_mismatch)
    for Q in (97, 250, 400):
        for _ in range(2):
            root = rand_seq(w.rng, Q)
            qi = w.query(sprinkle(w.rng, root, 0.02, b"N") if n_mismatch and w.rng.random() < 0.5 else root)
            for _ in range(2):
                cands = [w.candidate(root) for _ in range(w.next_size())]
                if n_mismatch:
                    cands = [sprinkle(w.rng, c, 0.02, b"Nn") if w.rng.random() < 0.5 else c for c in cands]
                w.group(qi, cands)
    return w


def world_chunks():
    """a 1 MB scratch budget: a few long tasks per chunk, leaders planned before or after their followers"""
    w = World(4001, budget="1", strict=False)
    for Q in (250, 400):
        for _ in range(3):
            root = rand_seq(w.rng, 1500)
            qi = w.query(w.mutant(root[:Q], 0.0, 0.05))
            for _ in range(2):
                cands = []
                for _ in range(w.next_size()):
                    L = int(w.rng.integers(Q, 1501))
                    s = int(w.rng.integers(0, 1500 - L + 1))
                    cands.append(w.mutant(root[s:s + L], 0.0, 0.1))
                w.group(qi, cands)
    return w


def world_no_verdict():
    """leaders without a device verdict (empty query or target, Q > 512, the exact kernel) and the same pairs as
    followers: the followers of such a leader are always walked"""
    w = World(5001, pen=PEN_WIDE, strict=False)
    root = rand_seq(w.rng, 100)
    qi = w.query(root)
    near = lambda: w.mutant(root, 0.0, 0.05)                                   # noqa: E731
    exact = lambda: near() + rand_seq(w.rng, 1100)                            # noqa: E731  Q 100 x D 1200: exact kernel
    short = lambda: near() + rand_seq(w.rng, int(w.rng.integers(0, 300)))    # noqa: E731  checkpoint kernel
    w.group(qi, [exact(), short(), short(), short(), short()], no_verdict=True)
    w.group(qi, [b"", short(), short(), short()], no_verdict=True)
    w.group(qi, [short(), exact(), b"", short(), short(), short()])
    w.group(qi, [short(), short(), short()])
    root6 = rand_seq(w.rng, 600)
    q6 = w.query(root6)
    w.group(q6, [w.mutant(root6[:100], 0.0, 0.05), w.mutant(root6[:150]), w.mutant(root6), rand_seq(w.rng, 90)],
            no_verdict=True)
    w.group(q6, [w.mutant(root6[:120], 0.0, 0.05), w.mutant(root6[:110])], no_verdict=True)
    q0 = w.query(b"")
    w.group(q0, [rand_seq(w.rng, 50), rand_seq(w.rng, 7), b""], no_verdict=True)
    return w


WORLDS = {
    **{f"prof-Q{Q}": (lambda Q=Q: world_rows_per_lane(Q)) for Q in (1, 31, 33, 65, 97, 160, 161, 200, 250, 256)},
    **{f"lut-Q{Q}": (lambda Q=Q: world_rows_per_lane(Q)) for Q in (257, 300, 384, 448, 512)},
    **{f"gen-Q{Q}": (lambda Q=Q: world_rows_per_lane(Q, general=True)) for Q in (100, 200, 450)},
    **{f"mixed-Q{Q}": (lambda Q=Q: world_rows_per_lane(Q, mixed=True)) for Q in (120, 250, 400)},
    "edges": world_edges,
    "pen-a": lambda: world_penalties(np.array(PEN_A, dtype=np.int64), seed=1),
    "pen-b": lambda: world_penalties(np.array(PEN_B, dtype=np.int64), seed=2),
    "n-mismatch": lambda: world_penalties(n_mismatch=1, seed=3),
    "chunks": world_chunks,
    "no-verdict": world_no_verdict,
}


def make_ctx(w):
    pen = w.pen if w.pen is not None else vlib.DEFAULT_PEN
    if w.budget is None:
        return vlib.Context(0, pen=pen, n_mismatch=w.n_mismatch)
    with env(VSG_DIR_BUDGET_MB=w.budget):
        return vlib.Context(0, pen=pen, n_mismatch=w.n_mismatch)


def stats_of(res, k):
    return (int(res.aligned[k]), int(res.matches[k]), int(res.mismatches[k]), int(res.gaps[k]), tuple(int(x) for x in res.trims[k]))


@pytest.mark.parametrize("name", list(WORLDS))
def test_gated_pairs_vs_oracle(name):
    w = WORLDS[name]()
    lead = np.array(w.leader_of, dtype=np.int32)
    qi = np.array([p[0] for p in w.pairs], dtype=np.uint32)
    ti = np.array([p[1] for p in w.pairs], dtype=np.uint32)
    n = len(w.pairs)
    followers = np.flatnonzero(lead >= 0)
    assert followers.size > 0
    orc = [checkers.oracle_nw16(w.q[a], w.t[b], w.pen, w.n_mismatch) for a, b in w.pairs]
    want = [(o[1], o[2], o[3], o[4], checkers.trims_from_cigar(o[5])) for o in orc]
    ctx = make_ctx(w)
    qs = ctx.seqset(synth.SeqSet(w.q)); ts = ctx.seqset(synth.SeqSet(w.t))
    try:
        with env(VSG_CKPT_MIN_PAIRS="0"):
            plain = ctx.align_pairs(qs, ts, qi, ti)
            for k in range(n):
                assert (int(plain.score[k]),) + stats_of(plain, k) == (orc[k][0],) + want[k], (name, k)
            for threshold, iddef in GATES:
                res, (stored, scoreonly, rerun), skipped = ctx.align_pairs_gated(qs, ts, qi, ti, lead, threshold, iddef)
                with env(VSG_CK_SCOREONLY="0"):
                    res0, counts0, skipped0 = ctx.align_pairs_gated(qs, ts, qi, ti, lead, threshold, iddef)
                case = (name, threshold, iddef, (stored, scoreonly, rerun))
                passes = [checkers.leader_accepted(len(w.q[w.pairs[k][0]]), len(w.t[w.pairs[k][1]]), *want[k][:4], want[k][4],
                                                   iddef, threshold) for k in range(n)]
                bad = []
                nc = np.zeros(n, dtype=bool)
                for k in range(n):
                    g = stats_of(res, k)
                    nc[k] = g[0] == NC and g[1] == NC and g[2] == NC
                    if int(res.score[k]) != orc[k][0]:
                        bad.append(("score", k, int(res.score[k]), orc[k][0]))
                    if lead[k] < 0 or not nc[k]:
                        # `plain` (ungated) equals the oracle: so does every computed pair here
                        if g != want[k]:
                            bad.append(("statistics", k, int(lead[k]), g, want[k]))
                        continue
                    L = int(lead[k])
                    if not passes[L]:
                        bad.append(("skipped, leader not accepted", k, L, want[L]))
                    if L in w.no_verdict:
                        bad.append(("skipped, leader has no verdict", k, L))
                if w.strict:
                    for k in followers:
                        if passes[int(lead[k])] and not nc[k]:
                            bad.append(("walked, leader accepted", int(k), int(lead[k]), want[int(lead[k])]))
                assert not bad, f"{case}: {len(bad)} differences; first: {bad[:4]}"
                assert skipped == int(nc[followers].sum()), case
                # the same result byte for byte with every checkpoint task storing
                for f in ("score", "aligned", "matches", "mismatches", "gaps", "trims"):
                    assert np.array_equal(getattr(res, f), getattr(res0, f)), (case, f)
                assert skipped0 == skipped and counts0 == (stored + scoreonly, 0, 0), (case, counts0)
                # the kernels this test is about ran
                assert scoreonly > 0, case
                assert 0 <= rerun <= scoreonly, case
                if threshold > 1e8:
                    assert skipped == 0 and rerun == scoreonly, case
                if threshold < 0 and w.strict and all(want[k][1] > 0 for k in range(n) if lead[k] < 0):
                    assert rerun == 0 and skipped == followers.size, case
    finally:
        qs.close(); ts.close(); ctx.close()


def test_gated_rejects_bad_leader_lists():
    """leader_of must name, for every follower, a leader of the same call"""
    rng = np.random.default_rng(7)
    root = rand_seq(rng, 120)
    ctx = vlib.Context(0)
    qs = ctx.seqset(synth.SeqSet([root])); ts = ctx.seqset(synth.SeqSet([root, root[:100], root[10:]]))
    qi = np.zeros(3, dtype=np.uint32); ti = np.arange(3, dtype=np.uint32)
    try:
        for lead in ([-1, 3, 0], [-1, 0, 1], [-1, -2, 0], [2, 2, 2], [-1, 1, 0]):
            with pytest.raises(vlib.VsgError, match="leader_of"):
                ctx.align_pairs_gated(qs, ts, qi, ti, np.array(lead, dtype=np.int32), 90.0, 2)
        # a leader may come after its followers
        with env(VSG_CKPT_MIN_PAIRS="0"):
            res, _, skipped = ctx.align_pairs_gated(qs, ts, qi, ti, np.array([2, 2, -1], dtype=np.int32), -1.0, 2)
        assert skipped == 2 and int(res.matches[2]) == 110 and int(res.score[0]) == 240
    finally:
        qs.close(); ts.close(); ctx.close()
