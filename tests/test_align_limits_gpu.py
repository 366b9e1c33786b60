"""The aligner at the edges of its kernel classes, against the oracle.

vsg_api.cu's plan_pairs sends each pair to one of five paths from its lengths and the scoring: resolved on the host
(a sentinel when the pair does not fit the reference's 16-bit aligner), the exact kernel (one saturating thread per
pair), the checkpoint kernels (align_ckpt.cuh + tb_ckpt.h, under the shifted scoring), or the direction-bit kernel in
one or in several strips.  The bounds that pick a path are conservative by design; these tests put pairs on both sides
of every bound, check that each pair ran where `path_of` (the planner's rules restated) says, and drive the values
towards the 16-bit limits the bounds protect:
  - the sweep: every rows-per-lane class, D at the last checkpoint and the last 16-bit-kernel length and one either
    side, under penalty sets that reach scores of -20 000 and +25 000 and the exact kernel's overflow sentinel;
  - the checkpoint kernels against targets up to their bound (~10 kb under default penalties), the usual amplicon
    against reference shape, ungated and gated;
  - the direction-bit and exact kernels up to the first target length at which the reference's overflow flag fires,
    and the fits16 limits (Q * D = 25 000 000, Q + D = 65 535);
  - tasks larger than the whole direction budget, and the search driver on 3-15 kb targets.
Every pair is compared with checkers.oracle_nw16: score, statistics, trims and CIGAR."""
import concurrent.futures
import contextlib
import os

import numpy as np
import pytest

import checkers
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu

SENTINEL = 32767
NC = 0xFFFF   # aligned = matches = mismatches = 0xffff: a follower whose walk was skipped
DEFAULT = list(vlib.DEFAULT_PEN)
PEN_A = [1, -2, 3, 3, 10, 10, 3, 3, 1, 1, 1, 1, 1, 1]          # test_stress_gpu.py's penalty sets
PEN_B = [5, -4, 0, 0, 12, 16, 0, 0, 0, 0, 3, 2, 0, 0]
PEN_WIDE = [2, -4, 1, 1, 18, 18, 1, 1, 1, 1, 40, 40, 1, 1]    # test_gated_align_gpu.py
HARSH = [2, -80] + [20] * 6 + [40] * 6
BIG60 = [60, -4] + DEFAULT[2:]
BIG64 = [64, -4] + DEFAULT[2:]
CKPT_MIN_PAIRS = 2048   # plan_pairs' default VSG_CKPT_MIN_PAIRS


@contextlib.contextmanager
def env(**kv):
    """set (str) or unset (None) environment variables for the duration"""
    old = {k: os.environ.get(k) for k in kv}
    for k, v in kv.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- the planner's rules, restated (vsg_api.cu: build_score_params, shifted_params, fits16, fast_shape,
# ---- fast_bound_of / fast_path_ok, plan_pairs) -----------------------------------------------------------------------

def score_params(pen):
    """(match, mismatch, go[6], ge[6], fallback): the clamps of build_score_params"""
    lim = [32767, 32767] + [32767 // 5] * 12
    fallback = any(int(v) > m or int(v) < -m for v, m in zip(pen, lim))
    v = [max(-m, min(m, int(x))) for x, m in zip(pen, lim)]
    return v[0], v[1], v[2:8], v[8:14], fallback


def bound_of(table, go, ge):
    """fast_bound_of: `table` holds the values of the 16 x 16 score table.  The table always has ambiguous-symbol
    entries besides match and mismatch, so n_mismatch (which turns some of them into mismatches) leaves the set of
    values, and with it every bound, as it is."""
    return (all(x >= 0 for x in go + ge), max(a + b for a, b in zip(go, ge)), max(ge), max(table), min(table))


def path_ok(b, qpad, d):
    """fast_path_ok: every intermediate of a (qpad x d) problem fits the biased 16-bit kernels"""
    valid, G, Rm, smax, smin = b
    if not valid:
        return False
    lb = -(G + qpad * Rm) - G - (d + 4) * Rm - 2 * G + smin
    ub = smax * min(qpad, d + 4) + smax
    return lb > -32700 and ub < 32700


def bounds(pen):
    """(fallback, bound of the scoring, bound of the shifted scoring or None when shifted_params refuses it)"""
    match, mismatch, go, ge, fallback = score_params(pen)
    b = bound_of((match, mismatch, 0), go, ge)
    c = (max(match, mismatch, 0) + 1) // 2
    table2 = (match - 2 * c, mismatch - 2 * c, -2 * c)
    ge2 = [g + c for g in ge]
    ok = all(-32767 <= v <= 32767 for v in table2 + tuple(ge2)) and table2[0] >= table2[1]
    return fallback, b, (bound_of(table2, go, ge2) if ok else None)


def fits16(q, d):
    return q + d <= 65535 and q * d <= 25_000_000


def fast_shape(Q, general):
    """(rows per lane, strips)"""
    ns = (Q + 511) // 512
    R = max(1, (Q + 32 * ns - 1) // (32 * ns))
    if general:
        R = 4 if R <= 4 else (8 if R <= 8 else 16)
    return R, (Q + 32 * R - 1) // (32 * R)


def path_of(Q, D, general, pen, n_mismatch=0, any_size=False):
    """The kernel plan_pairs gives a pair that is alone in its task (its query has no other target of the same
    alphabet class in the call): "host", "exact", "ckpt", "dirbits" or "strips".  any_size: the call has at least
    VSG_CKPT_MIN_PAIRS pairs.  n_mismatch does not move a bound (bound_of)."""
    fallback, b, b2 = bounds(pen)
    if fallback or Q == 0 or D == 0 or not fits16(Q, D):
        return "host"
    R, ns = fast_shape(Q, general)
    if not path_ok(b, ns * 32 * R, D):
        return "exact"
    if ns == 1 and b2 is not None and (any_size or D >= 3 * Q) and path_ok(b2, 32 * R, D):
        return "ckpt"
    return "dirbits" if ns == 1 else "strips"


def last_d(pred, hi=65535):
    """the largest D in [1, hi] for which pred holds, pred true up to it and false beyond (0: none)"""
    if not pred(1):
        return 0
    lo = 1
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if pred(mid):
            lo = mid
        else:
            hi = mid - 1
    return lo


def limits(Q, general, pen):
    """(D_ck, D_fast): the last target length on the checkpoint kernels (at any call size) and on the 16-bit kernels"""
    d_ck = last_d(lambda D: path_of(Q, D, general, pen, any_size=True) == "ckpt")
    d_fast = last_d(lambda D: path_of(Q, D, general, pen, any_size=True) in ("ckpt", "dirbits", "strips"))
    return d_ck, d_fast


def test_path_predictor_restates_the_planner():
    """path_of by hand at a few points, so that a slip in the restatement does not hide behind the sweep"""
    assert path_of(0, 10, False, DEFAULT) == "host" and path_of(10, 0, False, DEFAULT) == "host"
    assert path_of(500, 50000, False, DEFAULT) == "exact" and path_of(500, 50001, False, DEFAULT) == "host"
    assert path_of(1, 65534, False, DEFAULT) == "exact" and path_of(1, 65535, False, DEFAULT) == "host"
    assert path_of(250, 1000, False, DEFAULT) == "ckpt" and path_of(250, 700, False, DEFAULT) == "dirbits"
    assert path_of(250, 700, False, DEFAULT, any_size=True) == "ckpt"
    assert path_of(513, 700, False, DEFAULT, any_size=True) == "strips"
    # default penalties, R = 16: shifted bound G 21, Rm 3, smin -6 -> (D + 4) * 3 < 32700 - 21 - 1536 - 21 - 42 - 6
    assert limits(512, False, DEFAULT)[0] == (32700 - 21 - 512 * 3 - 21 - 42 - 6 - 1) // 3 - 4
    # match 64, R = 16: the upper bound 64 * min(512, D + 4) + 64 < 32700 decides
    assert limits(512, False, BIG64)[1] == 505
    assert bounds([2, -4, 7000] + DEFAULT[3:])[0]


# ---- the oracle, cached per pair and run on every core (ctypes drops the GIL) ---------------------------------------

_oracle_cache = {}


def oracle_many(pairs, pen=None, n_mismatch=0):
    """checkers.oracle_nw16 of every (query bytes, target bytes) in `pairs`"""
    key = lambda q, t: (q, t, None if pen is None else tuple(int(x) for x in pen), n_mismatch)   # noqa: E731
    todo = list({key(q, t): (q, t) for q, t in pairs if key(q, t) not in _oracle_cache}.items())
    if todo:
        checkers.oracle()
        penarr = None if pen is None else np.array(pen, dtype=np.int64)
        with concurrent.futures.ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
            outs = ex.map(lambda kv: checkers.oracle_nw16(kv[1][0], kv[1][1], penarr, n_mismatch), todo)
            for (k, _), o in zip(todo, outs):
                _oracle_cache[k] = o
    return [_oracle_cache[key(q, t)] for q, t in pairs]


def rand_seq(rng, n, alphabet=b"ACGT"):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, a.shape[0], size=n)].tobytes()


def mutant(rng, s, rate):
    return synth.mutate(rng, np.frombuffer(s, dtype=np.uint8), rate).tobytes() or b"A"


def sprinkle(rng, s, p=0.03, alphabet=b"NRYKMSWacgtn"):
    """IUPAC / lower-case symbols at a share p of the positions and at least one N: the general-alphabet kernels"""
    a = np.frombuffer(s, dtype=np.uint8).copy()
    hit = rng.random(a.shape[0]) < p
    sym = np.frombuffer(alphabet, dtype=np.uint8)
    a[hit] = sym[rng.integers(0, sym.shape[0], size=int(hit.sum()))]
    a[int(rng.integers(0, a.shape[0]))] = sym[0]
    return a.tobytes()


def fit_to(rng, m, D, where):
    """a target of exactly D symbols holding m (a relative of the query) at the start, end or middle of random
    flanks, split in two around a random insert, or a window of m when D is shorter"""
    if D <= len(m):
        s = int(rng.integers(0, len(m) - D + 1))
        return m[s:s + D]
    fill = rand_seq(rng, D - len(m))
    if where == "start":
        return m + fill
    if where == "end":
        return fill + m
    if where == "split" and len(m) >= 2:
        h = len(m) // 2
        return m[:h] + fill + m[h:]
    a = len(fill) // 2
    return fill[:a] + m + fill[a:]


# ---- checking one call's pairs --------------------------------------------------------------------------------------

def stats_of(res, k):
    return (int(res.score[k]), int(res.aligned[k]), int(res.matches[k]), int(res.mismatches[k]), int(res.gaps[k]),
            tuple(int(x) for x in res.trims[k]))


def want_of(o):
    return (o[0], o[1], o[2], o[3], o[4], checkers.trims_from_cigar(o[5]))


class Call:
    """one aligner call: queries, targets and pairs uploaded once, the oracle's answer for every pair"""

    def __init__(self, ctx, qseqs, tseqs, pairs, pen=None, n_mismatch=0, leader_of=None):
        self.ctx, self.qseqs, self.tseqs, self.pairs = ctx, qseqs, tseqs, pairs
        self.qs = ctx.seqset(synth.SeqSet(qseqs))
        self.ts = ctx.seqset(synth.SeqSet(tseqs))
        self.qi = np.array([p[0] for p in pairs], dtype=np.uint32)
        self.ti = np.array([p[1] for p in pairs], dtype=np.uint32)
        self.lead = np.full(len(pairs), -1, dtype=np.int32) if leader_of is None else np.array(leader_of, dtype=np.int32)
        self.orc = oracle_many([(qseqs[a], tseqs[b]) for a, b in pairs], pen, n_mismatch)
        self.want = [want_of(o) for o in self.orc]

    def close(self):
        self.qs.close(); self.ts.close()

    def describe(self, k):
        a, b = self.pairs[k]
        return dict(pair=k, Q=len(self.qseqs[a]), D=len(self.tseqs[b]))

    def ungated(self, what):
        """align_pairs with and without CIGARs: every pair equals the oracle; returns the CIGAR call's result"""
        res = self.ctx.align_pairs(self.qs, self.ts, self.qi, self.ti, cigar=True)
        res2 = self.ctx.align_pairs(self.qs, self.ts, self.qi, self.ti, cigar=False)
        bad = []
        for k in range(len(self.pairs)):
            g, g2 = stats_of(res, k), stats_of(res2, k)
            if g != self.want[k] or g2 != self.want[k] or res.cigars[k] != self.orc[k][5]:
                bad.append((self.describe(k), self.want[k], g, g2, res.cigars[k][:40], self.orc[k][5][:40]))
            if self.orc[k][0] == SENTINEL:   # include/vsg.h: zero statistics and an empty CIGAR
                assert g[1:] == (0, 0, 0, 0, (0, 0, 0, 0)) and res.cigars[k] == "", (what, self.describe(k), g)
        assert not bad, f"{what}: {len(bad)} of {len(self.pairs)} pairs differ from the oracle; first: {bad[:3]}"
        assert (res.fast_pairs, res.exact_pairs) == (res2.fast_pairs, res2.exact_pairs), what
        return res

    def gated(self, what, threshold=-1.0, iddef=2):
        """align_pairs_gated with this call's leader list, checked as test_gated_align_gpu.py does; returns
        (result, checkpoint task counts, skipped walks)"""
        res, counts, skipped = self.ctx.align_pairs_gated(self.qs, self.ts, self.qi, self.ti, self.lead, threshold, iddef)
        n = len(self.pairs)
        bad = []
        nc = 0
        for k in range(n):
            g = stats_of(res, k)
            if g[0] != self.want[k][0]:
                bad.append(("score", self.describe(k), g[0], self.want[k][0]))
            skip = self.lead[k] >= 0 and g[1] == NC and g[2] == NC and g[3] == NC
            if not skip:
                if g != self.want[k]:
                    bad.append(("statistics", self.describe(k), g, self.want[k]))
                continue
            nc += 1
            L = int(self.lead[k])
            a, b = self.pairs[L]
            if not checkers.leader_accepted(len(self.qseqs[a]), len(self.tseqs[b]), *self.want[L][1:5], self.want[L][5],
                                            iddef, threshold):
                bad.append(("skipped, leader not accepted", self.describe(k), L))
        assert not bad, f"{what}: {len(bad)} differences; first: {bad[:3]}"
        assert skipped == nc, what
        return res, counts, skipped


# ---- a. the boundary sweep ------------------------------------------------------------------------------------------

R_CLASSES = [(R, False) for R in range(1, 17)] + [(R, True) for R in (4, 8, 16)]
SWEEP = {
    "default": (DEFAULT, 0),
    "pen-a": (PEN_A, 0),
    "pen-b": (PEN_B, 0),
    "pen-wide": (PEN_WIDE, 0),
    "harsh": (HARSH, 0),
    "big-match-60": (BIG60, 0),
    "big-match-64": (BIG64, 0),
    "n-mismatch": (DEFAULT, 1),
}


def sweep_world(name, pen):
    """per R class and Q in {32R, 32R - 1}: a near-copy of the query and an unrelated sequence at each D of
    {D_ck - 1, D_ck, D_ck + 1, D_fast - 1, D_fast, D_fast + 1}; one target per query, so tasks are pairs"""
    rng = np.random.default_rng(7000 + sorted(SWEEP).index(name))
    qseqs, tseqs, pairs, meta = [], [], [], []
    for R, general in R_CLASSES:
        for Q in (32 * R, 32 * R - 1):
            d_ck, d_fast = limits(Q, general, pen)
            Ds = sorted({D for D in (d_ck - 1, d_ck, d_ck + 1, d_fast - 1, d_fast, d_fast + 1) if D >= 1 and fits16(Q, D)})
            root = rand_seq(rng, Q)
            q = sprinkle(rng, root) if general else root
            for D in Ds:
                near = fit_to(rng, mutant(rng, root, 0.01), D, "middle")
                for kind, t in (("near", near), ("unrelated", rand_seq(rng, D))):
                    qseqs.append(q)
                    tseqs.append(sprinkle(rng, t) if general else t)
                    pairs.append((len(qseqs) - 1, len(tseqs) - 1))
                    meta.append(dict(R=R, general=general, Q=Q, D=D, kind=kind, d_ck=d_ck, d_fast=d_fast))
    return qseqs, tseqs, pairs, meta


@pytest.mark.parametrize("name", list(SWEEP))
def test_boundary_sweep(name):
    pen, nm = SWEEP[name]
    qseqs, tseqs, pairs, meta = sweep_world(name, pen)
    ctx = vlib.Context(0, pen=pen, n_mismatch=nm)
    call = Call(ctx, qseqs, tseqs, pairs, pen, nm)
    try:
        n = len(pairs)
        for min_pairs in ("0", None):
            with env(VSG_CKPT_MIN_PAIRS=min_pairs):
                paths = [path_of(m["Q"], m["D"], m["general"], pen, nm, any_size(n)) for m in meta]
                want = {p: paths.count(p) for p in ("host", "exact", "ckpt", "dirbits", "strips")}
                what = (name, "VSG_CKPT_MIN_PAIRS", min_pairs, want)
                res = call.ungated(what)
                _, (stored, scoreonly, rerun), _ = call.gated(what)
            assert res.exact_pairs == want["exact"], (what, res.exact_pairs)
            assert res.fast_pairs == want["ckpt"] + want["dirbits"] + want["strips"], (what, res.fast_pairs)
            assert (stored, scoreonly, rerun) == (want["ckpt"], 0, 0), (what, stored, scoreonly, rerun)
            assert want["ckpt"] > 0 and want["dirbits"] > 0 and want["exact"] > 0, what
        score = {(m["R"], m["general"], m["Q"], m["D"], m["kind"]): o[0] for m, o in zip(meta, call.orc)}
        if pen is HARSH:
            # the sweep only bites where the values really approach the limits: an unrelated pair at the bounds
            # scores below -12 000 at every R, and below -20 000 at R <= 4, where the target's end gap dominates
            for R, general in R_CLASSES:
                Q = 32 * R
                d_ck, d_fast = limits(Q, general, pen)
                for D in (d_ck, d_fast):
                    s = score[(R, general, Q, D, "unrelated")]
                    assert s < (-20000 if R <= 4 else -12000), (R, general, D, s)
        if pen is BIG60 or pen is BIG64:
            near = [s for (R, g, Q, D, kind), s in score.items() if kind == "near" and s != SENTINEL]
            assert max(near) > 25000, max(near)
    finally:
        call.close(); ctx.close()


def test_identical_pair_overflows_at_match_64():
    """512 x 512 identical under match 64 scores 32 768: the reference's overflow flag, so a sentinel"""
    rng = np.random.default_rng(7100)
    q = rand_seq(rng, 512)
    ctx = vlib.Context(0, pen=BIG64)
    call = Call(ctx, [q], [q, q[:500], mutant(rng, q, 0.01)], [(0, 0), (0, 1), (0, 2)], BIG64)
    try:
        assert call.orc[0][0] == SENTINEL and call.orc[1][0] != SENTINEL and call.orc[1][0] > 25000
        res = call.ungated("match 64")
        assert int(res.score[0]) == SENTINEL and res.exact_pairs >= 1
    finally:
        call.close(); ctx.close()


# ---- b. long targets on the checkpoint kernels ----------------------------------------------------------------------

LONG_Q = (1, 33, 100, 250, 256, 257, 400, 512)
SHAPES = ("start", "end", "middle", "split", "unrelated")


def long_world(seed, n_mismatch=0):
    """per query length: the five target shapes at D in {2 600, 6 000, D_ck - 1, D_ck}, one group per D with the leader
    first; a query copy whose only task pairs a 10 000 nt target with a 40 nt one; a query copy with IUPAC targets.
    n_mismatch: N in every query, so every pair runs on the general-alphabet kernels.  Each query copy holds one
    alphabet class, so the planner pairs its targets two by two.  Returns (qseqs, tseqs, pairs, leader_of, general
    per pair, number of tasks)."""
    rng = np.random.default_rng(seed)
    qseqs, tseqs, pairs, lead, general = [], [], [], [], []
    ntasks = 0

    def group(q, targets, g):
        nonlocal ntasks
        qseqs.append(q)
        first = len(pairs)
        for k, t in enumerate(targets):
            tseqs.append(t)
            pairs.append((len(qseqs) - 1, len(tseqs) - 1))
            lead.append(-1 if k == 0 else first)
            general.append(g)
        ntasks += (len(targets) + 1) // 2
    for Q in LONG_Q:
        root = rand_seq(rng, Q)
        g = bool(n_mismatch)
        q = sprinkle(rng, root, 0.02, b"N") if g else root
        d_ck = limits(Q, g, DEFAULT)[0]
        for D in sorted({2600, 6000, d_ck - 1, d_ck}):
            targets = [rand_seq(rng, D) if shape == "unrelated" else fit_to(rng, mutant(rng, root, 0.04), D, shape)
                       for shape in SHAPES]
            group(q, [sprinkle(rng, t, 0.01, b"Nn") for t in targets] if g else targets, g)
        group(q, [fit_to(rng, mutant(rng, root, 0.03), 10000, "end"), fit_to(rng, mutant(rng, root, 0.03), 40, "start")], g)
        if not g:
            d_gen = limits(Q, True, DEFAULT)[0]
            group(q, [sprinkle(rng, fit_to(rng, mutant(rng, root, 0.04), D, shape))
                      for D, shape in ((d_gen, "start"), (d_gen - 1, "end"), (4000, "middle"))], True)
    return qseqs, tseqs, pairs, lead, general, ntasks


@pytest.mark.parametrize("n_mismatch", [0, 1])
def test_long_targets_on_checkpoint_kernels(n_mismatch):
    qseqs, tseqs, pairs, lead, general, ntasks = long_world(8000 + n_mismatch, n_mismatch)
    for (a, b), g in zip(pairs, general):
        Q, D = len(qseqs[a]), len(tseqs[b])
        assert D == 40 or path_of(Q, D, g, DEFAULT) == "ckpt", (Q, D, g)   # the 40 nt half rides in a 10 000 nt task
    ctx = vlib.Context(0, n_mismatch=n_mismatch)
    call = Call(ctx, qseqs, tseqs, pairs, None, n_mismatch, lead)
    try:
        assert sum(o[0] == SENTINEL for o in call.orc) == 0
        n = len(pairs)
        for min_pairs in ("0", None):
            with env(VSG_CKPT_MIN_PAIRS=min_pairs):
                res = call.ungated(("long", n_mismatch, min_pairs))
                assert (res.fast_pairs, res.exact_pairs) == (n, 0)
                for threshold in (-1.0, 1e9):
                    what = ("long", n_mismatch, min_pairs, threshold)
                    r1, (stored, scoreonly, rerun), skipped = call.gated(what, threshold)
                    with env(VSG_CK_SCOREONLY="0"):
                        r0, counts0, skipped0 = call.gated(what + ("VSG_CK_SCOREONLY=0",), threshold)
                    assert stored + scoreonly == ntasks and counts0 == (ntasks, 0, 0), (what, stored, scoreonly, counts0)
                    assert scoreonly > 0 and 0 <= rerun <= scoreonly, what
                    assert skipped0 == skipped, what
                    for f in ("score", "aligned", "matches", "mismatches", "gaps", "trims"):
                        assert np.array_equal(getattr(r1, f), getattr(r0, f)), (what, f)
                    if threshold > 1e8:
                        assert skipped == 0 and rerun == scoreonly, what
                    else:
                        assert skipped > 0, what
    finally:
        call.close(); ctx.close()


# ---- c. direction bits and the exact kernel up to the 16-bit limits -------------------------------------------------

def first_sentinel(q, family, lo, hi):
    """bisection on D with the oracle: the first D in (lo, hi] at which (q, family(D)) is a sentinel, given that lo
    is not and hi is"""
    is_sent = lambda D: oracle_many([(q, family(D))])[0][0] == SENTINEL   # noqa: E731
    assert not is_sent(lo) and is_sent(hi), (lo, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if is_sent(mid):
            hi = mid
        else:
            lo = mid
    return hi


def exact_world():
    """Q 250 against D from D_ck + 1 to past the overflow edge, both sides of the edge, and the fits16 limits:
    Q * D = 25 000 000 (500 x 50 000, 1 000 x 25 000) and one more, Q + D = 65 535 (1 x 65 534) and one more.
    Returns (qseqs, tseqs, pairs, the first D at which the Q 250 family is a sentinel)."""
    rng = np.random.default_rng(9000)
    root, r1000 = rand_seq(rng, 250), rand_seq(rng, 1000)
    qseqs = [root, rand_seq(rng, 500), r1000, b"G"]
    base = mutant(rng, root, 0.03) + rand_seq(rng, 40000)
    family = lambda D: base[:D]   # noqa: E731  the query at the start: a trailing end gap of D - 250
    d_ck, d_fast = limits(250, False, DEFAULT)
    edge = first_sentinel(root, family, d_fast + 1, 40000)
    tseqs, pairs = [], []

    def add(qi, t):
        tseqs.append(t)
        pairs.append((qi, len(tseqs) - 1))
    for D in sorted({d_ck + 1, d_ck + 2, 12000, d_fast - 1, d_fast, d_fast + 1, 20000, 25000, 30000, edge - 1, edge, 33000}):
        add(0, family(D))
    add(0, fit_to(rng, mutant(rng, root, 0.03), d_ck + 1, "end"))
    add(0, fit_to(rng, mutant(rng, root, 0.03), d_fast, "split"))
    add(0, fit_to(rng, mutant(rng, root, 0.03), d_fast + 1, "end"))
    add(1, rand_seq(rng, 50000)); add(1, rand_seq(rng, 50001))
    add(2, fit_to(rng, mutant(rng, r1000, 0.03), 25000, "middle")); add(2, fit_to(rng, r1000, 25001, "middle"))
    add(3, rand_seq(rng, 65534)); add(3, rand_seq(rng, 65535))
    return qseqs, tseqs, pairs, edge


def any_size(npairs):
    """does a call of npairs pairs reach VSG_CKPT_MIN_PAIRS as the environment sets it now"""
    return npairs >= int(os.environ.get("VSG_CKPT_MIN_PAIRS", CKPT_MIN_PAIRS))


def predicted(qseqs, tseqs, pairs):
    """(fast, exact) pair counts of a call of plain pairs, and each pair's path (path_of: as if alone in its task)"""
    paths = [path_of(len(qseqs[a]), len(tseqs[b]), False, DEFAULT, any_size=any_size(len(pairs))) for a, b in pairs]
    return sum(p in ("ckpt", "dirbits", "strips") for p in paths), paths.count("exact"), paths


def test_direction_bits_and_exact_kernel_to_the_limits():
    """(VSG_CKPT_MIN_PAIRS does not matter here: every pair is past the checkpoint bound)"""
    qseqs, tseqs, pairs, edge = exact_world()
    ctx = vlib.Context(0)
    call = Call(ctx, qseqs, tseqs, pairs)
    try:
        score = {(len(qseqs[a]), len(tseqs[b])): o[0] for (a, b), o in zip(pairs, call.orc)}
        assert score[(250, edge)] == SENTINEL and score[(250, edge - 1)] != SENTINEL
        assert score[(1000, 25000)] != SENTINEL and score[(1000, 25001)] == SENTINEL and score[(500, 50001)] == SENTINEL
        nfast, nexact, paths = predicted(qseqs, tseqs, pairs)
        assert paths[-6:] == ["exact", "host", "exact", "host", "exact", "host"], paths
        assert "ckpt" not in paths and paths.count("dirbits") >= 5, paths
        res = call.ungated("exact")
        call.gated("exact")
        assert (res.fast_pairs, res.exact_pairs) == (nfast, nexact), (res.fast_pairs, res.exact_pairs, paths)
    finally:
        call.close(); ctx.close()


# ---- d. tasks larger than the whole direction budget -----------------------------------------------------------------

def test_tasks_larger_than_the_budget():
    """A 1 MB direction budget.  Every task here needs more on its own: a checkpoint task of D >= 5 000 about 256 bytes
    a column, a direction-bit task of R = 8 about 256, an exact task Q * D.  So each one gets a chunk, and a forward
    launch, of its own.  One target per query: tasks are pairs."""
    rng = np.random.default_rng(9300)
    qseqs, tseqs = [], []
    for Q in (1, 250, 512):
        root = rand_seq(rng, Q)
        d_ck = limits(Q, False, DEFAULT)[0]
        for D, shape in ((6000, "start"), (d_ck, "end"), (d_ck - 1, "split"), (10000, "unrelated")):
            qseqs.append(root)
            tseqs.append(rand_seq(rng, D) if shape == "unrelated" else fit_to(rng, mutant(rng, root, 0.04), D, shape))
    eq, et, ep, edge = exact_world()
    for a, b in ep:
        if (len(eq[a]), len(et[b])) in ((250, 12000), (250, 20000), (250, edge), (1000, 25000)):
            qseqs.append(eq[a]); tseqs.append(et[b])
    pairs = [(k, k) for k in range(len(qseqs))]
    with env(VSG_DIR_BUDGET_MB="1"):
        ctx = vlib.Context(0)
    call = Call(ctx, qseqs, tseqs, pairs)
    try:
        nfast, nexact, paths = predicted(qseqs, tseqs, pairs)
        assert paths.count("ckpt") == 12 and paths.count("dirbits") == 1 and paths.count("exact") == 3, paths
        res = call.ungated("budget")
        assert ctx.profile().fwd_launches == len(pairs)
        assert (res.fast_pairs, res.exact_pairs) == (nfast, nexact), paths
        call.gated("budget")
        assert ctx.profile().fwd_launches == len(pairs)
    finally:
        call.close(); ctx.close()


# ---- e. the search shape ----------------------------------------------------------------------------------------------

def test_search_amplicons_against_long_references():
    """250 nt queries sampled from 40 references of 3-15 kb and mutated, searched with default options: the search
    driver's gated rounds on the checkpoint kernels, every row against the oracle"""
    rng = np.random.default_rng(9500)
    dbl = [rand_seq(rng, int(rng.integers(3000, 15001))) for _ in range(40)]
    qsl = []
    for i in range(96):
        src = dbl[int(rng.integers(0, 40))]
        s = int(rng.integers(0, len(src) - 250 + 1))
        qsl.append(mutant(rng, src[s:s + 250], float(rng.uniform(0.0, 0.08))))
    dbs, qss = synth.SeqSet(dbl), synth.SeqSet(qsl)
    ctx = vlib.Context(0)
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, 8, 0)
    try:
        o = vlib.default_search_opts()
        res, counts, _ = ctx.search(ix, db, qs, 0, len(qsl), o, len(dbl))
        assert checkers.check_search_rows(res, counts, len(dbl), qss, dbs) >= len(qsl)
    finally:
        ix.close(); db.close(); qs.close(); ctx.close()
