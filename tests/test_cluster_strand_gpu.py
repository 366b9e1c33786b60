"""--strand both for vsg_cluster_fast, cluster sessions and the clustering shim.

Every sequence is searched as itself and as its reverse complement (the reference's cluster.cpp:162-189, 920-957):
the reads here come in both orientations, so that many sequences join a cluster through the reverse complement.  The
results must be those of the unmodified reference, strand column and CIGAR of the reverse-complemented query included.
The reference's CLI records are stored as digests in tests/golden/cluster_strand_reference.json (see _reference)."""
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
RESULTS = os.path.join(ROOT, "tests", "golden", "cluster_strand_reference.json")


def _reference(name, inputs, compute, available):
    """checkers.reference with this file's own record file: what the unmodified reference returned for `inputs`, keyed
    by `name` and a hash of the inputs.  With the compiled reference present and VSG_RECORD_REFERENCE=<file>,
    `compute()` runs it and the result is added to <file>; copying that file to RESULTS makes the record the tests use."""
    h = hashlib.sha256()
    checkers._feed(h, inputs)
    key = f"{name}:{h.hexdigest()[:24]}"
    out = os.environ.get("VSG_RECORD_REFERENCE")
    if out and available:
        val = checkers.canon(compute())
        rec = json.load(open(out)) if os.path.exists(out) else {}
        rec[key] = val
        with open(out, "w") as f:      # one record per line
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


_COMP = bytes.maketrans(b"ACGTURYSWKMBDHVNacgturyswkmbdhvn", b"TGCAAYRSWMKVHDBNtgcaayrswmkvhdbn")


def _rc(s: bytes) -> bytes:
    """reverse complement of an ASCII sequence; any byte that is not an IUPAC code becomes 'N'"""
    s = bytes(c if c in b"ACGTURYSWKMBDHVNacgturyswkmbdhvn" else ord("N") for c in s)
    return s.translate(_COMP)[::-1]


def _reads(n, nroots, seed, divs=(0.01, 0.01, 0.02, 0.035, 0.05), npal=3):
    """test_cluster_gpu's amplicon reads, about a third of them reverse-complemented, a few with IUPAC codes, DUST bait,
    and exact, symmetrically trimmed copies of palindromic roots (second half = reverse complement of the first):
    such a read is its own reverse complement, so its plus and minus alignments are the same and the plus strand wins"""
    rng = np.random.default_rng(seed)
    roots = synth.random_seqs(rng, nroots, 300)
    w = 1.0 / np.arange(1, nroots + 1); w /= w.sum()
    pick = rng.choice(nroots, size=n, p=w)
    pal = []
    for _ in range(npal):
        half = synth.random_seqs(rng, 1, 150)[0].tobytes()
        pal.append(half + _rc(half))
    seqs, palindromic = [], set()
    for i in range(n):
        if i % 50 == 3:
            p = pal[(i // 50) % npal]
            t = int(rng.integers(0, 6))
            s = p[t: len(p) - t]
            palindromic.add(i)
        else:
            m = synth.mutate(rng, roots[int(pick[i])], float(divs[int(rng.integers(0, len(divs)))]))
            a = int(rng.integers(0, 6)); b = int(rng.integers(0, 6))
            s = m[a: m.shape[0] - b].tobytes()
            if i % 97 == 5:
                s = s[:100] + b"AT" * 30 + s[100:]      # DUST bait
            if i % 89 == 7:
                s = s[:60] + b"NRY" + s[63:]            # IUPAC codes: the general kernels
            if rng.random() < 1.0 / 3.0:
                s = _rc(s)
        seqs.append(s)
    return seqs, palindromic


def _uc_records(text):
    rec = {}
    for line in text.decode().splitlines(True):
        f = line.rstrip("\n").split("\t")
        if f[0] == "S":
            rec[f[8]] = ("S", int(f[1]), "*", "*", "*", "*")
        elif f[0] == "H":
            rec[f[8]] = ("H", int(f[1]), f[3], f[4], f[9], f[7])
    return rec


def _sorted(seqs, labels):
    # Database::sortbylength (core/db.cpp:433-449): length descending, abundance descending, label ascending
    return sorted(range(len(seqs)), key=lambda i: (-len(seqs[i]), labels[i]))


CLI_CASES = {
    "dust": ([], {}),
    "qmask_none": (["--qmask", "none"], {"mask_lower": 0}),
    "id90": (["--id", "0.90", "--maxaccepts", "4", "--maxrejects", "16"], {"id": 0.90, "maxaccepts": 4, "maxrejects": 16}),
    "iddef1": (["--iddef", "1"], {"iddef": 1}),
}


@pytest.mark.parametrize("threads,n,nroots,case", [(1, 1500, 40, "dust"), (2, 2000, 40, "qmask_none"), (8, 3000, 120, "id90"),
                                                   (64, 6000, 400, "iddef1"), (128, 8000, 150, "dust"), (8, 3000, 120, "iddef1"),
                                                   (64, 6000, 400, "qmask_none")])
def test_cluster_fast_both_strands_equals_reference_cli(tmp_path, threads, n, nroots, case):
    seqs, palindromic = _reads(n, nroots, seed=300 + threads)
    labels = [f"b{i:07d}" for i in range(n)]
    extra, opts = CLI_CASES[case]
    fa = str(tmp_path / "reads.fasta")
    with open(fa, "wb") as f:
        for l, s in zip(labels, seqs):
            f.write(b">" + l.encode() + b"\n" + s + b"\n")
    uc = str(tmp_path / "ref.uc")

    def reduce(text):
        rec = _uc_records(text)
        return sum(1 for v in rec.values() if v[0] == "S"), checkers.digest(sorted(rec.items()))
    args = ["--id", "0.97"] + extra if "--id" not in extra else list(extra)
    nclusters, want = _reference(
        "cluster_fast_strand_both", (seqs, labels, args, threads),
        lambda: checkers.run_stock(["--cluster_fast", fa] + args + ["--strand", "both", "--threads", str(threads), "--uc", uc, "--quiet"],
                                   [uc], reduce), os.path.exists(STOCK))
    order = _sorted(seqs, labels)
    ctx = vlib.Context(0)
    ss = ctx.seqset(synth.SeqSet([seqs[i] for i in order]))
    o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxrejects = 8; o.strand_both = 1
    for k, v in opts.items():
        setattr(o, k, v)
    if o.mask_lower:
        ss.dust()                               # --qmask dust, the default (dust_all before clustering)
    res, ncl, work = vlib.cluster_fast(ctx, ss, o, threads)
    assert ncl == nclusters
    rc = ctx.revcomp(ss)
    cig = {}
    for strand, qs in ((0, ss), (1, rc)):
        hq = [k for k in range(n) if res["centroid"][k] >= 0 and res["strand"][k] == strand]
        al = ctx.align_pairs(qs, ss, np.array(hq, dtype=np.uint32), res["centroid"][hq].astype(np.uint32), cigar=True)
        cig.update(zip(hq, al.cigars))
    got = {}
    for k in range(n):
        lab = labels[order[k]]
        if res["centroid"][k] < 0:
            got[lab] = ("S", int(res["cluster"][k]), "*", "*", "*", "*")
        else:
            # '=': identical ignoring terminal gaps, matches == internal alignment length (core/results.cpp:84-90)
            internal = checkers.finish_hit(1, 1, int(res["alignment_length"][k]), int(res["matches"][k]), int(res["mismatches"][k]),
                                           int(res["gaps"][k]), checkers.trims_from_cigar(cig[k]), o.iddef)[0]
            got[lab] = ("H", int(res["cluster"][k]), f"{res['id'][k]:.1f}", "-" if res["strand"][k] else "+",
                        labels[order[int(res["centroid"][k])]], "=" if res["matches"][k] == internal else cig[k])
    assert checkers.digest(sorted(got.items())) == want
    # the data exercise the feature: many minus-strand hits, the plus-first tie rule, and (T > 1) a minus-strand hit
    # on a centroid founded earlier in the same round, which only evaluate_extra_hits of the minus strand can find
    h = res["centroid"] >= 0
    minus = h & (res["strand"] == 1)
    assert minus.sum() >= 0.2 * h.sum(), (int(minus.sum()), int(h.sum()))
    pal_sorted = [k for k in range(n) if order[k] in palindromic]
    assert any(res["centroid"][k] >= 0 and res["strand"][k] == 0 for k in pal_sorted)
    if threads > 1:
        pos = np.arange(n)
        assert np.any(minus & (res["centroid"] // threads == pos // threads))
    assert work[0] > 0 and work[1] > 0
    rc.close(); ss.close(); ctx.close()


def test_session_ranges_equal_cluster_fast_with_both_strands():
    """vsg_cluster_session_assign over ranges that do not line up with the rounds gives vsg_cluster_fast's results"""
    seqs, _ = _reads(3000, 80, seed=41)
    order = _sorted(seqs, [f"b{i:07d}" for i in range(len(seqs))])
    ctx = vlib.Context(0)
    ss = ctx.seqset(synth.SeqSet([seqs[i] for i in order]))
    ss.dust()
    o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxrejects = 8; o.strand_both = 1
    want, ncl, _ = vlib.cluster_fast(ctx, ss, o, 32)
    s = vlib.ClusterSession(ctx, ss, o)
    parts = [s.assign(start, min(257, ss.n - start), 32) for start in range(0, ss.n, 257)]
    got = np.concatenate(parts)
    assert s.clusters == ncl
    s.close()
    assert (want["strand"] == 1).sum() > 0.2 * (want["centroid"] >= 0).sum()
    assert got.tobytes() == want.tobytes()
    ss.close(); ctx.close()


def test_cluster_both_strands_defers_minus_pairs_to_the_fallback_with_strand_1(ctx):
    """with a gap penalty that does not fit a 16-bit cell every pair is deferred; the callback is told the strand, and
    answering from the default scoring's alignments (plus: the set, minus: its reverse complements) gives the default
    context's results field for field"""
    rng = np.random.default_rng(53)
    roots = synth.random_seqs(rng, 4, 200)
    seqs = []
    for i in range(72):
        s = synth.mutate(rng, roots[i % 4], 0.03).tobytes()
        seqs.append(_rc(s) if i % 3 == 1 else s)
    reads = synth.SeqSet(seqs)
    n = len(reads)
    qi, ti = (x.ravel() for x in np.meshgrid(np.arange(n), np.arange(n), indexing="ij"))
    ss = ctx.seqset(reads)
    rc = ctx.revcomp(ss)
    table = {}
    for strand, qs in ((0, ss), (1, rc)):
        al = ctx.align_pairs(qs, ss, qi, ti)
        for k in range(qi.shape[0]):
            table[(strand, int(qi[k]), int(ti[k]))] = [int(al.score[k]), int(al.aligned[k]), int(al.matches[k]),
                                                      int(al.mismatches[k]), int(al.gaps[k])] + [int(v) for v in al.trims[k]]
    rc.close(); ss.close()
    o = vlib.default_search_opts(); o.id = 0.9; o.strand_both = 1

    def run(c):
        s = c.seqset(reads)
        try:
            res, ncl, _ = vlib.cluster_fast(c, s, o, 8)
            return res.tolist(), ncl
        finally:
            s.close()

    want = run(ctx)
    pen = np.array(vlib.DEFAULT_PEN, dtype=np.int64); pen[4] = 2 ** 31 - 1
    c2 = vlib.Context(0, pen=pen)
    strands = []
    try:
        with pytest.raises(vlib.VsgError, match="linear-memory aligner"):
            run(c2)

        def fallback(q, strand, t):
            strands.append(strand)
            return table[(strand, q, t)]
        c2.set_fallback(fallback)
        got = run(c2)
    finally:
        c2.close()
    assert want[1] < n
    assert sum(1 for r in want[0] if r[1] >= 0 and r[7] == 1) > 0    # some reads joined through their reverse complement
    assert 0 in strands and 1 in strands
    assert got == want


def test_seqset_revcomp_symbols(ctx):
    """vsg_seqset_revcomp: the reverse complements' symbols are those of the host's reverse complement, case (soft mask)
    and IUPAC codes included; sub-ranges, empty ranges, and out-of-range arguments"""
    seqs = [b"ACGTacgtNRYSWKMBDHVnryswkmbdhv", b"AAAACCCGGT", b"x-X*ACg", b"", b"GATTACA", b"tttttG", b"RYKM"]
    reads = synth.SeqSet(seqs)
    ss = ctx.seqset(reads)

    def symbols(h):
        return h.symbols(int(h.lens.sum()))

    for q0, cnt in ((0, len(seqs)), (2, 4), (6, 1)):
        rc = ctx.revcomp(ss, q0, cnt)
        assert rc.n == cnt and vlib.load().vsg_seqset_count(rc.h) == cnt
        host = ctx.seqset(synth.SeqSet([_rc(s) for s in seqs[q0:q0 + cnt]]))
        assert symbols(rc).tolist() == symbols(host).tolist()
        host.close(); rc.close()
    for q0 in (0, 3, len(seqs)):
        rc = ctx.revcomp(ss, q0, 0)
        assert vlib.load().vsg_seqset_count(rc.h) == 0
        rc.close()
    for q0, cnt in ((-1, 1), (0, -1), (0, len(seqs) + 1), (len(seqs), 1), (len(seqs) + 1, 0), (3, 2 ** 62)):
        with pytest.raises(vlib.VsgError, match=r"\(-3\)"):
            ctx.revcomp(ss, q0, cnt)
    ss.close()


def test_strand_both_keeps_the_wordlength_limit(ctx):
    reads = synth.config1_allpairs(n_reads=20, n_roots=2, length=150, seed=3)
    ss = ctx.seqset(reads)
    o = vlib.default_search_opts(); o.strand_both = 1; o.wordlength = 11
    with pytest.raises(vlib.VsgError, match="wordlength 3..10"):
        vlib.cluster_fast(ctx, ss, o, 4)
    with pytest.raises(vlib.VsgError, match="wordlength 3..10"):
        vlib.ClusterSession(ctx, ss, o)
    ss.close()


# ---- the clustering shim (cluster_session_* / cluster_assign_*, src/core/cluster.hpp:78-118) with --strand both ----
# oracle/seam2_cluster_strand_driver.cpp: the key=value clustering-session driver with --strand both set, linked against
# the untouched reference (_ref) and against shim/cluster_session_vsg.cpp (_gpu) by oracle/strand.mk
needs_cluster_ref = pytest.mark.skipif(not os.path.exists(os.path.join(REF, "seam2_cluster_strand_driver_gpu")),
                                       reason="oracle/_ref (compiled reference + cluster shim) not present")


def _shim_reads(tmp_path):
    rng = np.random.default_rng(79)
    roots = synth.random_seqs(rng, 40, 320)
    recs = []
    for i in range(1500):
        m = synth.mutate(rng, roots[int(rng.integers(0, 40))], float(rng.uniform(0.0, 0.06))).tobytes()
        a, b = int(rng.integers(0, 25)), int(rng.integers(0, 25))
        s = m[a: len(m) - b]
        if i % 41 == 7:
            s = s[:100] + b"ACACACACACACACACACACACACACACACACACAC" + s[100:]   # DUST bait
        if i % 97 == 11:
            s = s[:50] + b"NRY" + s[53:]                                        # IUPAC -> the general kernel
        if rng.random() < 1.0 / 3.0:
            s = _rc(s)
        recs.append(f">r{i};size={int(rng.integers(1, 200))}\n{s.decode()}\n")
    path = str(tmp_path / "reads.fasta")
    with open(path, "w") as f:
        f.write("".join(recs))
    return path


@needs_cluster_ref
@pytest.mark.parametrize("case", [
    ["id=0.97", "threads=1", "chunk=-1"],
    ["id=0.97", "threads=8", "chunk=0"],
    ["id=0.95", "threads=32", "chunk=257", "maxrejects=16"],
    ["id=0.9", "threads=16", "chunk=700", "qmask=none", "maxaccepts=2", "iddef=1"],
    ["id=0.9", "threads=16", "chunk=300", "unoise_alpha=2.0"],
    ["id=0.9", "threads=8", "chunk=0", "maxaccepts=4", "maxrejects=16", "sizeorder=1"],
])
def test_cluster_session_shim_both_strands_equals_the_reference(tmp_path, case):
    reads = _shim_reads(tmp_path)
    outs = []
    for exe in ("seam2_cluster_strand_driver_ref", "seam2_cluster_strand_driver_gpu"):
        r = subprocess.run([os.path.join(REF, exe), reads] + case, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (exe, r.stdout[-2000:], r.stderr[-2000:])
        outs.append(r.stdout.splitlines())
    assert len(outs[0]) == 1500
    assert outs[0] == outs[1], [x for x in zip(outs[0], outs[1]) if x[0] != x[1]][:5]
    ncent = sum(1 for l in outs[0] if l.split("\t")[2] == "1")
    assert 30 <= ncent < 1500
