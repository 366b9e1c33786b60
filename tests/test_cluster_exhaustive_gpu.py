"""Greedy clustering with limits above the ranker's 1 024 shared-memory slots: --maxaccepts 0 --maxrejects 0 (every
centroid is a candidate) and any maxaccepts + maxrejects + 8 > 1024 on a set of more than 1 024 sequences.  Each round's
strands are ranked into back-to-back lists of any length, and a strand whose remaining list can reach neither limit is
aligned whole in one device call.  vsg_cluster_fast must give `vsearch --cluster_fast --threads T --uc`'s records, the
cluster sessions vsg_cluster_fast's results, and the clustering shim the reference library's records.  The reference
CLI's records are stored as digests in tests/golden/cluster_exhaustive_reference.json (see _reference)."""
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
RESULTS = os.path.join(ROOT, "tests", "golden", "cluster_exhaustive_reference.json")
SLOTS = 1024        # candidates per query the shared-memory ranker holds


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
        with open(out, "w") as f:      # one record per line
            f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(rec[k], separators=(",", ":"))
                                        for k in sorted(rec)) + "\n}\n")
        return val
    stored = json.load(open(RESULTS))
    if key not in stored:
        raise AssertionError(f"no stored reference result {key} in {RESULTS}")
    return stored[key]


_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def _rc(s: bytes) -> bytes:
    return s.translate(_COMP)[::-1]


def _reads(n, nroots, seed, divs, rc_share=0.0):
    """n 300-nt reads spread evenly over nroots random roots, each at a divergence drawn from divs and trimmed by up to
    five bases at each end.  Reads 3-5 % away from their root are 6-10 % apart from each other, so nearly every one of
    them founds a cluster, and all of a root's clusters share enough 8-mers with its later reads to be candidates."""
    rng = np.random.default_rng(seed)
    roots = synth.random_seqs(rng, nroots, 300)
    seqs = []
    for i in range(n):
        m = synth.mutate(rng, roots[i % nroots], float(divs[int(rng.integers(0, len(divs)))]))
        a = int(rng.integers(0, 6)); b = int(rng.integers(0, 6))
        s = m[a: m.shape[0] - b].tobytes()
        if rng.random() < rc_share:
            s = _rc(s)
        seqs.append(s)
    sizes = [int(x) for x in rng.integers(1, 200, size=n)]
    return seqs, sizes


def _uc_records(text):
    """S/H records of a .uc file by label (any ;size= annotation dropped): type, cluster, identity, strand, centroid,
    CIGAR"""
    rec = {}
    for line in text.decode().splitlines(True):
        f = line.rstrip("\n").split("\t")
        if f[0] == "S":
            rec[f[8].split(";")[0]] = ("S", int(f[1]), "*", "*", "*", "*")
        elif f[0] == "H":
            rec[f[8].split(";")[0]] = ("H", int(f[1]), f[3], f[4], f[9].split(";")[0], f[7])
    return rec


def _records(ctx, ss, res, order, labels, iddef, strand_both):
    """vsg_cluster_fast's results as _uc_records' records, CIGARs from the aligner"""
    n = ss.n
    quer = [(0, ss)]
    rc = None
    if strand_both:
        rc = ctx.revcomp(ss)
        quer.append((1, rc))
    cig = {}
    for strand, qs in quer:
        hq = [k for k in range(n) if res["centroid"][k] >= 0 and res["strand"][k] == strand]
        if hq:
            al = ctx.align_pairs(qs, ss, np.array(hq, dtype=np.uint32), res["centroid"][hq].astype(np.uint32), cigar=True)
            cig.update(zip(hq, al.cigars))
    if rc is not None:
        rc.close()
    got = {}
    for k in range(n):
        lab = labels[order[k]]
        if res["centroid"][k] < 0:
            got[lab] = ("S", int(res["cluster"][k]), "*", "*", "*", "*")
        else:
            # '=': identical ignoring terminal gaps, matches == internal alignment length (core/results.cpp:84-90)
            internal = checkers.finish_hit(1, 1, int(res["alignment_length"][k]), int(res["matches"][k]), int(res["mismatches"][k]),
                                           int(res["gaps"][k]), checkers.trims_from_cigar(cig[k]), iddef)[0]
            got[lab] = ("H", int(res["cluster"][k]), f"{res['id'][k]:.1f}", "-" if res["strand"][k] else "+",
                        labels[order[int(res["centroid"][k])]], "=" if res["matches"][k] == internal else cig[k])
    return got


def _kmers(s: bytes, k=8):
    """the distinct k-mers of an A/C/G/T sequence (unique_count with nothing masked)"""
    code = np.frombuffer(s, dtype=np.uint8)
    v = np.select([code == ord("C"), code == ord("G"), code == ord("T")], [1, 2, 3], 0).astype(np.int64)
    w = np.zeros(len(s) - k + 1, dtype=np.int64)
    for j in range(k):
        w = (w << 2) | v[j: j + len(w)]
    return np.unique(w)


# (extra CLI arguments, option fields, the reads' generator arguments and reverse-complemented share)
CASES = {
    "exhaustive": (["--maxaccepts", "0", "--maxrejects", "0"], {"maxaccepts": 0, "maxrejects": 0}, 0.0),
    "strand_both": (["--maxaccepts", "0", "--maxrejects", "0", "--strand", "both"],
                    {"maxaccepts": 0, "maxrejects": 0, "strand_both": 1}, 1.0 / 3.0),
    "qmask_none": (["--maxaccepts", "0", "--maxrejects", "0", "--qmask", "none"],
                   {"maxaccepts": 0, "maxrejects": 0, "mask_lower": 0}, 0.0),
    # the limits can be reached: groups of eight
    "limits": (["--maxaccepts", "4", "--maxrejects", "2000"], {"maxaccepts": 4, "maxrejects": 2000}, 0.0),
    "sizeorder": (["--maxaccepts", "0", "--maxrejects", "0", "--sizein", "--sizeorder"],
                  {"maxaccepts": 0, "maxrejects": 0, "sizeorder": 1}, 0.0),
}


def _data(threads, rc_share):
    """--threads 1: 1 500 reads from one root at --id 0.97; rounds of several: 4 000 reads from two roots at --id 0.99,
    a quarter of them close to their root, so that some queries have several acceptable centroids"""
    if threads == 1:
        return _reads(1500, 1, seed=11, divs=(0.03, 0.04, 0.05), rc_share=rc_share) + (0.97,)
    return _reads(4000, 2, seed=12, divs=(0.005, 0.03, 0.04, 0.05), rc_share=rc_share) + (0.99,)


@pytest.mark.parametrize("threads,case", [(1, "exhaustive"), (8, "exhaustive"), (64, "exhaustive"),
                                          (1, "strand_both"), (8, "strand_both"), (64, "strand_both"),
                                          (1, "qmask_none"), (8, "qmask_none"), (64, "qmask_none"),
                                          (8, "limits"), (8, "sizeorder")])
def test_cluster_fast_without_limits_equals_reference_cli(tmp_path, threads, case):
    extra, fields, rc_share = CASES[case]
    seqs, sizes, ident = _data(threads, rc_share)
    n = len(seqs)
    sized = case == "sizeorder"
    labels = [f"c{i:07d}" for i in range(n)]
    fa = str(tmp_path / "reads.fasta")
    with open(fa, "wb") as f:
        for l, s, z in zip(labels, seqs, sizes):
            f.write(b">" + l.encode() + (f";size={z}".encode() if sized else b"") + b"\n" + s + b"\n")
    uc = str(tmp_path / "ref.uc")

    def reduce(text):
        rec = _uc_records(text)
        return sum(1 for v in rec.values() if v[0] == "S"), checkers.digest(sorted(rec.items()))
    args = ["--id", str(ident)] + extra
    nclusters, want = _reference(
        "cluster_fast_exhaustive", (seqs, labels, sizes if sized else None, args, threads),
        lambda: checkers.run_stock(["--cluster_fast", fa] + args + ["--threads", str(threads), "--uc", uc, "--quiet"], [uc], reduce),
        os.path.exists(STOCK))
    # Database::sortbylength (core/db.cpp:433-449): length descending, abundance descending (--sizein), label ascending
    order = sorted(range(n), key=lambda i: (-len(seqs[i]), -sizes[i] if sized else 0, labels[i]))
    ctx = vlib.Context(0)
    ss = ctx.seqset(synth.SeqSet([seqs[i] for i in order]))
    o = vlib.default_search_opts(); o.id = ident; o.mask_lower = 1; o.maxrejects = 8
    for k, v in fields.items():
        setattr(o, k, v)
    tsz = np.array([sizes[i] for i in order], dtype=np.int64)
    if sized:
        o.target_sizes = tsz.ctypes.data_as(vlib.C.POINTER(vlib.C.c_int64))
    if o.mask_lower:
        ss.dust()                               # --qmask dust, the default (dust_all before clustering)
    res, ncl, work = vlib.cluster_fast(ctx, ss, o, threads)
    assert ncl == nclusters
    got = _records(ctx, ss, res, order, labels, o.iddef, o.strand_both)
    assert checkers.digest(sorted(got.items())) == want
    # the data exercise the unbounded lists: more than 1 024 centroids, nearly all of them candidates of later reads
    assert ncl > SLOTS, ncl
    if case == "qmask_none":
        # counted on the host: the last sequence's candidates are the clusters founded before its round that share at
        # least min(minwordmatches, its distinct k-mers) 8-mers with it
        last = n - 1
        qk = _kmers(bytes(seqs[order[last]]))
        cents = [k for k in range(last - last % threads) if res["centroid"][k] < 0]
        cand = sum(1 for k in cents if np.intersect1d(qk, _kmers(bytes(seqs[order[k]])), assume_unique=True).size >= min(12, qk.size))
        assert cand > SLOTS, cand
    if case == "sizeorder":
        assert (res["centroid"] >= 0).sum() > 100
    if case == "strand_both" and threads > 1:
        assert (res["strand"][res["centroid"] >= 0] == 1).sum() > 0     # some reads join through their reverse complement
    assert work[0] > 0 and work[1] > 0
    ss.close(); ctx.close()


def _cluster(ctx, reads, opts, round_size, dust=True):
    ss = ctx.seqset(reads)
    if dust:
        ss.dust()
    try:
        return vlib.cluster_fast(ctx, ss, opts, round_size)
    finally:
        ss.close()


def test_cap_equivalence_of_the_two_rankers():
    """lists shorter than both limits: (500, 508) ranks in shared memory (tophits 1 016), (500, 600) through the unbounded
    lists (tophits 1 108).  Every decision, every result field and the work are the same."""
    seqs, _ = _reads(3000, 40, seed=21, divs=(0.005, 0.01, 0.015))
    reads = synth.SeqSet(seqs)
    ctx = vlib.Context(0)
    out = []
    for ma, mr in ((500, 508), (500, 600)):
        o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxaccepts = ma; o.maxrejects = mr
        for round_size in (1, 16):
            res, ncl, work = _cluster(ctx, reads, o, round_size)
            out.append((round_size, res.tobytes(), ncl, work.tolist()))
    ctx.close()
    assert out[0] == out[2] and out[1] == out[3]
    ncl = out[0][2]
    assert 40 <= ncl < 500, ncl          # every list is shorter than both limits
    assert len(seqs) > 1108


def _exhaustive_opts():
    o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxaccepts = 0; o.maxrejects = 0
    return o


def test_session_ranges_equal_cluster_fast_without_limits():
    """vsg_cluster_session_assign over ranges that do not line up with the rounds gives vsg_cluster_fast's results"""
    seqs, _ = _reads(2000, 1, seed=31, divs=(0.03, 0.04, 0.05))
    ctx = vlib.Context(0)
    ss = ctx.seqset(synth.SeqSet(seqs))
    ss.dust()
    o = _exhaustive_opts()
    want, ncl, _ = vlib.cluster_fast(ctx, ss, o, 32)
    s = vlib.ClusterSession(ctx, ss, o)
    got = np.concatenate([s.assign(start, min(257, ss.n - start), 32) for start in range(0, ss.n, 257)])
    assert s.clusters == ncl
    s.close()
    assert ncl > SLOTS
    assert got.tobytes() == want.tobytes()
    ss.close(); ctx.close()


def test_ranker_in_chunks_equals_one_chunk():
    """a device key budget far below a round's candidates (VSG_DIR_BUDGET_MB=1: about 10 900 keys per chunk): every
    round's lists are ranked in several query ranges, with the same results"""
    seqs, _ = _reads(2000, 1, seed=37, divs=(0.03, 0.04, 0.05))
    reads = synth.SeqSet(seqs)
    o = _exhaustive_opts()
    ctx = vlib.Context(0)
    want = _cluster(ctx, reads, o, 64)
    ctx.close()
    old = os.environ.get("VSG_DIR_BUDGET_MB")
    os.environ["VSG_DIR_BUDGET_MB"] = "1"
    try:
        small = vlib.Context(0)
    finally:
        if old is None:
            del os.environ["VSG_DIR_BUDGET_MB"]
        else:
            os.environ["VSG_DIR_BUDGET_MB"] = old
    got = _cluster(small, reads, o, 64)
    small.close()
    assert want[1] > SLOTS
    assert got[0].tobytes() == want[0].tobytes() and got[1] == want[1] and got[2].tolist() == want[2].tolist()


# ---- the clustering shim (cluster_session_* / cluster_assign_*, src/core/cluster.hpp:78-118) with large limits --------
# oracle/seam2_cluster_driver.cpp and seam2_cluster_strand_driver.cpp linked against the untouched reference (_ref) and
# against shim/cluster_session_vsg.cpp (_gpu)
@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "seam2_cluster_strand_driver_gpu")),
                    reason="oracle/_ref (compiled reference + cluster shim) not present")
@pytest.mark.parametrize("driver", ["seam2_cluster_driver", "seam2_cluster_strand_driver"])
@pytest.mark.parametrize("case", [
    ["id=0.99", "threads=8", "chunk=0", "maxaccepts=1500", "maxrejects=3000"],
    ["id=0.99", "threads=16", "chunk=300", "maxaccepts=1500", "maxrejects=3000", "sizeorder=1"],
])
def test_cluster_session_shim_with_large_limits_equals_the_reference(tmp_path, driver, case):
    seqs, sizes = _reads(2000, 1, seed=43, divs=(0.005, 0.03, 0.04, 0.05), rc_share=0.25)
    path = str(tmp_path / "reads.fasta")
    with open(path, "wb") as f:
        for i, (s, z) in enumerate(zip(seqs, sizes)):
            f.write(f">r{i};size={z}\n".encode() + s + b"\n")
    outs = []
    for exe in (driver + "_ref", driver + "_gpu"):
        r = subprocess.run([os.path.join(REF, exe), path] + case, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, (exe, r.stdout[-2000:], r.stderr[-2000:])
        outs.append(r.stdout.splitlines())
    assert len(outs[0]) == 2000
    assert outs[0] == outs[1], [x for x in zip(outs[0], outs[1]) if x[0] != x[1]][:5]
    ncent = sum(1 for l in outs[0] if l.split("\t")[2] == "1")
    assert SLOTS < ncent < 2000, ncent
