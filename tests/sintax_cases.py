"""The SINTAX parity cases shared by test_sintax_cpu.py and test_sintax_gpu.py: the synthetic taxonomy data, the option
sets (a)-(e), their FASTA / UDB files, and the reference's results, stored as digests in
tests/golden/sintax_reference.json under checkers.reference's keying (a name and a hash of the inputs)."""
from __future__ import annotations

import ctypes as C
import functools
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np

import checkers
from vsearch_b200 import synth

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "sintax_reference.json")
UDB_GZ = os.path.join(checkers.ROOT, "tests", "golden", "sintax_db.udb.gz")
SHIM = os.path.join(checkers.ORACLE_DIR, "_ref", "libvsref_sintax.so")

# name: (wordlength, dbmask lower-case excluded, strand both, cutoff, seed, database from the UDB file)
CASES = {
    "a_defaults": (8, 1, 0, 0.0, 42, False),
    "b_nomask_both_cutoff": (8, 0, 1, 0.8, 2 ** 33 + 5, False),
    "c_k12_both": (12, 1, 1, 0.0, 42, False),
    "d_udb": (8, 1, 0, 0.0, 42, True),
    "e_seed": (8, 1, 0, 0.0, 7, False),
}
PER_BOOTSTRAP = ("a_defaults", "b_nomask_both_cutoff", "c_k12_both")


@functools.lru_cache(maxsize=None)
def data():
    return synth.sintax_data()


def database():
    """the database as --sintax reads it (db.read drops records under 32 nt): (headers, sequences)"""
    d = data()
    keep = [i for i, s in enumerate(d["db_seqs"]) if len(s) >= 32]
    return [d["db_heads"][i] for i in keep], [d["db_seqs"][i] for i in keep]


def write_inputs(tmp):
    d = data()
    dbf, qf = os.path.join(tmp, "db.fa"), os.path.join(tmp, "q.fa")
    synth.write_records(dbf, d["db_heads"], d["db_seqs"])
    synth.write_records(qf, d["q_heads"], d["q_seqs"])
    return dbf, qf


def udb_path(tmp):
    """the database as the reference's --makeudb_usearch wrote it (stored gzipped under tests/golden)"""
    out = os.path.join(tmp, "db.udb")
    with gzip.open(UDB_GZ, "rb") as f, open(out, "wb") as g:
        g.write(f.read())
    return out


def cli_args(case, dbf, qf, out):
    k, mask, both, cutoff, seed, _ = CASES[case]
    a = ["--sintax", qf, "--db", dbf, "--tabbedout", out, "--threads", "1", "--quiet", "--randseed", str(seed)]
    if k != 8:
        a += ["--wordlength", str(k)]
    if mask == 0:
        a += ["--dbmask", "none"]
    if both:
        a += ["--strand", "both"]
    if cutoff > 0:
        a += ["--sintax_cutoff", repr(cutoff)]
    return a


def run_cli(case, tmp):
    dbf, qf = write_inputs(tmp)
    if CASES[case][5]:
        dbf = udb_path(tmp)
    out = os.path.join(tmp, f"{case}.tsv")
    p = subprocess.run([checkers.STOCK] + cli_args(case, dbf, qf, out), capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-2000:]
    return open(out, "rb").read()


def reference_available():
    return os.path.exists(checkers.STOCK) and os.path.exists(SHIM)


def _inputs(case):
    d = data()
    return [case, CASES[case], d["db_heads"], d["db_seqs"], d["q_heads"], d["q_seqs"]]


_stored = None


def reference(kind, case, compute):
    """the stored digest of the reference's `kind` result for `case`; VSG_RECORD_REFERENCE=1 with the compiled
    reference present recomputes it and writes it to tests/golden/sintax_reference.json"""
    global _stored
    h = hashlib.sha256()
    checkers._feed(h, _inputs(case))
    key = f"sintax_{kind}:{h.hexdigest()[:24]}"
    if os.environ.get("VSG_RECORD_REFERENCE") and reference_available():
        val = checkers.digest(compute())
        rec = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
        rec[key] = val
        with open(GOLDEN, "w") as f:
            json.dump(rec, f, indent=1, sort_keys=True)
            f.write("\n")
        _stored = rec
        return val
    if _stored is None:
        _stored = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
    assert key in _stored, f"no stored reference result {key} in {GOLDEN}"
    return _stored[key]


_shim = None


def shim():
    global _shim
    if _shim is None:
        _shim = C.CDLL(SHIM)
        _shim.vsref_sintax_db_create.restype = C.c_void_p
        _shim.vsref_sintax_db_create.argtypes = [C.c_int, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_int), C.c_int, C.c_int]
        _shim.vsref_sintax_db_free.argtypes = [C.c_void_p]
        _shim.vsref_sintax.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int64, C.c_uint64, C.c_int, C.POINTER(C.c_int32)]
    return _shim


def ref_bootstraps(case):
    """vsref_sintax for every query of the case: an (nq, 205) int32 array laid out as vsg_sintax_result"""
    k, mask, both, _, seed, _ = CASES[case]
    _, seqs = database()
    ss = synth.SeqSet(seqs)
    lens = ss.lens.astype(np.int32)
    h = shim().vsref_sintax_db_create(len(ss), ss.cat.tobytes(), ss.offs.ctypes.data_as(C.POINTER(C.c_int64)),
                                      lens.ctypes.data_as(C.POINTER(C.c_int)), k, mask)
    q = data()["q_seqs"]
    out = np.zeros((len(q), 205), dtype=np.int32)
    for i, s in enumerate(q):
        shim().vsref_sintax(h, s, len(s), i, seed, both, out[i].ctypes.data_as(C.POINTER(C.c_int32)))
    shim().vsref_sintax_db_free(h)
    return out


SHARD = 32766   # targets per static index shard


def _repeat_tail(s: bytes) -> bytes:
    """s with its last 20 nt repeated: at every k <= 20 it holds the same k-mers as itself one base shorter"""
    return s + s[-20:]


@functools.lru_cache(maxsize=None)
def three_shard_data(n: int = 70_001, seed: int = 4242):
    """A database of `n` targets, so three static index shards, the last one partial with an odd number of targets:
    random background sequences of 100-260 nt, and 20 families of 2-6 % variants of 400-nt roots spread over the whole
    database.  Planted across the shards (each pair holds the same k-mers at every k, so only length and number can
    decide between them):
      - an exact copy in shard 2 of a member in shard 1 (the shard-1 one wins: same length, lower number);
      - in shard 2, a copy one base shorter of a member in shard 0 (the shard-2 one wins: shorter);
      - one base shorter / longer pairs on either side of both shard boundaries, and the last target (the low half of
        the last counter word of the partial shard) one base shorter than a target in shard 0.
    Queries: 2 % variants of 200-nt windows of the planted members (one of each pair reverse-complemented), of members
    of the other families, random sequences and one too short for bootstraps.
    Returns dict(db_seqs, q_seqs, meta) with meta["never"]: targets that can never win a bootstrap, meta["wins"]:
    their partners."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(100, 261, size=n)
    m = synth.random_seqs(rng, n, 260)
    seqs = [m[i, :lens[i]].tobytes() for i in range(n)]
    roots = synth.random_seqs(rng, 20, 400)
    fam = {}
    for f in range(20):
        idx = rng.choice(n, size=30, replace=False)
        fam[f] = idx
        for i in idx:
            seqs[i] = synth.mutate(rng, roots[f], float(rng.uniform(0.02, 0.06))).tobytes()
    last = n - 1
    planted = {}   # family: (winner, loser, sequence of the winner, sequence of the loser)

    def member(f):
        return _repeat_tail(synth.mutate(rng, roots[f], 0.02).tobytes())

    x = synth.mutate(rng, roots[1], 0.02).tobytes()
    planted[1] = (40_000, 68_000, x, x)                          # exact copies in shards 1 and 2
    y = member(2)
    planted[2] = (69_000, 5_000, y[:-1], y)                      # shorter copy in shard 2 of a shard-0 member
    w = member(3)
    planted[3] = (SHARD, SHARD - 1, w[:-1], w)                   # across the 0 | 1 boundary: the higher number is shorter
    v = member(4)
    planted[4] = (2 * SHARD - 1, 2 * SHARD, v[:-1], v)           # across the 1 | 2 boundary: the lower number is shorter
    u = member(5)
    planted[5] = (last, 100, u[:-1], u)                          # the last target against a shard-0 one
    for f, (win, lose, sw, sl) in planted.items():
        seqs[win], seqs[lose] = sw, sl
    queries = []
    for f, (win, lose, sw, _) in planted.items():
        for j in range(2):
            p = int(rng.integers(0, len(sw) - 240))
            qv = synth.mutate(rng, np.frombuffer(sw[p:p + 200], dtype=np.uint8), 0.02).tobytes()
            queries.append(synth.revcomp(qv) if j else qv)
    for f in range(6, 20):
        s = seqs[int(fam[f][int(rng.integers(0, 30))])]
        p = int(rng.integers(0, len(s) - 200))
        queries.append(synth.mutate(rng, np.frombuffer(s[p:p + 200], dtype=np.uint8), 0.02).tobytes())
    queries += [r.tobytes() for r in synth.random_seqs(rng, 3, 200)] + [b"ACGTTGCAACGTAGGC"]
    meta = {"never": [p[1] for p in planted.values()], "wins": [p[0] for p in planted.values()]}
    return {"db_seqs": seqs, "q_seqs": queries, "meta": meta}


def as_array(res):
    """Context.sintax's dict -> the (nq, 205) layout of ref_bootstraps"""
    n = res["strand"].shape[0]
    return np.concatenate([res["strand"].reshape(n, 1), res["nboot"], res["best_count"], res["seqno"].reshape(n, 200)],
                          axis=1).astype(np.int32)


def to_results(arr):
    """the (nq, 205) layout -> a lib.SINTAX_DT array for vsg_sintax_rows"""
    from vsearch_b200 import lib
    r = np.zeros(arr.shape[0], dtype=lib.SINTAX_DT)
    r["strand"] = arr[:, 0]
    r["nboot"] = arr[:, 1:3]
    r["best_count"] = arr[:, 3:5]
    r["seqno"] = arr[:, 5:].reshape(-1, 2, 100)
    return r
