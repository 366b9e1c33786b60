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
