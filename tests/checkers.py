"""ctypes loaders for the CHECKERS (oracle/liboracle.so and oracle/_ref/libvsref.so).

Test infrastructure only — the product never imports this module.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
STOCK = os.path.join(ORACLE_DIR, "_ref", "vsearch")
REFERENCE_RESULTS = os.path.join(ROOT, "tests", "golden", "reference_results.json")


def _feed(h, obj):
    """hash an input structurally: raw bytes for byte strings and arrays, a tag and a length before each item"""
    if hasattr(obj, "cat") and hasattr(obj, "lens"):        # synth.SeqSet
        obj = ("seqset", obj.cat, obj.offs, obj.lens)
    if isinstance(obj, (bytes, bytearray)):
        h.update(b"b%d:" % len(obj)); h.update(bytes(obj))
    elif isinstance(obj, np.ndarray):
        a = np.ascontiguousarray(obj)
        h.update(b"a%s%r:" % (a.dtype.str.encode(), a.shape)); h.update(a.tobytes())
    elif isinstance(obj, (list, tuple)):
        h.update(b"l%d:" % len(obj))
        for x in obj:
            _feed(h, x)
    elif isinstance(obj, dict):
        _feed(h, sorted(obj.items()))
    else:
        h.update(b"s" + repr(canon(obj)).encode() + b";")


def canon(obj):
    """plain JSON-able Python values (tuples as lists, numpy scalars and arrays as Python numbers and lists)"""
    if isinstance(obj, (list, tuple)):
        return [canon(x) for x in obj]
    if isinstance(obj, dict):
        return {str(k): canon(v) for k, v in obj.items()}
    if isinstance(obj, np.ndarray):
        return canon(obj.tolist())
    if isinstance(obj, np.generic):
        return obj.item()
    if isinstance(obj, (bytes, bytearray)):
        return bytes(obj).decode("latin-1")
    return obj


def digest(obj) -> str:
    """sha256 of a result's canonical JSON: large reference results are stored as this digest"""
    return hashlib.sha256(json.dumps(canon(obj), separators=(",", ":")).encode()).hexdigest()


_results = None


def reference(name, inputs, compute, available):
    """What the unmodified reference returned for `inputs`, from tests/golden/reference_results.json.

    The record is keyed by `name` and a hash of the inputs, so a test whose inputs change no longer finds one and
    fails instead of comparing against a stale result.  With the compiled reference present (`available`) and
    VSG_RECORD_REFERENCE=<file>, `compute()` runs it and its canonical result is added to <file>; copying that file
    to tests/golden/reference_results.json makes the record the tests use."""
    global _results
    h = hashlib.sha256()
    _feed(h, inputs)
    key = f"{name}:{h.hexdigest()[:24]}"
    out = os.environ.get("VSG_RECORD_REFERENCE")
    if out and available:
        val = canon(compute())
        rec = json.load(open(out)) if os.path.exists(out) else {}
        rec[key] = val
        with open(out, "w") as f:      # one record per line
            f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(rec[k], separators=(",", ":"))
                                        for k in sorted(rec)) + "\n}\n")
        return val
    if _results is None:
        _results = json.load(open(REFERENCE_RESULTS)) if os.path.exists(REFERENCE_RESULTS) else {}
    if key not in _results:
        raise AssertionError(f"no stored reference result {key} in {REFERENCE_RESULTS}")
    return _results[key]


def ref_search(dbs, qss, filters=None, **kw):
    """the reference's rows for every query (RefDb.search with max_results = tophits) and its tophits"""
    r = RefDb(dbs, **kw)
    if filters is not None:
        ref().vsref_db_set_filters(C.c_void_p(r.h), (C.c_double * 14)(*filters))
    want = r.search(qss, max_results=r.tophits)
    th = r.tophits
    r.close()
    return want, th


def run_stock(args, outputs, reduce):
    """run the reference CLI and return reduce(contents of each output file, in order)"""
    p = subprocess.run([STOCK] + args, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-2000:]
    return reduce(*[open(o, "rb").read() for o in outputs])


DEFAULT_PEN = np.array([2, -4, 1, 1, 18, 18, 1, 1, 1, 1, 2, 2, 1, 1], dtype=np.int64)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Scoring(C.Structure):
    _fields_ = [("v", C.c_int64 * 14), ("n_mismatch", C.c_int)]


def make_scoring(pen=None, n_mismatch=0):
    s = Scoring()
    pen = DEFAULT_PEN if pen is None else pen
    for i in range(14):
        s.v[i] = int(pen[i])
    s.n_mismatch = int(n_mismatch)
    return s


_oracle = None


def oracle():
    global _oracle
    if _oracle is None:
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-C", ORACLE_DIR, "oracle"], stdout=subprocess.DEVNULL)
        _oracle = C.CDLL(path)
        _oracle.oracle_unique_kmers.restype = C.c_uint
        _oracle.oracle_index_build.restype = C.c_void_p
        _oracle.oracle_map_4bit.restype = C.c_ubyte
    return _oracle


_ref = None


def ref():
    """The unmodified reference behind a C ABI, or None when oracle/_ref was not built."""
    global _ref
    if _ref is None:
        path = os.path.join(ORACLE_DIR, "_ref", "libvsref.so")
        if not os.path.exists(path):
            return None
        _ref = C.CDLL(path)
        _ref.vsref_db_create.restype = C.c_void_p
    return _ref


def oracle_nw16(q: bytes, d: bytes, pen=None, n_mismatch=0):
    lib = oracle()
    sc = make_scoring(pen, n_mismatch)
    score = C.c_int16(); al = C.c_uint16(); ma = C.c_uint16(); mi = C.c_uint16(); ga = C.c_uint16()
    cap = len(q) + len(d) + 64
    buf = C.create_string_buffer(cap)
    rc = lib.oracle_nw16(C.byref(sc), q, C.c_int64(len(q)), d, C.c_int64(len(d)),
                         C.byref(score), C.byref(al), C.byref(ma), C.byref(mi), C.byref(ga),
                         buf, C.c_size_t(cap))
    assert rc == 0
    return score.value, al.value, ma.value, mi.value, ga.value, buf.value.decode()


def ref_search16(q: bytes, targets, pen=None, n_mismatch=0):
    lib = ref()
    pen = np.ascontiguousarray(DEFAULT_PEN if pen is None else pen, dtype=np.int64)
    n = len(targets)
    lens = np.array([len(t) for t in targets], dtype=np.int32)
    offs = np.zeros(n, dtype=np.int64)
    if n:
        np.cumsum(lens[:-1], out=offs[1:])
    cat = b"".join(targets) + b"\0"
    scores = np.zeros(n, dtype=np.int16)
    al = np.zeros(n, dtype=np.uint16); ma = np.zeros(n, dtype=np.uint16)
    mi = np.zeros(n, dtype=np.uint16); ga = np.zeros(n, dtype=np.uint16)
    stride = len(q) + (int(lens.max()) if n else 0) + 64
    cig = C.create_string_buffer(stride * max(n, 1))
    rc = lib.vsref_search16(_p(pen, C.c_int64), C.c_int(n_mismatch), q, C.c_int(len(q)),
                            C.c_int(n), cat, _p(offs, C.c_int64), _p(lens, C.c_int),
                            _p(scores, C.c_int16), _p(al, C.c_uint16), _p(ma, C.c_uint16),
                            _p(mi, C.c_uint16), _p(ga, C.c_uint16), cig, C.c_int64(stride))
    assert rc == 0
    out = []
    raw = cig.raw
    for i in range(n):
        c = raw[i * stride:(i + 1) * stride].split(b"\0", 1)[0].decode()
        out.append((int(scores[i]), int(al[i]), int(ma[i]), int(mi[i]), int(ga[i]), c))
    return out


def oracle_unique_kmers(seq: bytes, k=8, mask_lower=0):
    out = np.zeros(max(len(seq), 1), dtype=np.uint32)
    n = oracle().oracle_unique_kmers(C.c_int(k), seq, C.c_int64(len(seq)), C.c_int(mask_lower),
                                     _p(out, C.c_uint32))
    return out[:n].copy()


def ref_unique_kmers(seq: bytes, k=8, mask_lower=0):
    out = np.zeros(max(len(seq), 1), dtype=np.uint32)
    n = ref().vsref_unique_count(C.c_int(k), seq, C.c_int(len(seq)), C.c_int(mask_lower),
                                 _p(out, C.c_uint32), C.c_int(out.shape[0]))
    return out[:n].copy()


class OracleHit(C.Structure):
    _fields_ = [("target", C.c_int), ("strand", C.c_int), ("count", C.c_uint),
                ("accepted", C.c_int), ("rejected", C.c_int), ("aligned", C.c_int), ("weak", C.c_int),
                ("nwscore", C.c_int), ("nwdiff", C.c_int), ("nwgaps", C.c_int), ("nwindels", C.c_int),
                ("nwalignmentlength", C.c_int), ("matches", C.c_int), ("mismatches", C.c_int),
                ("internal_alignmentlength", C.c_int), ("internal_gaps", C.c_int),
                ("internal_indels", C.c_int),
                ("trim_q_left", C.c_int), ("trim_q_right", C.c_int), ("trim_t_left", C.c_int),
                ("trim_t_right", C.c_int),
                ("id", C.c_double), ("id0", C.c_double), ("id1", C.c_double), ("id2", C.c_double),
                ("id3", C.c_double), ("id4", C.c_double), ("shortest", C.c_int), ("longest", C.c_int)]


class SearchOpts(C.Structure):
    _fields_ = [("id", C.c_double), ("weak_id", C.c_double), ("maxaccepts", C.c_int),
                ("maxrejects", C.c_int), ("minwordmatches", C.c_int), ("tophits", C.c_int),
                ("iddef", C.c_int), ("mask_lower", C.c_int)]


MINWORDMATCHES = [-1, -1, -1, 18, 17, 16, 15, 14, 12, 11, 10, 9, 8, 7, 5, 3]


def search_opts(n_db, id=0.9, maxaccepts=1, maxrejects=32, k=8, minwordmatches=-1, iddef=2,
                weak_id=10.0, mask_lower=0):
    """Effective options after the reference's fix-ups (vsearch.cc:186-276,
    usearch_global.cpp:598-614)."""
    o = SearchOpts()
    o.id = id
    o.weak_id = min(weak_id, id)
    o.maxaccepts = min(maxaccepts, n_db)
    o.maxrejects = min(maxrejects, n_db)
    o.minwordmatches = MINWORDMATCHES[k] if minwordmatches < 0 else minwordmatches
    o.tophits = min(o.maxaccepts + o.maxrejects + 8, n_db)
    o.iddef = iddef
    o.mask_lower = mask_lower
    return o


class OracleDb:
    def __init__(self, ss, k=8, mask_lower=0):
        self.ss = ss
        self.k = k
        self.mask_lower = mask_lower
        self.h = oracle().oracle_index_build(C.c_int(k), C.c_int(len(ss)), _p(ss.cat, C.c_char),
                                             _p(ss.offs, C.c_int64), _p(ss.lens, C.c_int),
                                             C.c_int(mask_lower))

    def close(self):
        if self.h:
            oracle().oracle_index_free(C.c_void_p(self.h))
            self.h = None

    def topscores(self, q: bytes, opts):
        kmers = oracle_unique_kmers(q, self.k, opts.mask_lower)
        seqno = np.zeros(opts.tophits + 1, dtype=np.uint32)
        count = np.zeros(opts.tophits + 1, dtype=np.uint32)
        n = oracle().oracle_topscores(C.c_void_p(self.h), _p(self.ss.lens, C.c_int),
                                      _p(kmers, C.c_uint32), C.c_uint(kmers.shape[0]),
                                      C.c_int(opts.minwordmatches), C.c_int(opts.tophits),
                                      _p(seqno, C.c_uint32), _p(count, C.c_uint32))
        return seqno[:n].copy(), count[:n].copy()

    def search(self, q: bytes, opts, pen=None, strand=0):
        sc = make_scoring(pen)
        hits = (OracleHit * (opts.tophits + 1))()
        pairs = C.c_int64(); cells = C.c_int64()
        n = oracle().oracle_search_onequery(C.c_void_p(self.h), C.byref(sc), C.byref(opts),
                                            C.c_int(len(self.ss)), _p(self.ss.cat, C.c_char),
                                            _p(self.ss.offs, C.c_int64), _p(self.ss.lens, C.c_int),
                                            q, C.c_int(len(q)), C.c_int(strand),
                                            hits, C.c_int(opts.tophits + 1),
                                            C.byref(pairs), C.byref(cells))
        return [hits[i] for i in range(n)], pairs.value, cells.value

    def sintax(self, q: bytes, query_number: int, seed: int, strand_both: int = 0, trace: bool = False):
        """oracle_sintax: the bootstraps of one query as a 205-int row laid out as vsg_sintax_result; with trace, also
        every bootstrap (SintaxBoot * 200, strand s at [100 * s + b])"""
        out = np.zeros(205, dtype=np.int32)
        tr = (SintaxBoot * 200)() if trace else None
        oracle().oracle_sintax_trace(C.c_void_p(self.h), _p(self.ss.lens, C.c_int), q, C.c_int(len(q)),
                                     C.c_uint64(query_number), C.c_uint64(seed), C.c_int(strand_both),
                                     _p(out, C.c_int32), tr)
        return (out, tr) if trace else out


class SintaxBoot(C.Structure):
    _fields_ = [("winner", C.c_int32), ("count", C.c_int32), ("ntied", C.c_int32), ("tied_lo", C.c_int32),
                ("tied_hi", C.c_int32), ("nsamp", C.c_int32), ("samp", C.c_uint32 * 32)]


class RefDb:
    """Reference Database+Dbindex+session (one at a time per process)."""

    def __init__(self, ss, k=8, id=0.9, maxaccepts=1, maxrejects=32, minwordmatches=-1,
                 dust=0, strand_both=0, iddef=2):
        self.ss = ss
        self.h = ref().vsref_db_create(C.c_int(len(ss)), _p(ss.cat, C.c_char),
                                       _p(ss.offs, C.c_int64), _p(ss.lens, C.c_int),
                                       C.c_int(k), C.c_double(id), C.c_int(maxaccepts),
                                       C.c_int(maxrejects), C.c_int(minwordmatches), C.c_int(dust),
                                       C.c_int(strand_both), C.c_int(iddef))
        self.tophits = ref().vsref_db_tophits(C.c_void_p(self.h))

    def close(self):
        if self.h:
            ref().vsref_db_free(C.c_void_p(self.h))
            self.h = None

    def topscores(self, q: bytes):
        seqno = np.zeros(self.tophits + 1, dtype=np.uint32)
        count = np.zeros(self.tophits + 1, dtype=np.uint32)
        length = np.zeros(self.tophits + 1, dtype=np.uint32)
        n = ref().vsref_db_topscores(C.c_void_p(self.h), q, C.c_int(len(q)),
                                     _p(seqno, C.c_uint32), _p(count, C.c_uint32),
                                     _p(length, C.c_uint32))
        return seqno[:n].copy(), count[:n].copy()

    def search_rows(self, qs, max_results=8, threads=None):
        """the reference's own multi-threaded search_batch, every record kept: (counts, dict of flat arrays)"""
        nq = len(qs)
        threads = threads or (os.cpu_count() or 1)
        counts = np.zeros(nq, dtype=np.int32)
        m = nq * max_results
        a = {k: np.zeros(m, dtype=np.int32) for k in ("target", "matches", "mismatches", "gaps", "alnlen", "accepted", "strand")}
        a["id"] = np.zeros(m, dtype=np.float64)
        ref().vsref_db_search_batch_rows(C.c_void_p(self.h), C.c_int(nq), _p(qs.cat, C.c_char), _p(qs.offs, C.c_int64),
                                         _p(qs.lens, C.c_int), C.c_int(threads), C.c_int(max_results), _p(counts, C.c_int),
                                         _p(a["target"], C.c_int), _p(a["id"], C.c_double), _p(a["matches"], C.c_int),
                                         _p(a["mismatches"], C.c_int), _p(a["gaps"], C.c_int), _p(a["alnlen"], C.c_int),
                                         _p(a["accepted"], C.c_int), _p(a["strand"], C.c_int))
        return counts, a

    def search(self, qs, max_results=8):
        nq = len(qs)
        counts = np.zeros(nq, dtype=np.int32)
        m = nq * max_results
        target = np.zeros(m, dtype=np.int32); idv = np.zeros(m, dtype=np.float64)
        ma = np.zeros(m, dtype=np.int32); mi = np.zeros(m, dtype=np.int32)
        ga = np.zeros(m, dtype=np.int32); al = np.zeros(m, dtype=np.int32)
        acc = np.zeros(m, dtype=np.int32); st = np.zeros(m, dtype=np.int32)
        ref().vsref_db_search(C.c_void_p(self.h), C.c_int(nq), _p(qs.cat, C.c_char),
                              _p(qs.offs, C.c_int64), _p(qs.lens, C.c_int), C.c_int(max_results),
                              _p(counts, C.c_int), _p(target, C.c_int), _p(idv, C.c_double),
                              _p(ma, C.c_int), _p(mi, C.c_int), _p(ga, C.c_int), _p(al, C.c_int),
                              _p(acc, C.c_int), _p(st, C.c_int))
        out = []
        for q in range(nq):
            rows = []
            for j in range(counts[q]):
                o = q * max_results + j
                rows.append((int(target[o]), float(idv[o]), int(ma[o]), int(mi[o]), int(ga[o]),
                             int(al[o]), int(acc[o]), int(st[o])))
            out.append(rows)
        return out


def trims_from_cigar(c):
    """(trim_q_left, trim_t_left, trim_q_right, trim_t_right): run length of a leading / trailing D resp. I"""
    ops = re.findall(r"(\d*)([MID])", c)
    if not ops:
        return (0, 0, 0, 0)
    f, l = ops[0], ops[-1]
    fr = int(f[0]) if f[0] else 1
    lr = int(l[0]) if l[0] else 1
    return (fr if f[1] == "D" else 0, fr if f[1] == "I" else 0,
            lr if l[1] == "D" else 0, lr if l[1] == "I" else 0)


def finish_hit(qlen, tlen, aligned, matches, mismatches, gaps, trims, iddef):
    """align_trim and the identity definitions (searchcore.cpp:409-463) in float64, the host's finish_hit restated:
    (internal_alignment_length, internal_gaps, id under iddef)"""
    tql, ttl, tqr, ttr = trims
    if tql >= aligned:
        tqr = 0
    if ttl >= aligned:
        ttr = 0
    internal = aligned - (tql + ttl + tqr + ttr)
    internal_gaps = gaps - (1 if tql + ttl > 0 else 0) - (1 if tqr + ttr > 0 else 0)
    shortest, longest = min(qlen, tlen), max(qlen, tlen)
    if iddef == 0:
        ident = 100.0 * matches / shortest if shortest > 0 else 0.0
    elif iddef == 2:
        ident = 100.0 * matches / internal if internal > 0 else 0.0
    elif iddef == 3:
        ident = max(0.0, 100.0 * (1.0 - (1.0 * (mismatches + gaps) / longest)))
    else:                                                     # 1 and 4
        ident = 100.0 * matches / aligned if aligned > 0 else 0.0
    return internal, internal_gaps, ident


def leader_accepted(qlen, tlen, aligned, matches, mismatches, gaps, trims, iddef, threshold):
    """the device's verdict on a group leader (align_ckpt.cuh tb_leader_accepted) restated: the identity test of
    search_acceptable_aligned with every optional filter at its default"""
    return matches > 0 and finish_hit(qlen, tlen, aligned, matches, mismatches, gaps, trims, iddef)[2] >= threshold


def oracle_row_fields(q: bytes, t: bytes, iddef=2, pen=None, n_mismatch=0):
    """what a search result row for (q, t) holds according to the oracle: score and statistics of oracle_nw16, the
    trims of its CIGAR and finish_hit's internal length, internal gaps and identity"""
    score, al, ma, mi, ga, cig = oracle_nw16(q, t, pen, n_mismatch)
    trims = trims_from_cigar(cig)
    internal, igaps, ident = finish_hit(len(q), len(t), al, ma, mi, ga, trims, iddef)
    return dict(nwscore=score, aligned=al, matches=ma, mismatches=mi, gaps=ga, trims=trims,
                internal_alignment_length=internal, internal_gaps=igaps, id=ident)


ROW_FIELDS = ("nwscore", "query_length", "target_length", "matches", "mismatches", "gaps", "alignment_length",
              "internal_alignment_length", "internal_gaps", "id")


def check_search_rows(res, counts, max_results, queries, targets, iddef=2, pen=None, n_mismatch=0):
    """every returned row of a plus-strand search against the oracle, field by field (nwscore, lengths, statistics,
    internal alignment length and gaps, identity).  queries / targets: synth.SeqSet or lists of bytes.
    Returns the number of rows checked."""
    seq_q = queries.seq if hasattr(queries, "seq") else queries.__getitem__
    seq_t = targets.seq if hasattr(targets, "seq") else targets.__getitem__
    bad, n = [], 0
    cache = {}
    for i in range(len(counts)):
        for j in range(int(counts[i])):
            r = res[i * max_results + j]
            assert r.strand == 0, (i, j)
            key = (i, r.target)
            if key not in cache:
                q, t = seq_q(i), seq_t(r.target)
                o = oracle_row_fields(q, t, iddef, pen, n_mismatch)
                cache[key] = (o["nwscore"], len(q), len(t), o["matches"], o["mismatches"], o["gaps"], o["aligned"],
                              o["internal_alignment_length"], o["internal_gaps"], o["id"])
            got = tuple(getattr(r, f) for f in ROW_FIELDS)
            if got != cache[key]:
                bad.append((i, j, r.target, dict(zip(ROW_FIELDS, got)), dict(zip(ROW_FIELDS, cache[key]))))
            n += 1
    assert not bad, f"{len(bad)} of {n} rows differ from the oracle; first: {bad[:2]}"
    return n
