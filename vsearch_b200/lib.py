"""ctypes loader for the product library ``vsearch_b200/csrc/libvsg.so`` (C ABI: include/vsg.h).

This is host-side plumbing for tests and bench.py only.  There is no CPU implementation behind it:
if the library or a CUDA device is missing every call fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.environ.get("VSG_LIB") or os.path.join(ROOT, "vsearch_b200", "csrc", "libvsg.so")   # VSG_LIB: an experimental build (A/B runs)
HEADER = os.path.join(ROOT, "include", "vsg.h")

DEFAULT_PEN = (2, -4, 1, 1, 18, 18, 1, 1, 1, 1, 2, 2, 1, 1)
STAT_WORDS = 8

_lib = None


class VsgError(RuntimeError):
    pass


class Scoring(C.Structure):
    _fields_ = [("v", C.c_int64 * 14), ("n_mismatch", C.c_int32)]


class SearchOpts(C.Structure):
    _fields_ = [("id", C.c_double), ("weak_id", C.c_double), ("maxaccepts", C.c_int32),
                ("maxrejects", C.c_int32), ("wordlength", C.c_int32), ("minwordmatches", C.c_int32),
                ("iddef", C.c_int32), ("strand_both", C.c_int32), ("mask_lower", C.c_int32),
                ("lazy", C.c_int32),
                ("minqt", C.c_double), ("maxqt", C.c_double), ("minsl", C.c_double), ("maxsl", C.c_double),
                ("maxid", C.c_double), ("mid", C.c_double), ("query_cov", C.c_double), ("target_cov", C.c_double),
                ("maxsubs", C.c_int64), ("maxgaps", C.c_int64), ("mincols", C.c_int64), ("maxdiffs", C.c_int64),
                ("leftjust", C.c_int32), ("rightjust", C.c_int32),
                ("maxqsize", C.c_int64), ("mintsize", C.c_int64), ("minsizeratio", C.c_double),
                ("maxsizeratio", C.c_double), ("idprefix", C.c_int32), ("idsuffix", C.c_int32),
                ("self", C.c_int32), ("selfid", C.c_int32), ("qmask_dust", C.c_int32), ("unoise", C.c_int32),
                ("query_sizes", C.POINTER(C.c_int64)), ("target_sizes", C.POINTER(C.c_int64)),
                ("query_labels", C.POINTER(C.c_int64)), ("target_labels", C.POINTER(C.c_int64)),
                ("unoise_alpha", C.c_double), ("sizeorder", C.c_int32), ("reserved1", C.c_int32)]


class Profile(C.Structure):
    _fields_ = [("cells", C.c_int64), ("fast_pairs", C.c_int64), ("exact_pairs", C.c_int64),
                ("fwd_launches", C.c_int64), ("fwd_ms", C.c_float), ("traceback_ms", C.c_float),
                ("rank_ms", C.c_float), ("reserved", C.c_float), ("tb_skipped", C.c_int64), ("tb_redone", C.c_int64)]


class SearchResult(C.Structure):
    _fields_ = [("target", C.c_int32), ("matches", C.c_int32), ("mismatches", C.c_int32),
                ("gaps", C.c_int32), ("alignment_length", C.c_int32), ("query_length", C.c_int32),
                ("target_length", C.c_int32), ("accepted", C.c_int32), ("strand", C.c_int32),
                ("nwscore", C.c_int32), ("id", C.c_double),
                ("internal_alignment_length", C.c_int32), ("internal_gaps", C.c_int32)]


class PairHit(C.Structure):
    _fields_ = [("query", C.c_int32), ("target", C.c_int32), ("matches", C.c_int32), ("mismatches", C.c_int32),
                ("gaps", C.c_int32), ("alignment_length", C.c_int32), ("nwscore", C.c_int32),
                ("internal_alignment_length", C.c_int32), ("id", C.c_double)]


def declared_symbols() -> List[str]:
    """Every function name include/vsg.h declares."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vsg_[a-z0-9_]+)\s*\(", text)))


def load():
    """dlopen libvsg.so and check that it exports everything the header declares."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VsgError(f"{LIB_PATH} not built: run `python __graft_entry__.py` (nvcc, sm_90a). "
                       "There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    if missing:
        raise VsgError(f"libvsg.so does not export: {missing}")
    lib.vsg_last_error.restype = C.c_char_p
    lib.vsg_version.restype = C.c_char_p
    lib.vsg_launch_count.restype = C.c_int64
    lib.vsg_ctx_stream.restype = C.c_void_p
    lib.vsg_seqset_count.restype = C.c_int64
    lib.vsg_group_ctx.restype = C.c_void_p
    lib.vsg_group_db.restype = C.c_void_p
    lib.vsg_group_index.restype = C.c_void_p
    lib.vsg_udb_header.restype = C.c_char_p
    _lib = lib
    return lib


def launch_count() -> int:
    return int(load().vsg_launch_count())


def _check(rc: int, what: str):
    if rc != 0:
        raise VsgError(f"{what} failed ({rc}): {load().vsg_last_error().decode()}")


def _ptr(a: Optional[np.ndarray], t):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.POINTER(t))


@dataclass
class AlignResult:
    score: np.ndarray
    aligned: np.ndarray
    matches: np.ndarray
    mismatches: np.ndarray
    gaps: np.ndarray
    trims: np.ndarray
    cigars: Optional[List[str]]
    cells: int = 0
    fwd_ms: float = 0.0
    tb_ms: float = 0.0
    fast_pairs: int = 0
    exact_pairs: int = 0


class SeqSetHandle:
    def __init__(self, ctx: "Context", h, n: int, lens: np.ndarray):
        self.ctx, self.h, self.n, self.lens = ctx, h, n, lens

    def close(self):
        if self.h:
            load().vsg_seqset_destroy(self.h)
            self.h = None

    def dust(self):
        """DUST soft-masking in place on the device (vsg_seqset_dust)"""
        _check(load().vsg_seqset_dust(self.ctx.h, self.h), "vsg_seqset_dust")

    def symbols(self, total: int) -> np.ndarray:
        out = np.zeros(total, dtype=np.uint8)
        _check(load().vsg_seqset_symbols(self.ctx.h, self.h, _ptr(out, C.c_uint8), C.c_int64(total)),
               "vsg_seqset_symbols")
        return out


class IndexHandle:
    def __init__(self, h):
        self.h = h

    def close(self):
        if self.h:
            load().vsg_index_destroy(self.h)
            self.h = None


class ClusterIndex:
    """vsg_cluster_index: the cluster driver's incremental index, grown by append(seqnos); rank() returns DENSE target
    numbers (append order)"""

    def __init__(self, ctx: "Context", ss: SeqSetHandle, wordlength: int, mask_lower: int):
        self._keep = (ctx, ss)
        self.ctx = ctx
        self.h = C.c_void_p()
        lib = load()
        lib.vsg_cluster_index_count.restype = C.c_int64
        _check(lib.vsg_cluster_index_create(ctx.h, ss.h, C.c_int(wordlength), C.c_int(mask_lower), C.byref(self.h)),
               "vsg_cluster_index_create")

    def append(self, seqnos):
        s = np.ascontiguousarray(seqnos, dtype=np.uint32)
        _check(load().vsg_cluster_index_append(self.ctx.h, self.h, _ptr(s, C.c_uint32), C.c_int64(s.shape[0])),
               "vsg_cluster_index_append")

    @property
    def count(self) -> int:
        return int(load().vsg_cluster_index_count(self.h))

    def rank(self, qs: SeqSetHandle, q0: int, nq: int, minwordmatches: int, tophits: int):
        """(cand[nq, tophits], count[nq, tophits], ncand[nq]) as Context.rank, candidates as dense numbers"""
        cand = np.zeros((nq, tophits), dtype=np.uint32)
        count = np.zeros((nq, tophits), dtype=np.uint32)
        nc = np.zeros(nq, dtype=np.int32)
        _check(load().vsg_cluster_index_rank(self.ctx.h, self.h, qs.h, C.c_int64(q0), C.c_int64(nq), C.c_int(minwordmatches),
                                             C.c_int(tophits), _ptr(cand, C.c_uint32), _ptr(count, C.c_uint32),
                                             _ptr(nc, C.c_int32)), "vsg_cluster_index_rank")
        return cand, count, nc

    def close(self):
        if self.h:
            load().vsg_cluster_index_destroy(self.h)
            self.h = C.c_void_p()


class Context:
    """vsg_ctx: one CUDA stream + scratch; mirrors the reference's per-thread s16info_s."""

    def __init__(self, device: int = 0, pen=DEFAULT_PEN, n_mismatch: int = 0):
        lib = load()
        sc = Scoring()
        for i in range(14):
            sc.v[i] = int(pen[i])
        sc.n_mismatch = int(n_mismatch)
        self.h = C.c_void_p()
        _check(lib.vsg_ctx_create(C.c_int(device), C.byref(sc), C.byref(self.h)), "vsg_ctx_create")

    def close(self):
        if self.h:
            load().vsg_ctx_destroy(self.h)
            self.h = None

    def set_fallback(self, fn):
        """fn(query_index, strand, target_index) -> 9 or 10 ints (score, alnlen, matches, mismatches, gaps,
        trim_q_left, trim_t_left, trim_q_right, trim_t_right[, forbidden]); see vsg_ctx_set_fallback."""
        proto = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.POINTER(C.c_int64))

        def tramp(_user, q, strand, t, out):
            try:
                vals = fn(int(q), int(strand), int(t))
                for i in range(len(vals)):
                    out[i] = int(vals[i])
                return 0
            except Exception:
                return 1
        self._fallback_keep = proto(tramp)
        _check(load().vsg_ctx_set_fallback(self.h, self._fallback_keep, None), "vsg_ctx_set_fallback")

    def profile_reset(self):
        _check(load().vsg_profile_reset(self.h), "vsg_profile_reset")

    def profile(self) -> Profile:
        p = Profile()
        _check(load().vsg_profile_get(self.h, C.byref(p)), "vsg_profile_get")
        return p

    def int_peak(self) -> float:
        v = C.c_double()
        _check(load().vsg_measure_int_peak(self.h, C.byref(v)), "vsg_measure_int_peak")
        return v.value

    def stream_ptr(self) -> int:
        return int(load().vsg_ctx_stream(self.h))

    def sync(self):
        _check(load().vsg_ctx_sync(self.h), "vsg_ctx_sync")

    def seqset(self, ss) -> SeqSetHandle:
        """Upload a synth.SeqSet-like object (cat uint8, offs int64, lens int32) into HBM."""
        h = C.c_void_p()
        cat = np.ascontiguousarray(ss.cat, dtype=np.uint8)
        offs = np.ascontiguousarray(ss.offs, dtype=np.int64)
        lens = np.ascontiguousarray(ss.lens, dtype=np.int32)
        _check(load().vsg_seqset_create(self.h, _ptr(cat, C.c_char), _ptr(offs, C.c_int64),
                                        _ptr(lens, C.c_int32), C.c_int64(lens.shape[0]), C.c_int(1),
                                        C.byref(h)), "vsg_seqset_create")
        return SeqSetHandle(self, h, int(lens.shape[0]), lens)

    def seqset_from_device(self, d_cat: int, d_off: int, d_len: int, n: int) -> SeqSetHandle:
        """Adopt ASCII/offset/length arrays that already live in this device's HBM (raw pointers)."""
        h = C.c_void_p()
        _check(load().vsg_seqset_create(self.h, C.cast(C.c_void_p(d_cat), C.POINTER(C.c_char)),
                                        C.cast(C.c_void_p(d_off), C.POINTER(C.c_int64)),
                                        C.cast(C.c_void_p(d_len), C.POINTER(C.c_int32)),
                                        C.c_int64(n), C.c_int(0), C.byref(h)), "vsg_seqset_create")
        return SeqSetHandle(self, h, n, None)

    def revcomp(self, ss: SeqSetHandle, q0: int = 0, n: Optional[int] = None) -> SeqSetHandle:
        """vsg_seqset_revcomp: the reverse complements of sequences [q0, q0 + n) of `ss` (default: to the end) as a
        new set, made on the device; the case (soft mask) of every symbol is kept."""
        if n is None:
            n = ss.n - q0
        h = C.c_void_p()
        _check(load().vsg_seqset_revcomp(self.h, ss.h, C.c_int64(q0), C.c_int64(n), C.byref(h)), "vsg_seqset_revcomp")
        lens = ss.lens[q0:q0 + n] if ss.lens is not None else None
        return SeqSetHandle(self, h, n, lens)

    def align_pairs(self, qs: SeqSetHandle, ts: SeqSetHandle, qidx: np.ndarray, tidx: np.ndarray,
                    cigar: bool = False) -> AlignResult:
        lib = load()
        qidx = np.ascontiguousarray(qidx, dtype=np.uint32)
        tidx = np.ascontiguousarray(tidx, dtype=np.uint32)
        n = int(qidx.shape[0])
        score = np.zeros(n, dtype=np.int16)
        al = np.zeros(n, dtype=np.uint16); ma = np.zeros(n, dtype=np.uint16)
        mi = np.zeros(n, dtype=np.uint16); ga = np.zeros(n, dtype=np.uint16)
        trims = np.zeros((n, 4), dtype=np.int32)
        cbuf = coff = None
        cap = 0
        if cigar:
            cap = int((qs.lens[qidx].astype(np.int64) + ts.lens[tidx].astype(np.int64) + 2).sum()) + 16
            cbuf = np.zeros(cap, dtype=np.uint8)
            coff = np.zeros(n + 1, dtype=np.int64)
        self.profile_reset()
        _check(lib.vsg_align_pairs(self.h, qs.h, ts.h, C.c_int64(n), _ptr(qidx, C.c_uint32),
                                   _ptr(tidx, C.c_uint32), _ptr(score, C.c_int16), _ptr(al, C.c_uint16),
                                   _ptr(ma, C.c_uint16), _ptr(mi, C.c_uint16), _ptr(ga, C.c_uint16),
                                   _ptr(trims, C.c_int32), _ptr(cbuf, C.c_char), C.c_int64(cap),
                                   _ptr(coff, C.c_int64)), "vsg_align_pairs")
        cigs = None
        if cigar:
            raw = cbuf.tobytes()
            cigs = [raw[int(coff[i]):int(coff[i + 1]) - 1].decode() for i in range(n)]
        pr = self.profile()
        return AlignResult(score, al, ma, mi, ga, trims, cigs, pr.cells, pr.fwd_ms, pr.traceback_ms,
                           pr.fast_pairs, pr.exact_pairs)

    def align_pairs_gated(self, qs: SeqSetHandle, ts: SeqSetHandle, qidx: np.ndarray, tidx: np.ndarray,
                          leader_of: np.ndarray, threshold: float, iddef: int):
        """vsg_align_pairs_gated -> (AlignResult, (stored, score-only, re-run) checkpoint task counts, tb_skipped)"""
        lib = load()
        qidx = np.ascontiguousarray(qidx, dtype=np.uint32)
        tidx = np.ascontiguousarray(tidx, dtype=np.uint32)
        lead = np.ascontiguousarray(leader_of, dtype=np.int32)
        n = int(qidx.shape[0])
        assert tidx.shape[0] == n and lead.shape[0] == n
        score = np.zeros(n, dtype=np.int16)
        al = np.zeros(n, dtype=np.uint16); ma = np.zeros(n, dtype=np.uint16)
        mi = np.zeros(n, dtype=np.uint16); ga = np.zeros(n, dtype=np.uint16)
        trims = np.zeros((n, 4), dtype=np.int32)
        ck = np.zeros(3, dtype=np.int64)
        self.profile_reset()
        _check(lib.vsg_align_pairs_gated(self.h, qs.h, ts.h, C.c_int64(n), _ptr(qidx, C.c_uint32), _ptr(tidx, C.c_uint32),
                                         _ptr(score, C.c_int16), _ptr(al, C.c_uint16), _ptr(ma, C.c_uint16),
                                         _ptr(mi, C.c_uint16), _ptr(ga, C.c_uint16), _ptr(trims, C.c_int32),
                                         _ptr(lead, C.c_int32), C.c_double(threshold), C.c_int(iddef),
                                         _ptr(ck, C.c_int64)), "vsg_align_pairs_gated")
        pr = self.profile()
        res = AlignResult(score, al, ma, mi, ga, trims, None, pr.cells, pr.fwd_ms, pr.traceback_ms,
                          pr.fast_pairs, pr.exact_pairs)
        return res, tuple(int(x) for x in ck), int(pr.tb_skipped)

    def index(self, db: SeqSetHandle, wordlength: int = 8, mask_lower: int = 0) -> IndexHandle:
        h = C.c_void_p()
        _check(load().vsg_index_create(self.h, db.h, C.c_int(wordlength), C.c_int(mask_lower),
                                       C.byref(h)), "vsg_index_create")
        return IndexHandle(h)

    def cluster_index(self, ss: SeqSetHandle, wordlength: int = 8, mask_lower: int = 0) -> "ClusterIndex":
        """vsg_cluster_index_create: the cluster driver's incremental index over sequences of `ss`, empty at first"""
        return ClusterIndex(self, ss, wordlength, mask_lower)

    def udb_make(self, seqs, headers, wordlength=8, dbmask="dust", hardmask=False) -> "Udb":
        """vsg_udb_make: the in-memory UDB database of the records `seqs` (bytes each) with `headers` (str each)"""
        o = makeudb_opts(wordlength=wordlength, dbmask=dbmask, hardmask=hardmask)
        cat = np.frombuffer(b"".join(seqs) + b"\0", dtype=np.uint8)
        ln = np.array([len(x) for x in seqs], dtype=np.int32)
        off = np.zeros(len(seqs), dtype=np.int64)
        if len(seqs) > 1:
            off[1:] = np.cumsum(ln[:-1], dtype=np.int64)
        hs = (C.c_char_p * max(1, len(headers)))(*[h.encode() for h in headers])
        h = C.c_void_p()
        _check(load().vsg_udb_make(self.h, cat.ctypes.data_as(C.c_char_p), _ptr(off, C.c_int64), _ptr(ln, C.c_int32), hs,
                                   C.c_int64(len(seqs)), C.byref(o), C.byref(h)), "vsg_udb_make")
        return Udb._wrap(h)

    def makeudb_usearch(self, input_path: str, output_path: Optional[str], **opts) -> dict:
        """vsg_makeudb_usearch (the --makeudb_usearch command); opts as makeudb_opts; returns the stats as a dict"""
        o = makeudb_opts(**opts)
        st = MakeudbStats()
        _check(load().vsg_makeudb_usearch(self.h, input_path.encode(), C.byref(o),
                                          output_path.encode() if output_path is not None else None, C.byref(st)),
               "vsg_makeudb_usearch")
        return {k: getattr(st, k) for k, _ in MakeudbStats._fields_}

    def cluster_command(self, input_path: str, uc: Optional[str] = None, centroids: Optional[str] = None,
                        clusters: Optional[str] = None, command: str = "cluster_fast", msaout: Optional[str] = None,
                        consout: Optional[str] = None, profile: Optional[str] = None, **opts) -> dict:
        """vsg_cluster_command_outputs (--cluster_fast / _size / _smallmem / _unoise: a key of CLUSTER_COMMANDS): reads
        input_path, writes --uc, --centroids, --clusters <prefix>, --msaout, --consout and --profile (None: not written);
        opts as cluster_cmd_opts (id=0.97, threads=8, qmask="soft", sizeout=1, ...).  Returns the stats as a dict."""
        c, s = cluster_cmd_opts(command, **opts)
        st = ClusterCmdStats()
        out = ClusterCmdOutputs(*_cluster_cmd_paths(uc, centroids, clusters), *_cluster_cmd_paths(msaout, consout, profile))
        _check(load().vsg_cluster_command_outputs(self.h, input_path.encode(), C.byref(c), C.byref(s), C.byref(out),
                                                  C.byref(st)), "vsg_cluster_command")
        return {k: getattr(st, k) for k, _ in ClusterCmdStats._fields_}

    def cluster_msa(self, ss: SeqSetHandle, results: np.ndarray, weights, cigars) -> dict:
        """vsg_cluster_msa: the column layout, profile and consensus of the clusters of `results` (records of `ss` in
        processing order, a cluster result array) with per-record `weights` and the CIGAR (str) of each H record.
        Returns numpy arrays: insertions (int32), col_first (int64, clusters + 1), profile (uint64, columns x 6: A, C, G,
        T, N, gap) and consensus (uint8, one char per column)."""
        res = np.ascontiguousarray(results, dtype=_CLUSTER_DT)
        n = res.shape[0]
        w = np.ascontiguousarray(weights, dtype=np.uint64)
        cbuf, coff = _cigar_buf(cigars, n)
        nins = int((ss.lens[:n][res["centroid"] < 0].astype(np.int64) + 1).sum()) if n else 0
        nclusters = int(res["cluster"].max()) + 1 if n else 0
        ins = np.zeros(max(nins, 1), dtype=np.int32)
        first = np.zeros(nclusters + 1, dtype=np.int64)
        ncols = C.c_int64()
        args = lambda prof, cons, cap: (self.h, ss.h, C.c_int64(n), res.ctypes.data_as(C.POINTER(ClusterResult)),  # noqa: E731
                                        _ptr(w, C.c_uint64), cbuf.ctypes.data_as(C.c_char_p), _ptr(coff, C.c_int64),
                                        _ptr(ins, C.c_int32), _ptr(first, C.c_int64), _ptr(prof, C.c_uint64),
                                        _ptr(cons, C.c_char), C.c_int64(cap), C.byref(ncols))
        rc = load().vsg_cluster_msa(*args(None, None, 0))
        if rc == -5:   # VSG_ECAP: sized by the first call
            prof = np.zeros((ncols.value, 6), dtype=np.uint64)
            cons = np.zeros(ncols.value, dtype=np.uint8)
            rc = load().vsg_cluster_msa(*args(prof, cons, ncols.value))
        else:
            prof = np.zeros((0, 6), dtype=np.uint64)
            cons = np.zeros(0, dtype=np.uint8)
        _check(rc, "vsg_cluster_msa")
        return {"insertions": ins[:nins], "col_first": first, "profile": prof, "consensus": cons}

    def exact_index(self, db: SeqSetHandle) -> "ExactIndex":
        """vsg_exact_index_create: the hash index of every sequence of `db` (which must outlive it)"""
        h = C.c_void_p()
        _check(load().vsg_exact_index_create(self.h, db.h, C.byref(h)), "vsg_exact_index_create")
        return ExactIndex(h)

    def search_exact(self, ix: "ExactIndex", qs: SeqSetHandle, q0: int, nq: int, opts: SearchOpts, maxhits: int = 0,
                     cap: Optional[int] = None):
        """vsg_search_exact -> (rows, first[nq + 1], work[4], unused); query i's rows are rows[first[i]:first[i + 1]].
        cap=None: the buffer is sized by a first call that reports the number of rows (VSG_ECAP)."""
        return _hits_call(lambda hits, c, first, n, _work: load().vsg_search_exact(
            self.h, ix.h, qs.h, C.c_int64(q0), C.c_int64(nq), C.byref(opts), C.c_int64(maxhits), hits, C.c_int64(c), first, n),
            nq, cap, "vsg_search_exact")

    def search_exact_command(self, query_path: str, db_path: str, /, **kw) -> dict:
        """vsg_search_exact_command (--search_exact): keywords naming an output of SearchExactOutputs give its path, those
        of vsg_search_exact_opts its value (qmask / dbmask may be "none" / "soft" / "dust"), the rest go to the search
        options (strand_both, self, mintsize, ...; the arguments before them are positional-only, so `self` can be one).
        Returns the stats as a dict."""
        e, s, o = search_exact_opts(**kw)
        st = SearchExactStats()
        _check(load().vsg_search_exact_command(self.h, query_path.encode(), db_path.encode(), C.byref(e), C.byref(s), C.byref(o),
                                               C.byref(st)), "vsg_search_exact_command")
        return {k: getattr(st, k) for k, _ in SearchExactStats._fields_}

    def usearch_global_command(self, query_path: str, db_path: str, /, **kw) -> dict:
        """vsg_usearch_global_command (--usearch_global): keywords naming an output of SearchExactOutputs give its path,
        those of vsg_usearch_global_opts its value (qmask / dbmask may be "none" / "soft" / "dust"), the rest go to the
        search options (id, weak_id, maxaccepts, strand_both, self, ...; the arguments before them are positional-only, so
        `self` can be one).  db_path may be a FASTA / FASTQ file or a UDB file.  Returns the stats as a dict."""
        u, s, o = usearch_global_opts(**kw)
        st = UsearchGlobalStats()
        _check(load().vsg_usearch_global_command(self.h, query_path.encode(), db_path.encode(), C.byref(u), C.byref(s), C.byref(o),
                                                 C.byref(st)), "vsg_usearch_global_command")
        return {k: getattr(st, k) for k, _ in UsearchGlobalStats._fields_}

    def uchime(self, input_path: str, db_path: Optional[str] = None, /, **kw) -> dict:
        """vsg_uchime_command: --uchime_ref with db_path a FASTA or UDB file, de novo (command=UCHIME_DENOVO, _2_, _3_ or CHIMERAS_DENOVO,
        or its name) with db_path None.  Keywords naming an output of UCHIME_OUTPUTS give its path, the rest the fields of
        vsg_uchime_opts (qmask / dbmask may be "none" / "soft" / "dust").
        Returns the stats as a dict."""
        o, out = uchime_opts(**kw)
        st = UchimeStats()
        _check(load().vsg_uchime_command(self.h, input_path.encode(), None if db_path is None else db_path.encode(), C.byref(o),
                                         C.byref(out), C.byref(st)), "vsg_uchime_command")
        return {k: getattr(st, k) for k, _ in UchimeStats._fields_}

    def udb_load(self, udb: "Udb"):
        """vsg_udb_load: (SeqSetHandle, IndexHandle, mask_lower) of a parsed UDB file"""
        sh = C.c_void_p(); ih = C.c_void_p(); ml = C.c_int(-1)
        _check(load().vsg_udb_load(self.h, udb.h, C.byref(sh), C.byref(ih), C.byref(ml)), "vsg_udb_load")
        _, _, lens = udb.sequences()
        return SeqSetHandle(self, sh, udb.n, lens), IndexHandle(ih), int(ml.value)

    def rank(self, ix: IndexHandle, qs: SeqSetHandle, q0: int, nq: int, minwordmatches: int,
             tophits: int, mask_lower: int = 0):
        seqno = np.zeros((nq, tophits), dtype=np.uint32)
        count = np.zeros((nq, tophits), dtype=np.uint32)
        nc = np.zeros(nq, dtype=np.int32)
        _check(load().vsg_rank(self.h, ix.h, qs.h, C.c_int64(q0), C.c_int64(nq), C.c_int(minwordmatches),
                               C.c_int(tophits), C.c_int(mask_lower), _ptr(seqno, C.c_uint32),
                               _ptr(count, C.c_uint32), _ptr(nc, C.c_int32)), "vsg_rank")
        return seqno, count, nc

    def rank_occupancy(self):
        """(full, short): CTAs per SM of the ranker's full and short-query instances"""
        full = C.c_int(); short = C.c_int()
        _check(load().vsg_rank_occupancy(self.h, C.byref(full), C.byref(short)), "vsg_rank_occupancy")
        return full.value, short.value

    def sintax(self, ix: IndexHandle, qs: SeqSetHandle, q0: int, nq: int, seed: int, strand_both: int = 0,
               query_number0: Optional[int] = None, random_ties: int = 0):
        """vsg_sintax -> dict of numpy arrays: strand[nq], nboot[nq, 2], best_count[nq, 2], seqno[nq, 2, 100] (-1 beyond
        nboot); query q0 + i uses random substream query_number0 + i (default: q0 + i)"""
        o = sintax_opts(seed, strand_both, query_number0=q0 if query_number0 is None else query_number0, random_ties=random_ties)
        res = np.zeros(nq, dtype=SINTAX_DT)
        _check(load().vsg_sintax(self.h, ix.h, qs.h, C.c_int64(q0), C.c_int64(nq), C.byref(o),
                                 res.ctypes.data_as(C.c_void_p) if nq > 0 else None), "vsg_sintax")
        return {k: res[k] for k in SINTAX_DT.names}

    def orient(self, ix: IndexHandle, qs: SeqSetHandle, q0: int, nq: int, query_mask_lower: int = 1) -> np.ndarray:
        """vsg_orient -> an (nq, 3) int64 array of (strand 0 '+' / 1 '-' / 2 '?', count_fwd, count_rev) for queries
        q0 .. q0 + nq - 1"""
        res = np.zeros(nq, dtype=ORIENT_DT)
        _check(load().vsg_orient(self.h, ix.h, qs.h, C.c_int64(q0), C.c_int64(nq), C.c_int(query_mask_lower),
                                 res.ctypes.data_as(C.c_void_p) if nq > 0 else None), "vsg_orient")
        return np.stack([res["strand"].astype(np.int64), res["count_fwd"].astype(np.int64),
                         res["count_rev"].astype(np.int64)], axis=1)

    def search(self, ix: IndexHandle, db: SeqSetHandle, qs: SeqSetHandle, q0: int, nq: int,
               opts: SearchOpts, max_results: int):
        res = (SearchResult * (nq * max_results))()
        counts = np.zeros(nq, dtype=np.int32)
        work = np.zeros(4, dtype=np.int64)
        _check(load().vsg_search_batch(self.h, ix.h, db.h, qs.h, C.c_int64(q0), C.c_int64(nq),
                                       C.byref(opts), res, C.c_int(max_results), _ptr(counts, C.c_int32),
                                       _ptr(work, C.c_int64)), "vsg_search_batch")
        return res, counts, work

    def search_hits(self, ix: IndexHandle, db: SeqSetHandle, qs: SeqSetHandle, q0: int, nq: int,
                    opts: SearchOpts, maxhits: int = 0, cap: Optional[int] = None):
        """vsg_search_hits -> (rows, first[nq + 1], work[4]); query i's rows are rows[first[i]:first[i + 1]].
        cap=None: the buffer is sized by a first call that reports the number of rows (VSG_ECAP) — that call runs the
        whole search, so cap=None costs two searches; pass the row count when it is known (e.g. to time one search)."""
        return _hits_call(lambda hits, c, first, n, work: load().vsg_search_hits(
            self.h, ix.h, db.h, qs.h, C.c_int64(q0), C.c_int64(nq), C.byref(opts), C.c_int64(maxhits), hits, C.c_int64(c),
            first, n, work), nq, cap, "vsg_search_hits")


def _hits_call(call, nq: int, cap: Optional[int], what: str):
    """a vsg_*search_hits call with a buffer of `cap` rows; cap=None: sized by a first call with cap 0 (VSG_ECAP), which
    runs the whole search once more"""
    first = np.zeros(nq + 1, dtype=np.int64)
    work = np.zeros(4, dtype=np.int64)
    n = C.c_int64()
    if cap is None:
        rc = call(None, 0, _ptr(first, C.c_int64), C.byref(n), _ptr(work, C.c_int64))
        if rc == 0:
            return (SearchResult * 0)(), first, work
        if rc != -5:
            _check(rc, what)
        cap = int(n.value)
    hits = (SearchResult * max(cap, 1))()
    _check(call(hits, cap, _ptr(first, C.c_int64), C.byref(n), _ptr(work, C.c_int64)), what)
    return hits, first, work


def allpairs(ctx: "Context", ss: SeqSetHandle, row0: int, nrows: int, opts: SearchOpts, cap: int):
    """vsg_allpairs -> (numpy structured array of hits, work[2])"""
    dt = np.dtype([("query", np.int32), ("target", np.int32), ("matches", np.int32), ("mismatches", np.int32),
                   ("gaps", np.int32), ("alignment_length", np.int32), ("nwscore", np.int32),
                   ("internal_alignment_length", np.int32), ("id", np.float64)])
    assert dt.itemsize == C.sizeof(PairHit)
    hits = np.zeros(cap, dtype=dt)
    n = C.c_int64()
    work = np.zeros(2, dtype=np.int64)
    _check(load().vsg_allpairs(ctx.h, ss.h, C.c_int64(row0), C.c_int64(nrows), C.byref(opts),
                               hits.ctypes.data_as(C.POINTER(PairHit)), C.c_int64(cap), C.byref(n),
                               _ptr(work, C.c_int64)), "vsg_allpairs")
    return hits[: n.value], work


class ClusterResult(C.Structure):
    _fields_ = [("cluster", C.c_int32), ("centroid", C.c_int32), ("matches", C.c_int32), ("mismatches", C.c_int32),
                ("gaps", C.c_int32), ("alignment_length", C.c_int32), ("nwscore", C.c_int32), ("strand", C.c_int32),
                ("id", C.c_double)]


def cluster_fast(ctx: "Context", ss: SeqSetHandle, opts: SearchOpts, round_size: int):
    """vsg_cluster_fast -> (numpy structured array of per-sequence results, number of clusters, work[2])"""
    dt = np.dtype([("cluster", np.int32), ("centroid", np.int32), ("matches", np.int32), ("mismatches", np.int32),
                   ("gaps", np.int32), ("alignment_length", np.int32), ("nwscore", np.int32), ("strand", np.int32),
                   ("id", np.float64)])
    assert dt.itemsize == C.sizeof(ClusterResult)
    res = np.zeros(ss.n, dtype=dt)
    ncl = C.c_int64()
    work = np.zeros(2, dtype=np.int64)
    _check(load().vsg_cluster_fast(ctx.h, ss.h, C.byref(opts), C.c_int(round_size), res.ctypes.data_as(C.POINTER(ClusterResult)),
                                   C.byref(ncl), _ptr(work, C.c_int64)), "vsg_cluster_fast")
    return res, int(ncl.value), work


_CLUSTER_DT = np.dtype([("cluster", np.int32), ("centroid", np.int32), ("matches", np.int32), ("mismatches", np.int32),
                        ("gaps", np.int32), ("alignment_length", np.int32), ("nwscore", np.int32), ("strand", np.int32),
                        ("id", np.float64)])
CLUSTER_DT = _CLUSTER_DT   # one vsg_cluster_result


class ClusterSession:
    """vsg_cluster_session: the clustering fed range by range (cluster_assign_batch / cluster_assign_single)"""

    def __init__(self, ctx: "Context", ss: SeqSetHandle, opts: SearchOpts):
        self._keep = (ctx, ss, opts)
        self.h = C.c_void_p()
        lib = load()
        lib.vsg_cluster_session_clusters.restype = C.c_int64
        _check(lib.vsg_cluster_session_create(ctx.h, ss.h, C.byref(opts), C.byref(self.h)), "vsg_cluster_session_create")

    def assign(self, start: int, count: int, round_size: int):
        res = np.zeros(count, dtype=_CLUSTER_DT)
        _check(load().vsg_cluster_session_assign(self.h, C.c_int64(start), C.c_int64(count), C.c_int(round_size),
                                                 res.ctypes.data_as(C.POINTER(ClusterResult))), "vsg_cluster_session_assign")
        return res

    @property
    def clusters(self) -> int:
        return int(load().vsg_cluster_session_clusters(self.h))

    def close(self):
        if self.h:
            load().vsg_cluster_session_destroy(self.h)
            self.h = C.c_void_p()


class Group:
    """vsg_group: one process, several GPUs (database copied device to device, queries / rows sharded)"""

    def __init__(self, devices, ss, wordlength=8, mask_lower=0, dust_db=0, pen=DEFAULT_PEN, n_mismatch=0):
        lib = load()
        sc = Scoring()
        for i in range(14):
            sc.v[i] = int(pen[i])
        sc.n_mismatch = int(n_mismatch)
        dev = np.ascontiguousarray(devices, dtype=np.int32)
        cat = np.ascontiguousarray(ss.cat, dtype=np.uint8)
        offs = np.ascontiguousarray(ss.offs, dtype=np.int64)
        lens = np.ascontiguousarray(ss.lens, dtype=np.int32)
        self.h = C.c_void_p()
        self.n = int(lens.shape[0])
        _check(lib.vsg_group_create(_ptr(dev, C.c_int), C.c_int(dev.shape[0]), C.byref(sc), _ptr(cat, C.c_char),
                                    _ptr(offs, C.c_int64), _ptr(lens, C.c_int32), C.c_int64(self.n), C.c_int(wordlength),
                                    C.c_int(mask_lower), C.c_int(dust_db), C.byref(self.h)), "vsg_group_create")

    @classmethod
    def from_udb(cls, devices, udb: "Udb", pen=DEFAULT_PEN, n_mismatch=0):
        """vsg_group_create_udb: the database of a parsed UDB file on every device"""
        self = cls.__new__(cls)
        sc = Scoring()
        for i in range(14):
            sc.v[i] = int(pen[i])
        sc.n_mismatch = int(n_mismatch)
        dev = np.ascontiguousarray(devices, dtype=np.int32)
        self.h = C.c_void_p()
        self.n = udb.n
        _check(load().vsg_group_create_udb(_ptr(dev, C.c_int), C.c_int(dev.shape[0]), C.byref(sc), udb.h, C.byref(self.h)),
               "vsg_group_create_udb")
        return self

    def close(self):
        if self.h:
            load().vsg_group_destroy(self.h)
            self.h = None

    def stats(self):
        ms = np.zeros(3, dtype=np.float64)
        b = C.c_int64()
        _check(load().vsg_group_stats(self.h, _ptr(ms, C.c_double), C.byref(b)), "vsg_group_stats")
        return {"upload_ms": float(ms[0]), "broadcast_ms": float(ms[1]), "index_ms": float(ms[2]), "broadcast_bytes": int(b.value)}

    def search(self, qs, opts: SearchOpts, max_results: int, dust_queries: int = 0):
        nq = len(qs)
        res = (SearchResult * (nq * max_results))()
        counts = np.zeros(nq, dtype=np.int32)
        work = np.zeros(4, dtype=np.int64)
        cat = np.ascontiguousarray(qs.cat, dtype=np.uint8)
        offs = np.ascontiguousarray(qs.offs, dtype=np.int64)
        lens = np.ascontiguousarray(qs.lens, dtype=np.int32)
        _check(load().vsg_group_search(self.h, _ptr(cat, C.c_char), _ptr(offs, C.c_int64), _ptr(lens, C.c_int32),
                                       C.c_int64(nq), C.c_int(dust_queries), C.byref(opts), res, C.c_int(max_results),
                                       _ptr(counts, C.c_int32), _ptr(work, C.c_int64)), "vsg_group_search")
        return res, counts, work

    def search_hits(self, qs, opts: SearchOpts, maxhits: int = 0, dust_queries: int = 0, cap: Optional[int] = None):
        """vsg_group_search_hits -> (rows, first[nq + 1], work[4]), as Context.search_hits (cap=None: two searches)"""
        nq = len(qs)
        cat = np.ascontiguousarray(qs.cat, dtype=np.uint8)
        offs = np.ascontiguousarray(qs.offs, dtype=np.int64)
        lens = np.ascontiguousarray(qs.lens, dtype=np.int32)
        return _hits_call(lambda hits, c, first, n, work: load().vsg_group_search_hits(
            self.h, _ptr(cat, C.c_char), _ptr(offs, C.c_int64), _ptr(lens, C.c_int32), C.c_int64(nq), C.c_int(dust_queries),
            C.byref(opts), C.c_int64(maxhits), hits, C.c_int64(c), first, n, work), nq, cap, "vsg_group_search_hits")

    def allpairs(self, opts: SearchOpts, cap: int):
        dt = np.dtype([("query", np.int32), ("target", np.int32), ("matches", np.int32), ("mismatches", np.int32),
                       ("gaps", np.int32), ("alignment_length", np.int32), ("nwscore", np.int32),
                       ("internal_alignment_length", np.int32), ("id", np.float64)])
        hits = np.zeros(cap, dtype=dt)
        n = C.c_int64()
        work = np.zeros(2, dtype=np.int64)
        _check(load().vsg_group_allpairs(self.h, C.byref(opts), hits.ctypes.data_as(C.POINTER(PairHit)), C.c_int64(cap),
                                         C.byref(n), _ptr(work, C.c_int64)), "vsg_group_allpairs")
        return hits[: n.value], work

    def stream(self, target_labels, query_fasta: str, opts: SearchOpts, blast6out: str, qmask_dust: int = 0, notrunclabels: int = 0,
               batch_queries: int = 65536, maxhits: int = 0, output_no_hits: int = 0):
        """vsg_usearch_stream: FASTA file in, --blast6out file out; returns the statistics record as a dict"""
        labs = (C.c_char_p * len(target_labels))(*[l if isinstance(l, bytes) else l.encode() for l in target_labels])
        st = StreamStats()
        _check(load().vsg_usearch_stream(self.h, labs, query_fasta.encode(), C.byref(opts), C.c_int(qmask_dust), C.c_int(notrunclabels),
                                         C.c_int(batch_queries), C.c_int64(maxhits), C.c_int(output_no_hits), blast6out.encode(),
                                         C.byref(st)), "vsg_usearch_stream")
        return {k: getattr(st, k) for k, _ in StreamStats._fields_}

    def sintax_stream(self, target_headers, query_fasta: str, tabbedout: str, seed: int, strand_both: int = 0,
                      cutoff: float = 0.0, batch_queries: int = 65536, random_ties: int = 0):
        """vsg_sintax_stream: the --sintax command, FASTA file in, --tabbedout file out; returns the statistics as a dict"""
        st = StreamStats()
        o = sintax_opts(seed, strand_both, cutoff, random_ties=random_ties)
        _check(load().vsg_sintax_stream(self.h, _strings(target_headers), query_fasta.encode(), C.byref(o), C.c_int(batch_queries),
                                        tabbedout.encode(), C.byref(st)), "vsg_sintax_stream")
        return {k: getattr(st, k) for k, _ in StreamStats._fields_}

    def orient_stream(self, query_path: str, fastaout: Optional[str] = None, fastqout: Optional[str] = None,
                      notmatched: Optional[str] = None, tabbedout: Optional[str] = None, query_mask_lower: int = 1,
                      notrunclabels: int = 0, fasta_width: int = 80, batch_queries: int = 65536):
        """vsg_orient_stream: the --orient command, FASTA or FASTQ file in, the given outputs out (None: off); returns
        (statistics dict, (reads '+', '-', '?'))"""
        st = StreamStats()
        ns = np.zeros(3, dtype=np.int64)
        enc = (lambda p: None if p is None else p.encode())
        _check(load().vsg_orient_stream(self.h, query_path.encode(), C.c_int(query_mask_lower), C.c_int(notrunclabels),
                                        C.c_int(fasta_width), C.c_int(batch_queries), enc(fastaout), enc(fastqout),
                                        enc(notmatched), enc(tabbedout), C.byref(st), _ptr(ns, C.c_int64)),
               "vsg_orient_stream")
        return {k: getattr(st, k) for k, _ in StreamStats._fields_}, tuple(int(x) for x in ns)


ORIENT_DT = np.dtype([("strand", np.int32), ("count_fwd", np.uint32), ("count_rev", np.uint32)])


class SintaxOpts(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("query_number0", C.c_int64), ("strand_both", C.c_int32), ("random_ties", C.c_int32),
                ("cutoff", C.c_double)]


SINTAX_BOOTSTRAPS = 100
SINTAX_DT = np.dtype([("strand", np.int32), ("nboot", np.int32, (2,)), ("best_count", np.int32, (2,)),
                      ("seqno", np.int32, (2, SINTAX_BOOTSTRAPS))])


def sintax_opts(seed: int, strand_both: int = 0, cutoff: float = 0.0, query_number0: int = 0, random_ties: int = 0) -> SintaxOpts:
    return SintaxOpts(seed=seed, query_number0=query_number0, strand_both=strand_both, random_ties=random_ties, cutoff=cutoff)


def _strings(xs):
    return (C.c_char_p * len(xs))(*[x if isinstance(x, bytes) else x.encode() for x in xs])


def sintax_rows(results: np.ndarray, query_headers, target_headers, cutoff: float = 0.0, strand_both: int = 0,
                random_ties: int = 0) -> bytes:
    """vsg_sintax_rows (host only, no device): the --tabbedout rows of a SINTAX_DT array of results"""
    res = np.ascontiguousarray(results, dtype=SINTAX_DT)
    o = sintax_opts(0, strand_both, cutoff, random_ties=random_ties)
    qh, th = _strings(query_headers), _strings(target_headers)
    n = C.c_int64()
    rp = res.ctypes.data_as(C.c_void_p) if res.shape[0] > 0 else None
    rc = load().vsg_sintax_rows(rp, C.c_int64(res.shape[0]), qh, th, C.byref(o), None, C.c_int64(0), C.byref(n))
    if rc == 0:
        return b""
    if rc != -5:
        _check(rc, "vsg_sintax_rows")
    buf = C.create_string_buffer(int(n.value))
    _check(load().vsg_sintax_rows(rp, C.c_int64(res.shape[0]), qh, th, C.byref(o), buf, C.c_int64(n.value), C.byref(n)),
           "vsg_sintax_rows")
    return buf.raw[: n.value]


class UdbInfo(C.Structure):
    _fields_ = [("sequences", C.c_int64), ("nucleotides", C.c_int64), ("header_chars", C.c_int64), ("index_entries", C.c_int64),
                ("longest_header", C.c_int64), ("wordlength", C.c_int32), ("dbaccel", C.c_int32), ("shortest", C.c_int32),
                ("longest", C.c_int32)]


def udb_detect(path: str) -> bool:
    rc = load().vsg_udb_detect(path.encode())
    if rc < 0:
        _check(rc, "vsg_udb_detect")
    return rc == 1


class Udb:
    """A parsed UDB file (host side; no GPU needed): vsg_udb_open and its accessors; or a database made by
    Context.udb_make (vsg_udb_make)."""

    def __init__(self, path: Optional[str], _handle=None):
        self.h = C.c_void_p()
        if _handle is not None:
            self.h = _handle
        else:
            _check(load().vsg_udb_open(path.encode(), C.byref(self.h)), "vsg_udb_open")
        self.info = UdbInfo()
        _check(load().vsg_udb_info_get(self.h, C.byref(self.info)), "vsg_udb_info_get")
        self.n = int(self.info.sequences)

    @classmethod
    def _wrap(cls, handle) -> "Udb":
        return cls(None, _handle=handle)

    def write(self, path: str):
        """vsg_udb_write: the file makeudb_usearch would write"""
        _check(load().vsg_udb_write(self.h, path.encode()), "vsg_udb_write")

    def close(self):
        if self.h:
            load().vsg_udb_close(self.h)
            self.h = C.c_void_p()

    def sequences(self):
        """(cat bytes, offsets, lengths) as numpy copies"""
        cat = C.c_char_p(); off = C.POINTER(C.c_int64)(); ln = C.POINTER(C.c_int32)()
        cat_p = C.c_void_p()
        _check(load().vsg_udb_sequences(self.h, C.byref(cat_p), C.byref(off), C.byref(ln)), "vsg_udb_sequences")
        total = int(self.info.nucleotides)
        catb = np.frombuffer(C.string_at(cat_p.value, total), dtype=np.uint8).copy()
        return catb, np.ctypeslib.as_array(off, shape=(self.n,)).copy(), np.ctypeslib.as_array(ln, shape=(self.n,)).copy()

    def header(self, i: int) -> str:
        return load().vsg_udb_header(self.h, C.c_int64(i)).decode()

    def words(self):
        """the stored index: (kmercount[4^k], kmerindex[index_entries]) as numpy copies"""
        kc = C.POINTER(C.c_uint32)(); ki = C.POINTER(C.c_uint32)()
        _check(load().vsg_udb_words(self.h, C.byref(kc), C.byref(ki)), "vsg_udb_words")
        nk = 1 << (2 * int(self.info.wordlength))
        ne = int(self.info.index_entries)
        return (np.ctypeslib.as_array(kc, shape=(nk,)).copy(),
                np.ctypeslib.as_array(ki, shape=(ne,)).copy() if ne > 0 else np.zeros(0, dtype=np.uint32))


class StreamStats(C.Structure):
    _fields_ = [("queries", C.c_int64), ("matched", C.c_int64), ("rows", C.c_int64), ("batches", C.c_int64), ("nucleotides", C.c_int64),
                ("parse_s", C.c_double), ("search_s", C.c_double), ("write_s", C.c_double), ("wall_s", C.c_double)]


def default_search_opts() -> SearchOpts:
    o = SearchOpts()
    load().vsg_search_opts_default(C.byref(o))
    return o


DBMASK = {"none": 0, "soft": 1, "dust": 2}


class MakeudbOpts(C.Structure):
    _fields_ = [("wordlength", C.c_int32), ("dbmask", C.c_int32), ("hardmask", C.c_int32), ("notrunclabels", C.c_int32),
                ("minseqlength", C.c_int64), ("maxseqlength", C.c_int64)]


class MakeudbStats(C.Structure):
    _fields_ = [("sequences", C.c_int64), ("discarded_short", C.c_int64), ("discarded_long", C.c_int64),
                ("stripped", C.c_int64), ("nucleotides", C.c_int64), ("index_entries", C.c_int64),
                ("parse_s", C.c_double), ("device_s", C.c_double), ("write_s", C.c_double), ("wall_s", C.c_double)]


def makeudb_opts(**kw) -> MakeudbOpts:
    """vsg_makeudb_opts_default, then the given fields; dbmask may be "none" / "soft" / "dust" or the number"""
    o = MakeudbOpts()
    load().vsg_makeudb_opts_default(C.byref(o))
    for k, v in kw.items():
        if k == "dbmask" and isinstance(v, str):
            v = DBMASK[v]
        setattr(o, k, int(v))
    return o


CLUSTER_COMMANDS = {"cluster_fast": 0, "cluster_size": 1, "cluster_smallmem": 2, "cluster_unoise": 3}


class ClusterCmdOpts(C.Structure):
    _fields_ = [("command", C.c_int32), ("threads", C.c_int32), ("qmask", C.c_int32), ("hardmask", C.c_int32),
                ("usersort", C.c_int32), ("notrunclabels", C.c_int32), ("sizein", C.c_int32), ("sizeout", C.c_int32),
                ("xsize", C.c_int32), ("clusterout_id", C.c_int32), ("clusterout_sort", C.c_int32), ("fasta_width", C.c_int32),
                ("minseqlength", C.c_int64), ("maxseqlength", C.c_int64), ("minsize", C.c_int64), ("relabel", C.c_char_p)]


class ClusterCmdStats(C.Structure):
    _fields_ = [("sequences", C.c_int64), ("discarded_short", C.c_int64), ("discarded_long", C.c_int64),
                ("discarded_minsize", C.c_int64), ("clusters", C.c_int64), ("singletons", C.c_int64), ("nucleotides", C.c_int64),
                ("pairs", C.c_int64), ("cells", C.c_int64), ("parse_s", C.c_double), ("sort_s", C.c_double),
                ("device_s", C.c_double), ("cigar_s", C.c_double), ("write_s", C.c_double), ("wall_s", C.c_double)]


def cluster_cmd_opts(command: str = "cluster_fast", **kw):
    """vsg_cluster_cmd_opts_default for `command` (a key of CLUSTER_COMMANDS), then the given fields: those of
    vsg_cluster_cmd_opts go there (qmask may be "none" / "soft" / "dust", relabel a str), the rest to the search options.
    Returns (ClusterCmdOpts, SearchOpts)."""
    c, s = ClusterCmdOpts(), SearchOpts()
    load().vsg_cluster_cmd_opts_default(C.c_int(CLUSTER_COMMANDS[command]), C.byref(c), C.byref(s))
    names = {k for k, _ in ClusterCmdOpts._fields_}
    for k, v in kw.items():
        if k == "qmask" and isinstance(v, str):
            v = DBMASK[v]
        if k == "relabel":
            c.relabel = v.encode() if isinstance(v, str) else v
        elif k in names:
            setattr(c, k, int(v))
        else:
            setattr(s, k, v)
    return c, s


class ClusterCmdOutputs(C.Structure):
    _fields_ = [("uc", C.c_char_p), ("centroids", C.c_char_p), ("clusters_prefix", C.c_char_p), ("msaout", C.c_char_p),
                ("consout", C.c_char_p), ("profile", C.c_char_p)]


def _cluster_cmd_paths(uc, centroids, clusters):
    return tuple(p.encode() if p is not None else None for p in (uc, centroids, clusters))


def _cigar_buf(cigars, n):
    """the CIGARs (str, None for S records) back to back, NUL-terminated, and their offsets"""
    cig = [(x or "").encode() + b"\0" for x in cigars]
    cbuf = np.frombuffer(b"".join(cig) + b"\0", dtype=np.uint8)
    coff = np.zeros(max(n, 1), dtype=np.int64)
    if n > 1:
        coff[1:n] = np.cumsum([len(x) for x in cig[:-1]], dtype=np.int64)
    return cbuf, coff


def _records(seqs):
    n = len(seqs)
    cat = np.frombuffer(b"".join(seqs) + b"\0", dtype=np.uint8)
    ln = np.array([len(x) for x in seqs], dtype=np.int32)
    off = np.zeros(n, dtype=np.int64)
    if n > 1:
        off[1:] = np.cumsum(ln[:-1], dtype=np.int64)
    return cat, off, ln


def cluster_msa_write(headers, seqs, abundances, results: np.ndarray, cigars, msa: dict, msaout: Optional[str] = None,
                      consout: Optional[str] = None, profile: Optional[str] = None, command: str = "cluster_fast", **opts):
    """vsg_cluster_msa_write (host only, no device): --msaout, --consout and --profile of records in processing order
    (as cluster_write takes them) from `msa`, a dict of cluster_msa's arrays.  opts as cluster_cmd_opts."""
    c, _ = cluster_cmd_opts(command, **opts)
    n = len(headers)
    res = np.ascontiguousarray(results, dtype=_CLUSTER_DT)
    cat, off, ln = _records(seqs)
    cbuf, coff = _cigar_buf(cigars, n)
    ab = np.ascontiguousarray(abundances, dtype=np.int64)
    ins = np.ascontiguousarray(msa["insertions"], dtype=np.int32)
    first = np.ascontiguousarray(msa["col_first"], dtype=np.int64)
    prof = np.ascontiguousarray(msa["profile"], dtype=np.uint64)
    cons = np.ascontiguousarray(msa["consensus"], dtype=np.uint8)
    _check(load().vsg_cluster_msa_write(C.c_int64(n), _strings(headers) if n else None, cat.ctypes.data_as(C.c_char_p),
                                        _ptr(off, C.c_int64), _ptr(ln, C.c_int32), _ptr(ab, C.c_int64),
                                        res.ctypes.data_as(C.POINTER(ClusterResult)), cbuf.ctypes.data_as(C.c_char_p),
                                        _ptr(coff, C.c_int64), ins.ctypes.data_as(C.POINTER(C.c_int32)),
                                        first.ctypes.data_as(C.POINTER(C.c_int64)), prof.ctypes.data_as(C.POINTER(C.c_uint64)),
                                        cons.ctypes.data_as(C.c_char_p), C.byref(c),
                                        *_cluster_cmd_paths(msaout, consout, profile)), "vsg_cluster_msa_write")


def cluster_write(headers, seqs, abundances, results: np.ndarray, cigars, uc: Optional[str] = None,
                  centroids: Optional[str] = None, clusters: Optional[str] = None, command: str = "cluster_fast", **opts) -> int:
    """vsg_cluster_write (host only, no device): the output files of records in processing order; `seqs` as printed
    (bytes each), `results` a cluster result array (cluster_fast's dtype), `cigars` the CIGAR (str) of each H record
    (anything for S records).  opts as cluster_cmd_opts.  Returns the number of singleton clusters."""
    c, _ = cluster_cmd_opts(command, **opts)
    n = len(headers)
    res = np.ascontiguousarray(results, dtype=_CLUSTER_DT)
    cat, off, ln = _records(seqs)
    cbuf, coff = _cigar_buf(cigars, n)
    ab = np.ascontiguousarray(abundances, dtype=np.int64)
    single = C.c_int64()
    _check(load().vsg_cluster_write(C.c_int64(n), _strings(headers) if n else None, cat.ctypes.data_as(C.c_char_p),
                                    _ptr(off, C.c_int64), _ptr(ln, C.c_int32), _ptr(ab, C.c_int64),
                                    res.ctypes.data_as(C.POINTER(ClusterResult)), cbuf.ctypes.data_as(C.c_char_p),
                                    _ptr(coff, C.c_int64), C.byref(c), *_cluster_cmd_paths(uc, centroids, clusters),
                                    C.byref(single)), "vsg_cluster_write")
    return int(single.value)


class ExactIndex:
    """vsg_exact_index handle"""

    def __init__(self, h):
        self.h = h

    def close(self):
        if self.h:
            load().vsg_exact_index_destroy(self.h)
            self.h = None


class SearchExactOpts(C.Structure):
    _fields_ = [("dbmask", C.c_int32), ("qmask", C.c_int32), ("hardmask", C.c_int32), ("sizein", C.c_int32),
                ("sizeout", C.c_int32), ("xsize", C.c_int32), ("notrunclabels", C.c_int32), ("fasta_width", C.c_int32),
                ("minseqlength", C.c_int64), ("maxseqlength", C.c_int64), ("maxhits", C.c_int64), ("uc_allhits", C.c_int32),
                ("output_no_hits", C.c_int32), ("batch_queries", C.c_int32), ("reserved", C.c_int32)]


SEARCH_EXACT_OUTPUTS = ("blast6out", "uc", "matched", "notmatched", "dbmatched", "dbnotmatched", "otutabout", "mothur_shared_out")


class SearchExactOutputs(C.Structure):
    _fields_ = [(k, C.c_char_p) for k in SEARCH_EXACT_OUTPUTS]


class SearchExactStats(C.Structure):
    _fields_ = [("queries", C.c_int64), ("matched", C.c_int64), ("queries_abundance", C.c_int64), ("matched_abundance", C.c_int64),
                ("db_sequences", C.c_int64), ("db_discarded_short", C.c_int64), ("db_discarded_long", C.c_int64), ("hits", C.c_int64),
                ("parse_s", C.c_double), ("device_s", C.c_double), ("write_s", C.c_double), ("wall_s", C.c_double)]


def search_exact_opts(**kw):
    """vsg_search_exact_opts_default, then the given fields: output paths into SearchExactOutputs, the fields of
    vsg_search_exact_opts there, the rest into the search options.  Returns (SearchExactOpts, SearchOpts, SearchExactOutputs)."""
    e, s, o = SearchExactOpts(), SearchOpts(), SearchExactOutputs()
    load().vsg_search_exact_opts_default(C.byref(e), C.byref(s))
    names = {k for k, _ in SearchExactOpts._fields_}
    for k, v in kw.items():
        if k in SEARCH_EXACT_OUTPUTS:
            setattr(o, k, v.encode() if isinstance(v, str) else v)
        elif k in names:
            setattr(e, k, int(DBMASK[v] if isinstance(v, str) else v))
        else:
            setattr(s, k, v)
    return e, s, o


class UsearchGlobalOpts(C.Structure):
    _fields_ = [("dbmask", C.c_int32), ("qmask", C.c_int32), ("hardmask", C.c_int32), ("sizein", C.c_int32),
                ("sizeout", C.c_int32), ("xsize", C.c_int32), ("notrunclabels", C.c_int32), ("fasta_width", C.c_int32),
                ("minseqlength", C.c_int64), ("maxseqlength", C.c_int64), ("maxhits", C.c_int64), ("uc_allhits", C.c_int32),
                ("output_no_hits", C.c_int32), ("top_hits_only", C.c_int32), ("batch_queries", C.c_int32)]


class UsearchGlobalStats(C.Structure):
    _fields_ = [("queries", C.c_int64), ("matched", C.c_int64), ("queries_abundance", C.c_int64), ("matched_abundance", C.c_int64),
                ("db_sequences", C.c_int64), ("db_discarded_short", C.c_int64), ("db_discarded_long", C.c_int64), ("hits", C.c_int64),
                ("pairs", C.c_int64), ("cells", C.c_int64), ("parse_s", C.c_double), ("device_s", C.c_double),
                ("cigar_s", C.c_double), ("write_s", C.c_double), ("wall_s", C.c_double)]


def usearch_global_opts(**kw):
    """vsg_usearch_global_opts_default, then the given fields: output paths into SearchExactOutputs, the fields of
    vsg_usearch_global_opts there, the rest into the search options.  Returns (UsearchGlobalOpts, SearchOpts,
    SearchExactOutputs)."""
    u, s, o = UsearchGlobalOpts(), SearchOpts(), SearchExactOutputs()
    load().vsg_usearch_global_opts_default(C.byref(u), C.byref(s))
    names = {k for k, _ in UsearchGlobalOpts._fields_}
    for k, v in kw.items():
        if k in SEARCH_EXACT_OUTPUTS:
            setattr(o, k, v.encode() if isinstance(v, str) else v)
        elif k in names:
            setattr(u, k, int(DBMASK[v] if isinstance(v, str) else v))
        else:
            setattr(s, k, v)
    return u, s, o


UCHIME_REF, UCHIME_DENOVO, UCHIME_2_DENOVO, UCHIME_3_DENOVO, CHIMERAS_DENOVO = 0, 1, 2, 3, 4
UCHIME_COMMANDS = {"uchime_ref": UCHIME_REF, "uchime_denovo": UCHIME_DENOVO, "uchime2_denovo": UCHIME_2_DENOVO,
                   "uchime3_denovo": UCHIME_3_DENOVO, "chimeras_denovo": CHIMERAS_DENOVO}
UCHIME_OUTPUTS = ("chimeras", "nonchimeras", "borderline", "uchimeout", "uchimealns")


class UchimeOpts(C.Structure):
    _fields_ = [("command", C.c_int32), ("abskew", C.c_double), ("dn", C.c_double), ("xn", C.c_double), ("mindiv", C.c_double),
                ("minh", C.c_double), ("mindiffs", C.c_int32), ("qmask", C.c_int32), ("dbmask", C.c_int32), ("hardmask", C.c_int32),
                ("self", C.c_int32), ("selfid", C.c_int32), ("strand_both", C.c_int32), ("sizeout", C.c_int32), ("xsize", C.c_int32),
                ("fasta_score", C.c_int32), ("notrunclabels", C.c_int32), ("uchimeout5", C.c_int32), ("fasta_width", C.c_int32),
                ("alignwidth", C.c_int32), ("minseqlength", C.c_int64), ("maxseqlength", C.c_int64), ("batch_queries", C.c_int64),
                ("band_cap", C.c_int64), ("chimeras_parts", C.c_int32), ("chimeras_parents_max", C.c_int32),
                ("chimeras_length_min", C.c_int32), ("chimeras_diff_pct", C.c_double)]


class UchimeOutputs(C.Structure):
    _fields_ = [(k, C.c_char_p) for k in UCHIME_OUTPUTS]


class UchimeStats(C.Structure):
    _fields_ = [(k, C.c_int64) for k in ("queries", "chimeras", "nonchimeras", "borderline", "queries_abundance", "chimeras_abundance",
                                         "nonchimeras_abundance", "borderline_abundance", "db_sequences", "candidates", "part_pairs",
                                         "bands", "recomputed")] + \
               [(k, C.c_double) for k in ("parse_s", "search_s", "align_s", "parents_s", "eval_s", "serial_s", "write_s", "wall_s")]


def uchime_opts(command=UCHIME_REF, **kw):
    """vsg_uchime_opts_default(command), then the given fields: output paths into UchimeOutputs, the rest into
    vsg_uchime_opts.  Returns (UchimeOpts, UchimeOutputs)."""
    o, out = UchimeOpts(), UchimeOutputs()
    command = UCHIME_COMMANDS[command] if isinstance(command, str) else int(command)
    load().vsg_uchime_opts_default(command, C.byref(o))
    names = {k for k, _ in UchimeOpts._fields_}
    for k, v in kw.items():
        if k in UCHIME_OUTPUTS:
            setattr(out, k, v.encode() if isinstance(v, str) else v)
        elif k in names:
            setattr(o, k, DBMASK[v] if isinstance(v, str) else v)
        else:
            raise TypeError(f"uchime: unknown option {k}")
    return o, out


def _packed(seqs):
    """(cat, off, len) arrays of a list of bytes"""
    cat = np.frombuffer(b"".join(seqs) + b"\0", dtype=np.uint8)
    ln = np.array([len(x) for x in seqs], dtype=np.int32)
    off = np.zeros(max(len(seqs), 1), dtype=np.int64)
    if len(seqs) > 1:
        off[1:len(seqs)] = np.cumsum(ln[:-1], dtype=np.int64)
    return cat, off, ln


def search_write(query_headers, query_seqs, query_sizes, hits, db_headers, db_seqs, db_sizes, **kw) -> int:
    """vsg_search_write (host only, no device): the --usearch_global output files of one batch of queries.  hits[i] is
    query i's list of (SearchResult, CIGAR str, or None for none) in search_joinhits order; sequences are bytes as printed; kw as
    usearch_global_command (output paths and vsg_usearch_global_opts fields).  Returns the number of matched queries."""
    u, _, o = usearch_global_opts(**kw)
    nq, ndb = len(query_headers), len(db_headers)
    first = np.zeros(nq + 1, dtype=np.int64)
    first[1:] = np.cumsum([len(h) for h in hits], dtype=np.int64) if nq else []
    flat = [h for hs in hits for h in hs]
    rows = (SearchResult * max(len(flat), 1))(*[r for r, _ in flat])
    cig = [(c or "").encode() + b"\0" for _, c in flat]
    cbuf = np.frombuffer(b"".join(cig) + b"\0", dtype=np.uint8)
    coff = np.zeros(max(len(flat), 1), dtype=np.int64)
    if len(flat) > 1:
        coff[1:len(flat)] = np.cumsum([len(x) for x in cig[:-1]], dtype=np.int64)
    coff[[j for j, (_, c) in enumerate(flat) if c is None]] = -1   # no CIGAR
    qcat, qoff, qlen = _packed(query_seqs)
    dcat, doff, dlen = _packed(db_seqs)
    qs = np.ascontiguousarray(query_sizes, dtype=np.int64)
    ds = np.ascontiguousarray(db_sizes, dtype=np.int64)
    matched = C.c_int64()
    _check(load().vsg_search_write(C.c_int64(nq), _strings(query_headers) if nq else None, qcat.ctypes.data_as(C.c_char_p),
                                   _ptr(qoff, C.c_int64), _ptr(qlen, C.c_int32), _ptr(qs, C.c_int64), rows, _ptr(first, C.c_int64),
                                   cbuf.ctypes.data_as(C.c_char_p), _ptr(coff, C.c_int64), C.c_int64(ndb),
                                   _strings(db_headers) if ndb else None, dcat.ctypes.data_as(C.c_char_p), _ptr(doff, C.c_int64),
                                   _ptr(dlen, C.c_int32), _ptr(ds, C.c_int64), C.byref(u), C.byref(o), C.byref(matched)),
           "vsg_search_write")
    return int(matched.value)
