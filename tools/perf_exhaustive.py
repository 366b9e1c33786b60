"""Exhaustive search (--maxaccepts 0 --maxrejects 0: every candidate aligned) on a database shaped like a 16S
collection: one ancestor, families at up to 15 % divergence from it, members close to their family, and query windows
cut from mutated members.  Prints one JSON line: queries/s, GCUPS over the cells the reference's driver hands to its
aligner (work[1]), the ranker's share of the time (its kernels, sort and cut, as device time), the candidate volume,
and the card it ran on.

    python tools/perf_exhaustive.py [--targets 20000] [--length 1450] [--families 200] [--queries 4096] [--qlen 250]
    python tools/perf_exhaustive.py --impl reference --ref-queries 64     # the reference's search_batch, all host threads
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
from vsearch_b200 import lib as vlib, synth  # noqa: E402


def data(n_targets, length, n_fam, n_q, qlen, seed=11):
    rng = np.random.default_rng(seed)
    root = synth.random_seqs(rng, 1, length)[0]
    fams = [synth.mutate(rng, root, float(rng.uniform(0.02, 0.15))) for _ in range(n_fam)]
    seqs = [synth.mutate(rng, fams[i % n_fam], 0.02).tobytes() for i in range(n_targets)]
    qs = []
    for i in range(n_q):
        m = synth.mutate(rng, fams[int(rng.integers(0, n_fam))], 0.03)
        a = int(rng.integers(0, max(1, m.shape[0] - qlen)))
        qs.append(m[a: a + qlen].tobytes())
    return synth.SeqSet(seqs), synth.SeqSet(qs)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", type=int, default=20000)
    ap.add_argument("--length", type=int, default=1450)
    ap.add_argument("--families", type=int, default=200)
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--qlen", type=int, default=250)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--impl", choices=["gpu", "reference"], default="gpu")
    ap.add_argument("--ref-queries", type=int, default=64, help="query prefix the reference searches")
    a = ap.parse_args()
    dbs, qss = data(a.targets, a.length, a.families, a.queries, a.qlen)
    if a.impl == "reference":
        import checkers
        r = checkers.RefDb(dbs, k=8, id=0.97, maxaccepts=len(dbs), maxrejects=len(dbs), dust=0)
        sub = synth.SeqSet([qss.seq(i) for i in range(a.ref_queries)])
        threads = os.cpu_count() or 1
        checkers.ref().vsref_work_reset()
        first = np.zeros(len(sub), dtype=np.int32)
        t0 = time.perf_counter()
        checkers.ref().vsref_db_search_batch(checkers.C.c_void_p(r.h), checkers.C.c_int(len(sub)), checkers._p(sub.cat, checkers.C.c_char),
                                             checkers._p(sub.offs, checkers.C.c_int64), checkers._p(sub.lens, checkers.C.c_int),
                                             checkers.C.c_int(threads), checkers._p(first, checkers.C.c_int))
        dt = time.perf_counter() - t0
        pairs, cells, calls = (checkers.C.c_longlong() for _ in range(3))
        checkers.ref().vsref_work_get(checkers.C.byref(pairs), checkers.C.byref(cells), checkers.C.byref(calls))
        r.close()
        print(json.dumps({"impl": "reference", "threads": threads, "queries": len(sub), "seconds": round(dt, 3),
                          "queries_per_s": round(len(sub) / dt, 2), "pairs": pairs.value, "cells": cells.value,
                          "gcups": round(cells.value / dt / 1e9, 2)}))
        return
    ctx = vlib.Context(0)
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, 8, 0)
    o = vlib.default_search_opts(); o.id = 0.97; o.maxaccepts = 0; o.maxrejects = 0
    # an untimed call sizes the row buffer (and warms every shape up); each timed call is then one search
    _, first, _ = ctx.search_hits(ix, db, qs, 0, len(qss), o)
    cap = int(first[-1])
    best = None
    for _ in range(a.repeats):
        ctx.profile_reset()
        t0 = time.perf_counter()
        hits, first, work = ctx.search_hits(ix, db, qs, 0, len(qss), o, cap=cap)
        dt = time.perf_counter() - t0
        pr = ctx.profile()
        if best is None or dt < best[0]:
            best = (dt, work.copy(), pr.rank_ms, pr.fwd_ms, pr.traceback_ms, int(first[-1]))
    dt, work, rank_ms, fwd_ms, tb_ms, rows = best
    print(json.dumps({"impl": "gpu", "card": card(), "targets": len(dbs), "queries": len(qss), "seconds": round(dt, 3),
                      "queries_per_s": round(len(qss) / dt, 1), "candidates": int(work[0]), "cells": int(work[1]),
                      "gcups": round(work[1] / dt / 1e9, 1), "rank_ms": round(rank_ms, 1),
                      "rank_share": round(rank_ms / 1e3 / dt, 3), "fwd_ms": round(fwd_ms, 1), "tb_ms": round(tb_ms, 1),
                      "rows": rows}))
    ix.close(); db.close(); qs.close(); ctx.close()


if __name__ == "__main__":
    main()
