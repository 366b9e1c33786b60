"""A/B timing of the k-mer ranker (vsg_rank) on the shapes that take each of its paths, with the outputs kept so that
two builds can be compared byte for byte.  The benchmark only reaches the running-threshold path (250-nt queries,
wordlength 8, tophits 41); the other shapes here reach the fixed-threshold scan (1 500-nt queries), the k-mers
de-duplicated in HBM (3 000 nt), the sparse index (wordlength 12) and the unbounded ranker (tophits = every target).

Each shape is ranked once to warm up and then --repeats times; the time is the ranker's device time as the context's
profile reports it (vsg_profile.rank_ms), and the output of every repeat must equal the first.  Prints one JSON line per
shape (median / min / max rank_ms and a digest of the outputs) and one with the card.  --out DIR also writes each
shape's outputs there as <shape>.npz.  Run two builds by pointing VSG_LIB at one of them:

    python tools/perf_rank.py [--shapes c2,c4,...] [--repeats 5] [--out DIR]
    VSG_LIB=/path/to/other/libvsg.so python tools/perf_rank.py ...
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
from vsearch_b200 import lib as vlib, synth  # noqa: E402
import perf_exhaustive  # noqa: E402

MINWORDMATCHES = 12


def card():
    """name, power limit and maximum SM clock of device 0 (a read-only query)"""
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError:
        return "unknown"


def c2_db():
    return synth.config2_db(100_000, 1500, 2024)


def long_queries(dbm, n, seed=5):
    """n queries of two database sequences end to end, 5 % mutated (3 000 nt for the C2 database)"""
    rng = np.random.default_rng(seed)
    src = rng.integers(0, dbm.shape[0], size=(n, 2))
    return synth.mutate_batch(rng, np.concatenate([dbm[src[:, 0]], dbm[src[:, 1]]], axis=1), 0.05)


# shape -> (database, wordlength, queries, tophits); the database entry names a builder so that shapes share it
SHAPES = {
    "c2": ("c2", 8, lambda dbm: synth.config2_query_batch(dbm, 32768, q_len=250, batch=1)[0], 41),
    "c4": ("c4", 8, lambda dbm: synth.config2_query_batch(dbm, 16384, q_len=150, batch=1)[0], 41),
    "q1500": ("c2", 8, lambda dbm: synth.config2_query_batch(dbm, 4096, q_len=1500, batch=2)[0], 41),
    "q3000": ("c2", 8, lambda dbm: long_queries(dbm, 2048), 41),
    "c2k12": ("c2", 12, lambda dbm: synth.config2_query_batch(dbm, 32768, q_len=250, batch=1)[0], 41),
    "lists16s": ("16s", 8, None, None),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the outputs of every shape (<shape>.npz)")
    ap.add_argument("--lists-queries", type=int, default=1024, help="queries of the 16S-shaped set for lists16s")
    a = ap.parse_args()
    if a.repeats < 1:
        ap.error("--repeats must be at least 1")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    ctx = vlib.Context(0)
    print(json.dumps({"card": card(), "lib": vlib.LIB_PATH}), flush=True)
    dbs = {}   # database name -> (matrix or None, SeqSetHandle, {wordlength: IndexHandle}, 16S queries or None)

    def database(name, k):
        if name not in dbs:
            if name == "16s":
                d, q = perf_exhaustive.data(20000, 1450, 200, a.lists_queries, 250)
                dbs[name] = (None, ctx.seqset(d), {}, q)
            else:
                m = c2_db() if name == "c2" else synth.config2_db(1_000_000, 1200, 4048)
                dbs[name] = (m, ctx.seqset(synth.SeqSet.from_matrix(m)), {}, None)
        m, db, ixs, q16 = dbs[name]
        if k not in ixs:
            ixs[k] = ctx.index(db, k, 0)
        return m, db, ixs[k], q16

    for shape in a.shapes.split(","):
        dbname, k, make_queries, tophits = SHAPES[shape]
        m, db, ix, q16 = database(dbname, k)
        qss = q16 if shape == "lists16s" else make_queries(m)
        if tophits is None:
            tophits = db.n   # every target: the unbounded ranker (rank_lists)
        qs = ctx.seqset(qss)
        nq = len(qss)
        ref = ctx.rank(ix, qs, 0, nq, MINWORDMATCHES, tophits)   # warm-up, and the output every repeat must match
        times = []
        for _ in range(a.repeats):
            ctx.profile_reset()
            got = ctx.rank(ix, qs, 0, nq, MINWORDMATCHES, tophits)
            times.append(ctx.profile().rank_ms)
            if not all(np.array_equal(x, y) for x, y in zip(got, ref)):
                raise SystemExit(f"{shape}: a repeat's output differs from the first run's")
        seqno, count, nc = ref
        h = hashlib.sha256()
        for x in (seqno, count, nc):
            h.update(np.ascontiguousarray(x).tobytes())
        if a.out:
            np.savez_compressed(os.path.join(a.out, f"{shape}.npz"), seqno=seqno, count=count, ncand=nc)
        print(json.dumps({"shape": shape, "targets": db.n, "wordlength": k, "queries": nq, "tophits": tophits,
                          "candidates": int(nc.sum()), "rank_ms_median": round(statistics.median(times), 3),
                          "rank_ms_min": round(min(times), 3), "rank_ms_max": round(max(times), 3),
                          "repeats": a.repeats, "sha256": h.hexdigest()}), flush=True)
        qs.close()
    for _, db, ixs, _ in dbs.values():
        for ix in ixs.values():
            ix.close()
        db.close()
    ctx.close()


if __name__ == "__main__":
    main()
