"""Time vsg_sintax_stream on a 16S-shaped set and the reference CLI on the same files.

About 20 000 x 1 450-nt references (a tree of mutations with tax= headers) and 100 000 x 250-nt mutated windows as
queries, plus strand only and both strands.  The reference runs `--sintax` on the host's threads (--threads = CPU count)
over the first --ref-queries queries; the rows of both, sorted by query, must agree on those.  Prints one JSON line per
strand mode: queries/s of the device stream and of the reference, the device time of the counting kernel
(vsg_profile.rank_ms of a vsg_sintax call over all queries), the GPU name and its power limit.

    python tools/perf_sintax.py [--refs 20000] [--queries 100000] [--ref-queries 100000] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vsearch_b200 import lib, synth  # noqa: E402

STOCK = os.path.join(ROOT, "oracle", "_ref", "vsearch")


def make_set(n_ref, n_q, seed=16):
    rng = np.random.default_rng(seed)
    roots = synth.random_seqs(rng, 40, 1450)
    heads, seqs = [], []
    for i in range(n_ref):
        g = i % 400
        s = synth.mutate(rng, synth.mutate(rng, roots[g % 40], 0.06) if i < 400 else seqs[g], 0.02 if i >= 400 else 0.0)
        seqs.append(s)
        heads.append(f"r{i};tax=d:D{g % 2},p:P{g % 8},c:C{g % 20},o:O{g % 40},f:F{g % 100},g:G{g},s:S{i % 1200};")
    seqs = [s.tobytes() for s in seqs]
    src = rng.integers(0, n_ref, size=n_q)
    qs = []
    for j in range(n_q):
        s = seqs[src[j]]
        p = int(rng.integers(0, len(s) - 250))
        w = synth.mutate(rng, np.frombuffer(s[p:p + 250], dtype=np.uint8), 0.03).tobytes()
        qs.append(synth.revcomp(w) if j % 4 == 0 else w)
    return heads, seqs, [f"q{j}" for j in range(n_q)], qs


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--refs", type=int, default=20000)
    ap.add_argument("--queries", type=int, default=100000)
    ap.add_argument("--ref-queries", type=int, default=100000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    heads, seqs, qh, qs = make_set(a.refs, a.queries)
    tmp = tempfile.mkdtemp()
    dbf, qf, qf_ref = (os.path.join(tmp, x) for x in ("db.fa", "q.fa", "qref.fa"))
    synth.write_records(dbf, heads, seqs)
    synth.write_records(qf, qh, qs)
    synth.write_records(qf_ref, qh[:a.ref_queries], qs[:a.ref_queries])
    g = lib.Group([0], synth.SeqSet(seqs), wordlength=8, mask_lower=1)
    ctx = lib.Context(0)
    db = ctx.seqset(synth.SeqSet(seqs))
    ix = ctx.index(db, wordlength=8, mask_lower=1)
    qset = ctx.seqset(synth.SeqSet(qs))
    lines = []
    for both in (0, 1):
        out = os.path.join(tmp, f"gpu{both}.tsv")
        g.sintax_stream(heads, qf, out, 42, strand_both=both)             # warm-up
        t0 = time.perf_counter()
        st = g.sintax_stream(heads, qf, out, 42, strand_both=both)
        dt = time.perf_counter() - t0
        ctx.sintax(ix, qset, 0, len(qs), 42, strand_both=both)           # warm-up
        ctx.profile_reset()
        ctx.sintax(ix, qset, 0, len(qs), 42, strand_both=both)
        count_ms = float(ctx.profile().rank_ms)
        rec = {"strand_both": both, "queries": len(qs), "refs": len(seqs), "gpu_queries_per_s": len(qs) / dt,
               "gpu_stream_s": dt, "count_kernel_ms": count_ms, "stream_stats": st, "gpu": gpu_info()}
        if os.path.exists(STOCK) and a.ref_queries > 0:
            rout = os.path.join(tmp, f"ref{both}.tsv")
            args = [STOCK, "--sintax", qf_ref, "--db", dbf, "--tabbedout", rout, "--randseed", "42", "--quiet",
                    "--threads", str(os.cpu_count())] + (["--strand", "both"] if both else [])
            t0 = time.perf_counter()
            subprocess.run(args, check=True)
            rdt = time.perf_counter() - t0
            key = lambda r: int(r.split("\t", 1)[0][1:])   # noqa: E731
            want = sorted(open(rout).read().splitlines(), key=key)
            got = open(out).read().splitlines()[:a.ref_queries]
            rec.update({"ref_queries": a.ref_queries, "ref_threads": os.cpu_count(), "ref_queries_per_s": a.ref_queries / rdt,
                        "ref_s": rdt, "rows_equal": want == got})
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "perf_sintax.jsonl"), "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
