"""Throughput of vsg_cluster_fast with --strand both against plus strand only (not the bench contract).

The reads are those of bench.py's configs[2] cluster leg: 100 000 amplicon reads of 300 nt (1 % divergence, Zipf-ish
root choice), sorted by length, DUST on the device, --id 0.97, round size = the host's core count.  Three arms run in
one process, alternating, three times each:
  plus       plus strand only;
  both       --strand both on the same reads;
  both_rc3   --strand both on the same reads with every third read reverse-complemented.
A run is timed end to end as the bench leg is: upload, DUST, clustering and the result table.  Each run prints one
JSON line: reads/s, pairs and DP cells handed to the aligner, clusters, the driver's phase times (VSG_TRACE) and the
card it ran on (a read-only nvidia-smi query: name, power limit, maximum SM clock).  With oracle/_ref/vsearch present,
the reference's `--cluster_fast --strand both --threads T` is timed once per read set for context (--no-reference skips
it).  Nothing is written inside the repository.

    python tools/perf_cluster_strands.py [--reads 100000] [--reps 3] [--no-reference]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("VSG_TRACE", "1")   # the driver prints its phase times to stderr; read once, at the first call

import numpy as np  # noqa: E402

from vsearch_b200 import lib as vlib, synth  # noqa: E402

COMP = bytes.maketrans(b"ACGTacgt", b"TGCAtgca")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (x.strip() for x in out[0].split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the numbers are reported without the card rather than not at all
        return {"error": repr(e)[:200]}


def make_reads(n):
    """bench.py cluster_workload's reads (rank 0) and their Database::sortbylength order"""
    rng = np.random.default_rng([3, 0])
    nroots = max(50, n // 200)
    roots = synth.random_seqs(rng, nroots, 300)
    w = 1.0 / np.arange(1, nroots + 1); w /= w.sum()
    reads = synth.mutate_batch(rng, roots[rng.choice(nroots, size=n, p=w)], 0.01)
    seqs = [reads.seq(i) for i in range(n)]
    order = np.lexsort((np.arange(n), -reads.lens.astype(np.int64)))
    return seqs, order


class StderrCapture:
    """what the library writes to file descriptor 2 while the block runs"""

    def __enter__(self):
        sys.stderr.flush()
        self.f = tempfile.TemporaryFile()
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        return self

    def __exit__(self, *exc):
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read().decode(errors="replace")
        self.f.close()
        sys.stderr.write(self.text)


def phases(text):
    m = re.search(r"rank (\d+) ms, candidate groups (\d+) ms, speculative extras (\d+) ms, serial pass (\d+) ms, "
                  r"index append (\d+) ms", text)
    if m is None:
        return None
    return dict(zip(("rank_ms", "groups_ms", "spec_ms", "serial_ms", "append_ms"), (int(x) for x in m.groups())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--round", type=int, default=0, help="round size = the reference's --threads (0 = host cores)")
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    n = args.reads
    T = args.round if args.round > 0 else (os.cpu_count() or 1)
    seqs, order = make_reads(n)
    rc3 = [s.translate(COMP)[::-1] if i % 3 == 0 else s for i, s in enumerate(seqs)]
    plus = synth.SeqSet([seqs[i] for i in order])
    # reverse complementing keeps the lengths, so the sorted order is the same
    sets = {"plus": plus, "both": plus, "both_rc3": synth.SeqSet([rc3[i] for i in order])}
    ctx = vlib.Context(0)
    card = gpu_info()
    for rep in range(args.reps):
        for arm in ("plus", "both", "both_rc3"):
            o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxrejects = 8
            o.strand_both = 0 if arm == "plus" else 1
            with StderrCapture() as cap:
                ctx.sync()
                t0 = time.perf_counter()
                ss = ctx.seqset(sets[arm])
                ss.dust()
                res, ncl, work = vlib.cluster_fast(ctx, ss, o, T)
                ss.close()
                dt = time.perf_counter() - t0
            minus = int(((res["centroid"] >= 0) & (res["strand"] == 1)).sum())
            print(json.dumps({"arm": arm, "rep": rep, "reads": n, "round": T, "reads_per_s": n / dt, "seconds": dt,
                              "pairs": int(work[0]), "cells": int(work[1]), "clusters": ncl, "minus_hits": minus,
                              "phases": phases(cap.text), "gpu": card}), flush=True)
    ctx.close()
    stock = os.path.join(ROOT, "oracle", "_ref", "vsearch")
    if args.no_reference or not os.path.exists(stock):
        return
    with tempfile.TemporaryDirectory() as d:
        for arm, reads in (("both", seqs), ("both_rc3", rc3)):
            fa = os.path.join(d, "reads.fasta"); uc = os.path.join(d, "out.uc")
            with open(fa, "wb") as f:
                for i, s in enumerate(reads):
                    f.write(b">a%08d\n" % i + s + b"\n")
            t0 = time.perf_counter()
            p = subprocess.run([stock, "--cluster_fast", fa, "--id", "0.97", "--strand", "both", "--threads", str(T), "--uc", uc,
                                "--quiet"], capture_output=True, text=True)
            dt = time.perf_counter() - t0
            ncl = sum(1 for line in open(uc) if line.startswith("S")) if p.returncode == 0 else None
            print(json.dumps({"arm": "reference_" + arm, "reads": n, "threads": T, "reads_per_s": n / dt, "seconds": dt,
                              "clusters": ncl, "returncode": p.returncode, "cpu_cores": os.cpu_count(),
                              "note": "CLI wall time, FASTA read and uc write included"}), flush=True)


if __name__ == "__main__":
    main()
