"""Throughput of exhaustive greedy clustering, vsg_cluster_fast with --maxaccepts 0 --maxrejects 0 (not the bench
contract).

The reads: 20 000 amplicon reads of 300 nt from 100 roots (Zipf-ish root choice) at 1-5 % divergence, sorted by length,
DUST on the device, --id 0.97, round size 16.  Both limits are clamped to the number of reads, so every centroid that
shares enough k-mers with a read is a candidate and each round is ranked into lists of any length.  A run is timed end
to end: upload, DUST, clustering and the result table.  Each run prints one JSON line: reads/s, pairs and DP cells
handed to the aligner, GCUPS over those cells, clusters, the driver's phase times (VSG_TRACE) with the ranker's share,
and the card it ran on (a read-only nvidia-smi query: name, power limit, maximum SM clock).  With oracle/_ref/vsearch
present, the reference's `--cluster_fast --maxaccepts 0 --maxrejects 0 --threads <host cores>` is timed once on a
stated prefix of the same sorted reads (--no-reference skips it).  Nothing is written inside the repository.

    python tools/perf_cluster_exhaustive.py [--reads 20000] [--round 16] [--reps 3] [--ref-reads 2000] [--no-reference]
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (x.strip() for x in out[0].split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the numbers are reported without the card rather than not at all
        return {"error": repr(e)[:200]}


def make_reads(n, nroots=100, divs=(0.01, 0.02, 0.03, 0.05)):
    """the reads in Database::sortbylength order (length descending, then input order)"""
    rng = np.random.default_rng(20)
    roots = synth.random_seqs(rng, nroots, 300)
    w = 1.0 / np.arange(1, nroots + 1); w /= w.sum()
    pick = rng.choice(nroots, size=n, p=w)
    seqs = []
    for i in range(n):
        m = synth.mutate(rng, roots[int(pick[i])], float(divs[int(rng.integers(0, len(divs)))]))
        a = int(rng.integers(0, 6)); b = int(rng.integers(0, 6))
        seqs.append(m[a: m.shape[0] - b].tobytes())
    order = sorted(range(n), key=lambda i: (-len(seqs[i]), i))
    return [seqs[i] for i in order]


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
    p = dict(zip(("rank_ms", "groups_ms", "spec_ms", "serial_ms", "append_ms"), (int(x) for x in m.groups())))
    p["rank_share"] = p["rank_ms"] / max(1, sum(p.values()))
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000)
    ap.add_argument("--round", type=int, default=16, help="round size = the reference's --threads")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-reads", type=int, default=2_000, help="prefix of the sorted reads the reference CLI clusters")
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    n, T = args.reads, args.round
    seqs = make_reads(n)
    reads = synth.SeqSet(seqs)
    ctx = vlib.Context(0)
    card = gpu_info()
    o = vlib.default_search_opts(); o.id = 0.97; o.mask_lower = 1; o.maxaccepts = 0; o.maxrejects = 0
    for rep in range(args.reps):
        with StderrCapture() as cap:
            ctx.sync()
            t0 = time.perf_counter()
            ss = ctx.seqset(reads)
            ss.dust()
            res, ncl, work = vlib.cluster_fast(ctx, ss, o, T)
            ss.close()
            dt = time.perf_counter() - t0
        print(json.dumps({"arm": "vsg_cluster_fast", "rep": rep, "reads": n, "round": T, "reads_per_s": n / dt, "seconds": dt,
                          "pairs": int(work[0]), "cells": int(work[1]), "gcups": int(work[1]) / dt / 1e9, "clusters": ncl,
                          "hits": int((res["centroid"] >= 0).sum()), "phases": phases(cap.text), "gpu": card}), flush=True)
    ctx.close()
    stock = os.path.join(ROOT, "oracle", "_ref", "vsearch")
    if args.no_reference or not os.path.exists(stock):
        return
    m = min(args.ref_reads, n)
    threads = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as d:
        fa = os.path.join(d, "reads.fasta"); uc = os.path.join(d, "out.uc")
        with open(fa, "wb") as f:
            for i in range(m):
                f.write(b">a%08d\n" % i + seqs[i] + b"\n")
        t0 = time.perf_counter()
        p = subprocess.run([stock, "--cluster_fast", fa, "--id", "0.97", "--maxaccepts", "0", "--maxrejects", "0",
                            "--threads", str(threads), "--uc", uc, "--quiet"], capture_output=True, text=True)
        dt = time.perf_counter() - t0
        ncl = sum(1 for line in open(uc) if line.startswith("S")) if p.returncode == 0 else None
        print(json.dumps({"arm": "reference_cli", "reads": m, "threads": threads, "reads_per_s": m / dt, "seconds": dt,
                          "clusters": ncl, "returncode": p.returncode, "cpu_cores": os.cpu_count(),
                          "note": f"CLI wall time on the first {m} sorted reads, FASTA read and uc write included"}), flush=True)


if __name__ == "__main__":
    main()
