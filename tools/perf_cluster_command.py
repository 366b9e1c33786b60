"""Timing of the clustering command (vsg_cluster_command, --cluster_fast) on one GPU, against vsg_cluster_fast alone and the
reference CLI.

Workload: bench.py's configs[2]-shaped reads (300-nt amplicons, 1 % divergence, Zipf-ish root choice, 200 000 reads),
--id 0.97, --threads = the host's core count, --uc out.  Reported, in one run:
  - the card's name and power limit (nvidia-smi);
  - vsg_cluster_command's wall time and its stages (parse, sort, device, CIGAR, write);
  - vsg_cluster_fast alone on the pre-sorted set (upload + DUST + clustering, what bench.py --workload cluster times);
  - the reference CLI's wall time on the same FASTA, when oracle/_ref/vsearch is built (--ref);
  - whether the two --uc files are identical (sha256).
Inputs and outputs go to a temporary directory (or --dir) and are removed.

    python tools/perf_cluster_command.py [--reads 200000] [--runs 3] [--ref] [--out perf_cluster_command.json]
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vsearch_b200 import lib as vlib  # noqa: E402
from vsearch_b200 import synth  # noqa: E402

STOCK = os.path.join(ROOT, "oracle", "_ref", "vsearch")


def configs2_reads(n, seed=3):
    """bench.py's cluster workload reads (rank 0): roots of 300 nt, 1 % divergence, Zipf-ish root choice"""
    rng = np.random.default_rng([seed, 0])
    nroots = max(50, n // 200)
    roots = synth.random_seqs(rng, nroots, 300)
    w = 1.0 / np.arange(1, nroots + 1)
    w /= w.sum()
    return synth.mutate_batch(rng, roots[rng.choice(nroots, size=n, p=w)], 0.01)


def digest(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=200_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--threads", type=int, default=0, help="round size (0: the host's core count)")
    ap.add_argument("--ref", action="store_true", help="also time the reference CLI (oracle/_ref/vsearch)")
    ap.add_argument("--dir", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    T = a.threads if a.threads > 0 else (os.cpu_count() or 1)
    gpu = card()
    print(f"[card] {gpu}; host cores {os.cpu_count()}, --threads {T}", flush=True)
    d = tempfile.mkdtemp(dir=a.dir)
    out = {"card": gpu, "reads": a.reads, "threads": T, "command": [], "cluster_fast": []}
    try:
        reads = configs2_reads(a.reads)
        labels = [f"a{i:08d}" for i in range(a.reads)]
        fa = os.path.join(d, "reads.fasta")
        with open(fa, "wb") as f:
            f.write(b"".join(b">" + labels[i].encode() + b"\n" + reads.seq(i) + b"\n" for i in range(a.reads)))
        ctx = vlib.Context(0)
        uc = os.path.join(d, "gpu.uc")
        for r in range(a.runs):
            st = ctx.cluster_command(fa, uc=uc, id=0.97, threads=T)
            out["command"].append(st)
            print(f"[command run {r}] wall {st['wall_s']:.2f} s = parse {st['parse_s']:.2f} + sort {st['sort_s']:.2f} + device "
                  f"{st['device_s']:.2f} + cigar {st['cigar_s']:.2f} + write {st['write_s']:.2f}; {st['clusters']} clusters, "
                  f"{st['pairs']} pairs", flush=True)
        # vsg_cluster_fast alone on the pre-sorted set: what bench.py --workload cluster times
        order = np.lexsort((np.arange(a.reads), -reads.lens.astype(np.int64)))
        sorted_host = synth.SeqSet([reads.seq(int(i)) for i in order])
        o = vlib.default_search_opts()
        o.id = 0.97
        o.mask_lower = 1
        o.maxrejects = 8
        for r in range(a.runs):
            t0 = time.perf_counter()
            ss = ctx.seqset(sorted_host)
            ss.dust()
            res, ncl, _ = vlib.cluster_fast(ctx, ss, o, T)
            ss.close()
            dt = time.perf_counter() - t0
            out["cluster_fast"].append({"wall_s": dt, "clusters": ncl})
            print(f"[cluster_fast alone run {r}] {dt:.2f} s, {ncl} clusters", flush=True)
        ctx.close()
        out["uc_sha256"] = digest(uc)
        if a.ref and os.path.exists(STOCK):
            ref_uc = os.path.join(d, "ref.uc")
            t0 = time.perf_counter()
            subprocess.run([STOCK, "--cluster_fast", fa, "--id", "0.97", "--threads", str(T), "--uc", ref_uc, "--quiet"], check=True)
            wall = time.perf_counter() - t0
            out["reference"] = {"wall_s": wall, "uc_identical": digest(ref_uc) == out["uc_sha256"]}
            print(f"[reference CLI] wall {wall:.1f} s, --uc identical: {out['reference']['uc_identical']}", flush=True)
        elif a.ref:
            print("[reference CLI] not measured: oracle/_ref/vsearch is not built", flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
