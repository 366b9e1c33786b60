"""Measure chimera detection on one GPU against the reference CLI, with the GPU's name and power limit read in the same run.

  --uchime3_denovo: `--denovo N` unique 250-nt sequences (default 100 000) with power-law abundances, about 15 %
                    two-segment chimeras of more abundant sequences; the reference runs it with --threads 1 (what it
                    runs de novo anyway);
  --uchime_ref:     `--ref N` queries (default 100 000) against `--refs M` references of 1 450 nt (default 20 000); the
                    reference runs it on every host core.

For each: the wall time and the seconds per stage of vsg_uchime_command, the bands and the queries the serial pass
recomputed (de novo), the reference's wall time, whether every output file is identical, and whether every file holds
the same lines (the reference's files are in completion order when it runs several threads).  Prints one JSON line.
`--no-reference` skips the reference runs."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vsearch_b200 import lib as vlib  # noqa: E402

STOCK = os.path.join(ROOT, "oracle", "_ref", "vsearch")
OUTPUTS = ("chimeras", "nonchimeras", "borderline", "uchimeout", "uchimealns")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _seqs(rng, n, length):
    return rng.integers(0, 4, size=(n, length), dtype=np.uint8)


def _mut(rng, a, rate):
    b = a.copy()
    m = rng.random(b.shape) < rate
    b[m] = (b[m] + rng.integers(1, 4, size=int(m.sum()), dtype=np.uint8)) % 4
    return b


def _write(path, labels, arr):
    lut = np.frombuffer(b"ACGT", dtype=np.uint8)
    with open(path, "w") as f:
        for lab, row in zip(labels, arr):
            f.write(">" + lab + "\n" + lut[row].tobytes().decode() + "\n")


def denovo_input(d, n, seed=1):
    """n sequences of 250 nt: families of roots with 1-3 % diverged members, abundances from a power law sorted with
    them, and 15 % chimeras of two more abundant sequences at low abundance"""
    rng = np.random.default_rng(seed)
    nroot = max(1, n // 50)
    roots = _seqs(rng, nroot, 250)
    nchim = int(0.15 * n)
    nclean = n - nchim
    clean = _mut(rng, roots[rng.integers(0, nroot, size=nclean)], 0.02)
    size = np.sort((rng.pareto(1.0, size=nclean) * 2 + 1).astype(np.int64))[::-1]
    a = rng.integers(0, max(1, nclean // 10), size=nchim)
    b = rng.integers(0, max(1, nclean // 10), size=nchim)
    cut = rng.integers(60, 190, size=nchim)
    chim = clean[a].copy()
    for i in range(nchim):
        chim[i, cut[i]:] = clean[b[i], cut[i]:]
    arr = np.concatenate([clean, chim])
    sizes = np.concatenate([size, np.ones(nchim, dtype=np.int64)])
    labels = [f"u{i};size={int(s)}" for i, s in enumerate(sizes)]
    p = os.path.join(d, "denovo.fasta")
    _write(p, labels, arr)
    return p


def ref_inputs(d, nq, nref, seed=2):
    rng = np.random.default_rng(seed)
    roots = _seqs(rng, max(1, nref // 20), 1450)
    refs = _mut(rng, roots[rng.integers(0, roots.shape[0], size=nref)], 0.05)
    qsrc = refs[rng.integers(0, nref, size=nq)]
    q = _mut(rng, qsrc, 0.005)
    k = nq // 5
    other = refs[rng.integers(0, nref, size=k)]
    cut = rng.integers(300, 1150, size=k)
    for i in range(k):
        q[i, cut[i]:] = other[i, cut[i]:]
    pq, pr = os.path.join(d, "queries.fasta"), os.path.join(d, "refs.fasta")
    _write(pq, [f"q{i};size=1" for i in range(nq)], q)
    _write(pr, [f"r{i};size=1" for i in range(nref)], refs)
    return pq, pr


def digests(paths):
    return {k: hashlib.sha256(open(p, "rb").read()).hexdigest() for k, p in paths.items()}


def run(ctx, d, tag, inp, db, command, threads, reference):
    mine = {k: os.path.join(d, f"{tag}.mine.{k}") for k in OUTPUTS}
    t = time.perf_counter()
    st = ctx.uchime(inp, db, command=command, **mine)
    out = {"wall_s": round(time.perf_counter() - t, 3), "stats": st}
    if reference and os.path.exists(STOCK):
        ref = {k: os.path.join(d, f"{tag}.ref.{k}") for k in OUTPUTS}
        cmd = [STOCK, f"--{command}", inp, "--threads", str(threads), "--quiet"] + (["--db", db] if db else [])
        for k, p in ref.items():
            cmd += [f"--{k}", p]
        t = time.perf_counter()
        subprocess.run(cmd, check=True)
        out["reference_wall_s"] = round(time.perf_counter() - t, 3)
        out["reference_threads"] = threads
        out["identical"] = digests(mine) == digests(ref)
        # several reference threads write in completion order: compare the files' lines as multisets too
        out["same_lines"] = all(sorted(open(mine[k], "rb").read().splitlines()) == sorted(open(ref[k], "rb").read().splitlines())
                                for k in OUTPUTS)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--denovo", type=int, default=100000)
    ap.add_argument("--ref", type=int, default=100000)
    ap.add_argument("--refs", type=int, default=20000)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    res = {"gpu": gpu_info()}
    ctx = vlib.Context(0)
    with tempfile.TemporaryDirectory() as d:
        if a.denovo > 0:
            inp = denovo_input(d, a.denovo)
            res["uchime3_denovo"] = dict(run(ctx, d, "dn", inp, None, "uchime3_denovo", 1, not a.no_reference), sequences=a.denovo)
        if a.ref > 0:
            q, r = ref_inputs(d, a.ref, a.refs)
            res["uchime_ref"] = dict(run(ctx, d, "ref", q, r, "uchime_ref", os.cpu_count(), not a.no_reference),
                                     queries=a.ref, references=a.refs)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
