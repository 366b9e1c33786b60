"""Throughput of the --usearch_global command (vsg_usearch_global_command).

(a) Amplicon mapping: reads of 250 nt in 96 samples (0 to 3 substitutions, a tenth with one indel, 30 % reverse-
    complemented) against 20 000 ZOTUs, --id 0.97 --strand both --otutabout --uc.
(b) The configs[1] shape: 250-nt pieces (a few substitutions) of 100 000 targets of 1 500 nt, --id 0.9, with --blast6out
    alone and with --uc added, so the cost of the CIGAR step shows on its own.

For each: reads/s end to end (best of --repeats), the busy seconds of the reader, device, CIGAR and writer stages of the
best run, and with oracle/_ref/vsearch present the reference CLI at --threads 16 on the same inputs (and for (a) whether
the two --otutabout files are identical).  The GPU's name and power limit are read in the same run.  Prints one JSON line;
--out also writes it to a file.  Inputs are written to a temporary directory."""
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
_COMP = bytes.maketrans(b"ACGT", b"TGCA")
_ALPHA = np.frombuffer(b"ACGT", dtype=np.uint8)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _substitute(rng, reads, k, p):
    for _ in range(k):
        rows = np.nonzero(rng.random(reads.shape[0]) < p)[0]
        cols = rng.integers(0, reads.shape[1], size=rows.size)
        reads[rows, cols] = _ALPHA[(np.searchsorted(_ALPHA, reads[rows, cols]) + 1) % 4]


def _write(path, labels, seqs):
    with open(path, "w") as f:
        for h, s in zip(labels, seqs):
            f.write(f">{h}\n{s.decode()}\n")


def amplicon_inputs(d, nreads, nzotus, seed=5):
    rng = np.random.default_rng(seed)
    zot = _ALPHA[rng.integers(0, 4, size=(nzotus, 250))]
    _write(os.path.join(d, "zotus.fa"), [f"Zotu{i + 1};size={int(rng.integers(1, 1000))}" for i in range(nzotus)], (z.tobytes() for z in zot))
    reads = zot[rng.integers(0, nzotus, size=nreads)].copy()
    _substitute(rng, reads, 3, 0.35)
    indel = rng.random(nreads) < 0.1
    rc = rng.random(nreads) < 0.3

    def seqs():
        for i in range(nreads):
            s = reads[i].tobytes()
            if indel[i]:
                p = 100 + i % 50
                s = s[:p] + s[p + 1:] if i % 2 else s[:p] + b"G" + s[p:]
            yield s.translate(_COMP)[::-1] if rc[i] else s
    _write(os.path.join(d, "reads.fa"), (f"r{i};sample=S{i % 96}" for i in range(nreads)), seqs())
    return os.path.join(d, "reads.fa"), os.path.join(d, "zotus.fa")


def long_target_inputs(d, nreads, ntargets, seed=6):
    rng = np.random.default_rng(seed)
    tg = _ALPHA[rng.integers(0, 4, size=(ntargets, 1500))]
    _write(os.path.join(d, "targets.fa"), (f"T{i}" for i in range(ntargets)), (t.tobytes() for t in tg))
    pick = rng.integers(0, ntargets, size=nreads)
    start = rng.integers(0, 1500 - 250, size=nreads)
    reads = tg[pick[:, None], start[:, None] + np.arange(250)[None, :]]
    _substitute(rng, reads, 6, 0.5)
    _write(os.path.join(d, "pieces.fa"), (f"p{i}" for i in range(nreads)), (r.tobytes() for r in reads))
    return os.path.join(d, "pieces.fa"), os.path.join(d, "targets.fa")


def sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def timed(ctx, q, db, repeats, nreads, **kw):
    runs = []
    for _ in range(repeats):
        t = time.time()
        st = ctx.usearch_global_command(q, db, **kw)
        runs.append((time.time() - t, st))
    best, st = min(runs, key=lambda r: r[0])
    return {"runs_s": [round(r[0], 3) for r in runs], "reads_per_s": round(nreads / best, 0), "matched": st["matched"],
            "hits": st["hits"], "stages_s": {k: round(st[k], 3) for k in ("parse_s", "device_s", "cigar_s", "write_s", "wall_s")}}


def reference(q, db, args, nreads):
    t = time.time()
    r = subprocess.run([STOCK, "--usearch_global", q, "--db", db, "--threads", "16", "--quiet", *args], capture_output=True, text=True)
    dt = time.time() - t
    return {"s": round(dt, 2), "rc": r.returncode, "reads_per_s": round(nreads / dt, 0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2_000_000, help="(a) reads")
    ap.add_argument("--zotus", type=int, default=20_000)
    ap.add_argument("--pieces", type=int, default=200_000, help="(b) queries")
    ap.add_argument("--targets", type=int, default=100_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp()
    rec = {"gpu": gpu_info()}
    ctx = vlib.Context(0)
    ref = os.path.exists(STOCK) and not a.no_reference

    t = time.time()
    q, db = amplicon_inputs(tmp, a.reads, a.zotus)
    otu = os.path.join(tmp, "gpu.otu")
    ra = {"reads": a.reads, "zotus": a.zotus, "gen_s": round(time.time() - t, 1)}
    ra.update(timed(ctx, q, db, a.repeats, a.reads, id=0.97, strand_both=1, otutabout=otu, uc=os.path.join(tmp, "gpu.uc")))
    if ref:
        ref_otu = os.path.join(tmp, "ref.otu")
        ra["reference_t16"] = reference(q, db, ["--id", "0.97", "--strand", "both", "--otutabout", ref_otu, "--uc",
                                                os.path.join(tmp, "ref.uc")], a.reads)
        ra["otutab_equal"] = sha(ref_otu) == sha(otu)
    rec["amplicons"] = ra

    t = time.time()
    q, db = long_target_inputs(tmp, a.pieces, a.targets)
    rb = {"reads": a.pieces, "targets": a.targets, "gen_s": round(time.time() - t, 1)}
    b6 = os.path.join(tmp, "gpu.b6")
    rb["blast6out"] = timed(ctx, q, db, a.repeats, a.pieces, id=0.9, blast6out=b6)
    rb["blast6out_uc"] = timed(ctx, q, db, a.repeats, a.pieces, id=0.9, blast6out=b6, uc=os.path.join(tmp, "gpu2.uc"))
    if ref:
        rb["reference_t16"] = reference(q, db, ["--id", "0.9", "--blast6out", os.path.join(tmp, "ref.b6")], a.pieces)
    rec["long_targets"] = rb
    ctx.close()
    rec["gpu_after"] = gpu_info()
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
