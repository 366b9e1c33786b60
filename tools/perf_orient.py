"""Time --orient on the GPU (vsg_orient_stream end to end, vsg_orient's device time) and the reference CLI on a prefix of
the same files.

Database: 20 000 x 1 450-nt references, 400 families of 50 members (3 % substitutions from their root), default
options (--wordlength 12, --dbmask dust, --qmask dust).  Two read sets, each a third reverse-complemented and mutated by
3 %: 1 000 000 x 250-nt windows of the references, and 20 000 x ~10-kb reads made of seven references' windows.  Per
read set one JSON line: reads/s of the stream (--fastaout, --notmatched, --tabbedout; best of --repeats runs), the device
time of one vsg_orient call over all reads (vsg_profile.rank_ms), the GPU name and power limit, and for the reference
CLI (single-threaded by construction) on the first --ref-reads reads (a tenth of that for the 10-kb reads): its reads/s
without its start-up (the run on one read is subtracted) and whether the stream's three files on that prefix equal the
CLI's byte for byte.

    python tools/perf_orient.py [--short 1000000] [--long 20000] [--ref-reads 20000] [--repeats 3] [--out DIR]
"""
import argparse
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
from vsearch_b200 import lib, synth  # noqa: E402

STOCK = os.path.join(ROOT, "oracle", "_ref", "vsearch")
COMP = np.zeros(256, dtype=np.uint8)
COMP[np.frombuffer(b"ACGT", dtype=np.uint8)] = np.frombuffer(b"TGCA", dtype=np.uint8)
OUTS = ("fastaout", "notmatched", "tabbedout")


def make_db(rng, n_ref=20000, length=1450, families=400):
    roots = synth.random_seqs(rng, families, length)
    dbm = roots[np.arange(n_ref) % families].copy()
    sub = rng.random(dbm.shape) < 0.03
    dbm[sub] = synth.ACGT[rng.integers(0, 4, size=int(sub.sum()), dtype=np.uint8)]
    return dbm


def write_reads(path, rng, dbm, n, pieces, piece_len, chunk):
    """n reads of `pieces` windows of piece_len nt from random references, a third reverse-complemented, mutated 3 %"""
    with open(path, "wb") as f:
        for c0 in range(0, n, chunk):
            m = min(chunk, n - c0)
            src = rng.integers(0, dbm.shape[0], size=(m, pieces))
            start = rng.integers(0, dbm.shape[1] - piece_len + 1, size=(m, pieces))
            cols = start[:, :, None] + np.arange(piece_len)[None, None, :]
            win = dbm[src[:, :, None], cols].reshape(m, pieces * piece_len)
            rc = rng.random(m) < 1 / 3
            win[rc] = COMP[win[rc][:, ::-1]]
            ss = synth.mutate_batch(rng, win, 0.03)
            for i in range(m):
                f.write(b">r%d\n" % (c0 + i) + ss.seq(i) + b"\n")


def prefix(src, dst, n):
    with open(src, "rb") as f, open(dst, "wb") as g:
        for _ in range(2 * n):
            g.write(f.readline())


def read_records(path):
    heads, seqs = [], []
    with open(path, "rb") as f:
        for line in f:
            if line.startswith(b">"):
                heads.append(line[1:].rstrip(b"\n"))
            else:
                seqs.append(line.rstrip(b"\n"))
    return heads, seqs


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def run_ref(dbf, qf, tmp, tag):
    outs = {o: os.path.join(tmp, f"ref_{tag}.{o}") for o in OUTS}
    args = [STOCK, "--orient", qf, "--db", dbf, "--quiet"] + sum((["--" + o, p] for o, p in outs.items()), [])
    t0 = time.perf_counter()
    subprocess.run(args, check=True)
    return time.perf_counter() - t0, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--short", type=int, default=1_000_000)
    ap.add_argument("--long", type=int, default=20_000)
    ap.add_argument("--ref-reads", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = np.random.default_rng(29)
    tmp = tempfile.mkdtemp()
    dbm = make_db(rng)
    dbf = os.path.join(tmp, "db.fa")
    synth.write_records(dbf, [f"db{i}" for i in range(dbm.shape[0])], [r.tobytes() for r in dbm])
    # name: (reads, windows per read, window length, reads generated at a time, reads the reference CLI runs)
    sets = {"250nt": (a.short, 1, 250, 100_000, a.ref_reads), "10kb": (a.long, 7, 1450, 1_000, a.ref_reads // 10)}
    g = lib.Group([0], synth.SeqSet.from_matrix(dbm), wordlength=12, mask_lower=1, dust_db=1)
    ctx = lib.Context(0)
    db = ctx.seqset(synth.SeqSet.from_matrix(dbm))
    db.dust()
    ix = ctx.index(db, wordlength=12, mask_lower=1)
    lines = []
    for name, (n, pieces, plen, chunk, ref_reads) in sets.items():
        qf = os.path.join(tmp, f"{name}.fa")
        write_reads(qf, rng, dbm, n, pieces, plen, chunk)
        outs = {o: os.path.join(tmp, f"gpu_{name}.{o}") for o in OUTS}
        rec = {"reads": name, "n": n, "refs": int(dbm.shape[0]), "wordlength": 12, "gpu": gpu_info()}
        # the prefix first: the stream's warm-up, and its files against the reference CLI's
        nref = min(ref_reads, n)
        pf, one = os.path.join(tmp, f"{name}.prefix.fa"), os.path.join(tmp, f"{name}.one.fa")
        prefix(qf, pf, nref)
        prefix(qf, one, 1)
        g.orient_stream(pf, **outs)
        if os.path.exists(STOCK) and nref > 0:
            t1, _ = run_ref(dbf, one, tmp, name + "_one")
            tn, routs = run_ref(dbf, pf, tmp, name)
            rec.update({"ref_reads": nref, "ref_s": tn, "ref_startup_s": t1, "ref_reads_per_s": nref / max(tn - t1, 1e-9),
                        "ref_outputs_equal": all(open(outs[o], "rb").read() == open(routs[o], "rb").read() for o in OUTS)})
        best, st, ns = None, None, None
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            st, ns = g.orient_stream(qf, **outs)
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        rec.update({"stream_s": best, "stream_reads_per_s": n / best, "nstrand": list(ns), "stream_stats": st})
        heads, seqs = read_records(qf)
        qset = ctx.seqset(synth.SeqSet(seqs))
        ctx.orient(ix, qset, 0, n)   # warm-up
        ctx.profile_reset()
        rows = ctx.orient(ix, qset, 0, n)
        rec["orient_device_ms"] = float(ctx.profile().rank_ms)
        rec["orient_equals_stream"] = [int((rows[:, 0] == s).sum()) for s in range(3)] == list(ns)
        qset.close()
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    for h in (ix, db):
        h.close()
    ctx.close()
    g.close()
    shutil.rmtree(tmp, ignore_errors=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "perf_orient.jsonl"), "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
