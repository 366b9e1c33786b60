"""Throughput of --search_exact: 2 000 000 reads of 250 nt in 96 samples against 20 000 ZOTUs (60 % exact copies, a
tenth of those reverse-complemented, the rest one substitution away), --strand both, --otutabout and --uc.

Reports the reads/s of vsg_search_exact_command end to end (best of three), the device time of vsg_exact_index_create
(hash + sort of the ZOTUs) and of vsg_search_exact over all reads in one resident set (hash + lookup + verify; host
clocks around calls that end in a device synchronise), the GPU's name and power limit, and with oracle/_ref/vsearch
present the reference CLI at --threads 16 and whether the two OTU tables are equal.  Prints one JSON line; --out
also writes it to a file.  Inputs are written to a temporary directory."""
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_inputs(d, nreads, nzotus, length, seed=5):
    rng = np.random.default_rng(seed)
    zot = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=(nzotus, length))]
    with open(os.path.join(d, "zotus.fa"), "w") as f:
        for i in range(nzotus):
            f.write(f">Zotu{i + 1};size={int(rng.integers(1, 1000))}\n{zot[i].tobytes().decode()}\n")
    pick = rng.integers(0, nzotus, size=nreads)
    kind = rng.random(nreads)
    reads = zot[pick].copy()
    mut = kind >= 0.6
    pos = rng.integers(0, length, size=nreads)
    rows = np.nonzero(mut)[0]
    sub = np.frombuffer(b"CGTA", dtype=np.uint8)
    lut = np.zeros(256, dtype=np.uint8)
    lut[np.frombuffer(b"ACGT", dtype=np.uint8)] = sub
    reads[rows, pos[rows]] = lut[reads[rows, pos[rows]]]
    rc = (kind < 0.06)
    with open(os.path.join(d, "reads.fa"), "w") as f:
        for i in range(nreads):
            s = reads[i].tobytes()
            if rc[i]:
                s = s.translate(_COMP)[::-1]
            f.write(f">r{i};sample=S{i % 96}\n{s.decode()}\n")
    return os.path.join(d, "reads.fa"), os.path.join(d, "zotus.fa"), reads, zot, rc


class _Seqs:
    def __init__(self, mat):
        self.cat = np.ascontiguousarray(mat).reshape(-1)
        self.lens = np.full(mat.shape[0], mat.shape[1], dtype=np.int32)
        self.offs = np.arange(mat.shape[0], dtype=np.int64) * mat.shape[1]


def sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2_000_000)
    ap.add_argument("--zotus", type=int, default=20_000)
    ap.add_argument("--length", type=int, default=250)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp()
    t0 = time.time()
    q, db, reads, zot, rc = make_inputs(tmp, a.reads, a.zotus, a.length)
    rec = {"reads": a.reads, "zotus": a.zotus, "length": a.length, "gen_s": round(time.time() - t0, 1), "gpu": gpu_info()}
    ctx = vlib.Context(0)
    outs = {"otutabout": os.path.join(tmp, "gpu.otu"), "uc": os.path.join(tmp, "gpu.uc")}
    runs = []
    for _ in range(a.repeats):
        t = time.time()
        st = ctx.search_exact_command(q, db, strand_both=1, **outs)
        runs.append((time.time() - t, st))
    best, st = min(runs, key=lambda r: r[0])
    rec["command_s"] = [round(r[0], 3) for r in runs]
    rec["command_reads_per_s"] = round(a.reads / best, 0)
    rec["command_stages_s"] = {k: round(st[k], 3) for k in ("parse_s", "device_s", "write_s", "wall_s")}
    rec["matched"] = st["matched"]
    # the library call alone, every read resident on the device
    dset = ctx.seqset(_Seqs(zot))
    qset = ctx.seqset(_Seqs(reads))
    o = vlib.default_search_opts()
    o.strand_both = 1
    ctx.sync()
    t = time.time()
    ix = ctx.exact_index(dset)
    ctx.sync()
    rec["index_ms"] = round(1e3 * (time.time() - t), 2)
    rows, first, _ = ctx.search_exact(ix, qset, 0, min(a.reads, 65536), o)   # warm-up
    best = None
    for _ in range(3):
        t = time.time()
        rows, first, _ = ctx.search_exact(ix, qset, 0, a.reads, o, cap=int(2.5 * a.reads))
        ctx.sync()
        dt = time.time() - t
        best = dt if best is None else min(best, dt)
    rec["search_call_ms"] = round(1e3 * best, 1)
    rec["search_call_reads_per_s"] = round(a.reads / best, 0)
    rec["search_call_rows"] = int(first[-1])
    ix.close()
    qset.close()
    dset.close()
    ctx.close()
    if os.path.exists(STOCK):
        ref_otu = os.path.join(tmp, "ref.otu")
        t = time.time()
        r = subprocess.run([STOCK, "--search_exact", q, "--db", db, "--strand", "both", "--threads", "16", "--otutabout", ref_otu,
                            "--uc", os.path.join(tmp, "ref.uc"), "--quiet"], capture_output=True, text=True)
        rec["reference_t16_s"] = round(time.time() - t, 2)
        rec["reference_rc"] = r.returncode
        rec["reference_reads_per_s"] = round(a.reads / (time.time() - t), 0)
        rec["otutab_equal"] = sha(ref_otu) == sha(outs["otutabout"])
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
