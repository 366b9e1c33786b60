"""Timing of the --makeudb_usearch command (vsg_makeudb_usearch) on one GPU: parse, device and write seconds.

Workloads: 100 000 random sequences of 1 500 nt (defaults, --dbmask none, --wordlength 12) and a configs[3]-shaped
1 000 000 x 1 200-nt database (defaults).  With --ref, the reference CLI (oracle/_ref/vsearch) is timed on the first
workload with defaults on the same host, and its file is compared with ours.  Inputs and outputs go to a temporary
directory (or --dir) and are removed.

    python tools/perf_makeudb.py [--ref] [--runs 3] [--out perf_makeudb.json]
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

STOCK = os.path.join(ROOT, "oracle", "_ref", "vsearch")
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def write_fasta(path, n, length, seed):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        for a in range(0, n, 20000):
            m = min(20000, n - a)
            s = ACGT[rng.integers(0, 4, size=(m, length), dtype=np.uint8)]
            lines = bytearray()
            for i in range(m):
                lines += b">s%d\n" % (a + i) + s[i].tobytes() + b"\n"
            f.write(lines)


def digest(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--ref", action="store_true")
    ap.add_argument("--skip-large", action="store_true")
    ap.add_argument("--dir", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    d = tempfile.mkdtemp(dir=a.dir)
    results = []
    try:
        ctx = vlib.Context(0)
        work = [("100k x 1500", 100000, 1500, [("defaults", {}), ("dbmask none", dict(dbmask="none")),
                                                ("wordlength 12", dict(wordlength=12))])]
        if not a.skip_large:
            work.append(("1M x 1200", 1000000, 1200, [("defaults", {})]))
        for wname, n, length, cases in work:
            fa = os.path.join(d, "db.fasta")
            t0 = time.time()
            write_fasta(fa, n, length, seed=1)
            print(f"[{wname}] input {os.path.getsize(fa) / 1e6:.0f} MB written in {time.time() - t0:.1f} s", flush=True)
            for cname, opts in cases:
                out = os.path.join(d, "db.udb")
                for r in range(a.runs):
                    st = ctx.makeudb_usearch(fa, out, **opts)
                    rec = dict(workload=wname, case=cname, run=r, size=os.path.getsize(out), **st)
                    results.append(rec)
                    print(f"[{wname} / {cname}] wall {st['wall_s']:.2f} s = parse {st['parse_s']:.2f} + device {st['device_s']:.2f}"
                          f" + write {st['write_s']:.2f}; {st['index_entries']} index entries, {rec['size'] / 1e6:.0f} MB", flush=True)
                if a.ref and wname.startswith("100k") and cname == "defaults" and os.path.exists(STOCK):
                    ref = os.path.join(d, "ref.udb")
                    t0 = time.time()
                    subprocess.run([STOCK, "--makeudb_usearch", fa, "--output", ref, "--quiet"], check=True)
                    wall = time.time() - t0
                    same = digest(ref) == digest(out)
                    results.append(dict(workload=wname, case=cname, reference_wall_s=wall, identical=same))
                    print(f"[{wname} / {cname}] reference CLI wall {wall:.1f} s, files identical: {same}", flush=True)
                    os.remove(ref)
                os.remove(out)
            os.remove(fa)
        ctx.close()
    finally:
        shutil.rmtree(d, ignore_errors=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
