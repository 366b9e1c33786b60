"""Time --chimeras_denovo on the GPU against the reference CLI (oracle/_ref/vsearch --chimeras_denovo ... --threads 1) on
seeded long reads: prints the stage seconds, the bands, the recomputed queries and whether every file is identical.

    python tools/perf_chimeras_denovo.py [--nfam 20] [--per 10] [--nchim 300] [--nclean 100] [--no-ref]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import chimeras_denovo_cases as D  # noqa: E402
from vsearch_b200 import lib as vlib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfam", type=int, default=20)
    ap.add_argument("--per", type=int, default=10)
    ap.add_argument("--nchim", type=int, default=300)
    ap.add_argument("--nclean", type=int, default=100)
    ap.add_argument("--seed", type=int, default=99)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        q = D.reads(d, seed=a.seed, nfam=a.nfam, per=a.per, nchim=a.nchim, nclean=a.nclean, njunk=10, lo=1500, hi=3000)
        mine = {k: os.path.join(d, "mine." + k) for k in D.OUTPUTS}
        ctx = vlib.Context(0)
        st = ctx.uchime(q, None, command=D.C, **mine)
        ctx.close()
        print("gpu: wall %.2f s (parse %.2f, search %.2f, align %.2f, parents %.2f, eval %.2f, serial %.2f, write %.2f); "
              "queries %d, chimeras %d, candidates %d, bands %d, recomputed %d"
              % (st["wall_s"], st["parse_s"], st["search_s"], st["align_s"], st["parents_s"], st["eval_s"], st["serial_s"], st["write_s"],
                 st["queries"], st["chimeras"], st["candidates"], st["bands"], st["recomputed"]), flush=True)
        if a.no_ref or not os.path.exists(D.STOCK):
            print("reference: not run")
            return
        ref = {k: os.path.join(d, "ref." + k) for k in D.OUTPUTS}
        cmd = [D.STOCK, "--chimeras_denovo", q, "--threads", "1", "--quiet"]
        for k, p in ref.items():
            cmd += [f"--{D.OUTPUTS[k]}", p]
        t = time.perf_counter()
        subprocess.run(cmd, check=True)
        print("reference --threads 1: %.2f s; files identical: %s"
              % (time.perf_counter() - t, all(D.U.sha(mine[k]) == D.U.sha(ref[k]) for k in D.OUTPUTS)))


if __name__ == "__main__":
    main()
