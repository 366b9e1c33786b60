"""Cluster consensus (--consout, --msaout, --profile) of the clustering commands: time of the MSA stage and of the command.

Two seeded inputs, written to a temporary directory:
- amplicons: about 500 000 reads of about 250 nt; five roots own 60 000 reads each (clusters of more than 50 000
  members), the other 200 000 reads come from 20 000 roots in tens, all with 1 % substitutions and a few indels;
- long reads: 300 reads of 4 900-5 000 nt from six roots (5 000 nt is about the longest pair the 16-bit aligner takes
  without deferring it: 25 000 000 cells).
For each: `--cluster_fast --id 0.97` run once without and once with --consout (plus --msaout and --profile for the long
reads), as vsg_cluster_command_outputs in a child process with VSG_TRACE, which prints the MSA stage's kernel time (CUDA
events around its kernels), its device time (host clock around vsg_cluster_msa, which ends in a device synchronise) and
its write time.  With oracle/_ref/vsearch present, the reference CLI runs the same two commands (--threads = the CPUs).
Prints the GPU's name and power limit and one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STOCK = os.path.join(ROOT, "oracle", "_ref", "vsearch")

_CHILD = r"""
import json, sys, time
sys.path.insert(0, sys.argv[1])
from vsearch_b200 import lib as vlib
ctx = vlib.Context(0)
outs = json.loads(sys.argv[3])
t = time.perf_counter()
st = ctx.cluster_command(sys.argv[2], command="cluster_fast", id=0.97, threads=int(sys.argv[4]), **outs)
print(json.dumps({"wall_s": time.perf_counter() - t, "clusters": st["clusters"], "sequences": st["sequences"]}))
ctx.close()
"""


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _mutate(rng, root, rate):
    s = root.copy()
    k = rng.random(s.shape[0]) < rate
    s[k] = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=int(k.sum()))]
    b = bytearray(s.tobytes())
    if rng.random() < 0.2:
        p = int(rng.integers(10, len(b) - 10))
        if rng.random() < 0.5:
            del b[p:p + int(rng.integers(1, 4))]
        else:
            b[p:p] = bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, size=int(rng.integers(1, 4))))
    return bytes(b)


def make_amplicons(path, seed=11):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    big = acgt[rng.integers(0, 4, size=(5, 250))]
    small = acgt[rng.integers(0, 4, size=(20000, 250))]
    with open(path, "w") as f:
        i = 0
        for r in range(5):
            for _ in range(60000):
                f.write(f">a{i};size=1\n{_mutate(rng, big[r], 0.01).decode()}\n")
                i += 1
        for r in range(20000):
            for _ in range(10):
                f.write(f">a{i};size=1\n{_mutate(rng, small[r], 0.01).decode()}\n")
                i += 1


def make_long(path, seed=12):
    rng = np.random.default_rng(seed)
    roots = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=(6, 5000))]
    with open(path, "w") as f:
        for i in range(300):
            s = _mutate(rng, roots[i % 6], 0.01)[:5000]
            f.write(f">l{i}\n{s[int(rng.integers(0, 100)):].decode()}\n")


def run_gpu(inp, outs, threads):
    env = dict(os.environ, VSG_TRACE="1")
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, inp, json.dumps(outs), str(threads)], capture_output=True, text=True,
                       env=env)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-3000:])
    rec = json.loads(r.stdout.strip().splitlines()[-1])
    m = re.search(r"cluster_msa: .* (\d+) columns, .* kernels ([\d.]+) ms", r.stderr)
    if m:
        rec["msa_columns"] = int(m.group(1))
        rec["msa_kernel_ms"] = float(m.group(2))
    m = re.search(r"cluster_command: msa device ([\d.]+) s, msa write ([\d.]+) s", r.stderr)
    if m:
        rec["msa_device_s"] = float(m.group(1))
        rec["msa_write_s"] = float(m.group(2))
    return rec


def run_ref(inp, outs, threads):
    args = [STOCK, "--cluster_fast", inp, "--id", "0.97", "--threads", str(threads)]
    for k, p in outs.items():
        args += ["--" + k, p]
    t = time.perf_counter()
    r = subprocess.run(args, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return round(time.perf_counter() - t, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--threads", type=int, default=16, help="--threads of the GPU command (the round size)")
    a = ap.parse_args()
    d = tempfile.mkdtemp()
    result = {"gpu": gpu_info()}
    print("gpu:", result["gpu"], flush=True)
    inputs = {"amplicons": (make_amplicons, ("consout",)), "long_reads": (make_long, ("consout", "msaout", "profile"))}
    for name, (make, with_outs) in inputs.items():
        inp = os.path.join(d, name + ".fa")
        make(inp)
        base = {"uc": os.path.join(d, name + ".uc")}
        full = dict(base, **{o: os.path.join(d, f"{name}.{o}") for o in with_outs})
        rec = {"without": run_gpu(inp, base, a.threads), "with": run_gpu(inp, full, a.threads), "outputs": list(with_outs)}
        if os.path.exists(STOCK):
            cpus = os.cpu_count() or 1
            rref = {k: p + ".ref" for k, p in full.items()}
            rec["reference_threads"] = cpus
            rec["reference_without_s"] = run_ref(inp, {"uc": rref["uc"]}, cpus)
            rec["reference_with_s"] = run_ref(inp, rref, cpus)
            rec["consout_equal"] = open(full["consout"], "rb").read() == open(rref["consout"], "rb").read()
        result[name] = rec
        print(name, json.dumps(rec), flush=True)
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
