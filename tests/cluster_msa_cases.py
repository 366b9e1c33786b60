"""The cluster consensus cases (--msaout, --consout, --profile) shared by test_cluster_msa_gpu.py, test_cluster_msa_cpu.py
and tools: the inputs (cluster_command_cases.py's generators and a few of their own), the option sets and the reference
CLI's results, stored in tests/golden/cluster_msa_reference.json under the case name with the sha256 of the input.  A
record holds the sha256 of the --msaout, --consout, --profile and --uc files `vsearch --cluster_* ... --threads N` wrote;
the cases the CPU test rebuilds (CPU_CASES) also hold the reference's S / H records in processing order, as
cluster_command_cases.uc_records reads them.

`restate` is a plain numpy statement of the column layout, the profile and the consensus rules of msa() (core/msa.cpp);
both tests compare against it."""
from __future__ import annotations

import json
import os
import re
import subprocess

import numpy as np

import checkers
import cluster_command_cases as cc
from vsearch_b200 import synth

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "cluster_msa_reference.json")
STOCK = cc.STOCK
OUTPUTS = ("msaout", "consout", "profile", "uc")


def indels(path):
    """(m) 24 short roots of 120 nt, each a centroid of abundance 1000 with 7 or 11 members of abundance 1 (even cluster
    sizes): every member carries an inserted run of 1-12 nt at one of two shared positions of its root, half of them a
    deletion too, a few an overhang at either end, and at one shared position half the members swap A for C"""
    rng = np.random.default_rng(41)
    roots = synth.random_seqs(rng, 24, 120)
    labels, seqs = [], []
    for r in range(24):
        root = bytearray(roots[r].tobytes())
        sites = sorted(int(x) for x in rng.choice(np.arange(20, 100), size=3, replace=False))
        root[sites[2]] = ord("A")
        labels.append(f"m{r:02d}_0;size=1000")
        seqs.append(bytes(root))
        nm = 7 if r % 2 == 0 else 11
        for k in range(nm):
            s = bytearray(root)
            if k % 2 == 0:
                s[sites[2]] = ord("C")
            p = sites[k % 2]
            ins = synth.random_seqs(rng, 1, int(rng.integers(1, 13)))[0].tobytes()
            s = s[:p] + ins + s[p:]
            if k % 2 == 1:
                d = int(rng.integers(105, 115))
                del s[d:d + int(rng.integers(1, 4))]
            if k % 4 == 1:
                s = bytearray(synth.random_seqs(rng, 1, 5)[0].tobytes()) + s
            if k % 4 == 3:
                s = s + bytearray(synth.random_seqs(rng, 1, 6)[0].tobytes())
            labels.append(f"m{r:02d}_{k + 1};size=1")
            seqs.append(bytes(s))
    cc._write_fasta(path, labels, seqs)


def big_cluster(path):
    """(n) 20 000 reads of one 250-nt root with 1 % substitutions and a few indels, so one cluster holds them all"""
    rng = np.random.default_rng(42)
    root = synth.random_seqs(rng, 1, 250)[0]
    seqs = []
    for _ in range(20000):
        m = bytearray(synth.mutate(rng, root, 0.01).tobytes())
        seqs.append(bytes(m[int(rng.integers(0, 3)):]))
    cc._write_fasta(path, [f"n{i:05d}" for i in range(len(seqs))], seqs)


def long_reads(path):
    """(o) 240 reads of 4 900-5 000 nt from three roots with 1 % divergence: no pair passes the 16-bit aligner's
    25 000 000-cell bound, so none is deferred, and each cluster spans five 1 024-column tiles"""
    rng = np.random.default_rng(43)
    roots = synth.random_seqs(rng, 3, 5000)
    seqs = []
    for i in range(240):
        m = bytearray(synth.mutate(rng, roots[i % 3], 0.01).tobytes())[:5000]
        seqs.append(bytes(m[int(rng.integers(0, 100)):]))
    cc._write_fasta(path, [f"o{i:03d}" for i in range(len(seqs))], seqs)


def singletons(path):
    """(p) 200 unrelated random reads of 80-300 nt: every cluster is a singleton"""
    rng = np.random.default_rng(44)
    seqs = [synth.random_seqs(rng, 1, int(rng.integers(80, 301)))[0].tobytes() for _ in range(200)]
    cc._write_fasta(path, [f"p{i:03d}" for i in range(len(seqs))], seqs)


INPUTS = dict(cc.INPUTS, indels=(indels, "fasta"), big_cluster=(big_cluster, "fasta"), long_reads=(long_reads, "fasta"),
              singletons=(singletons, "fasta"))

# name: (input, command, CLI options, the same as cluster_cmd_opts keywords)
CASES = {
    "a_fast_dust": ("dust_bait", "cluster_fast", ["--id", "0.97", "--threads", "8"], dict(id=0.97, threads=8)),
    "b_fast_both": ("mixed_strands", "cluster_fast", ["--id", "0.95", "--threads", "16", "--strand", "both", "--qmask", "none"],
                    dict(id=0.95, threads=16, strand_both=1, qmask="none")),
    "c_size_sizes": ("sized", "cluster_size", ["--id", "0.97", "--threads", "4", "--sizein", "--sizeout", "--qmask", "none"],
                     dict(id=0.97, threads=4, sizein=1, sizeout=1, qmask="none")),
    "e_unoise": ("denoise", "cluster_unoise", ["--threads", "4", "--sizein", "--qmask", "none"],
                 dict(threads=4, sizein=1, qmask="none")),
    "f_relabel": ("described", "cluster_fast",
                  ["--id", "0.97", "--threads", "2", "--relabel", "OTU_", "--sizeout", "--xsize", "--clusterout_id",
                   "--clusterout_sort", "--fasta_width", "0", "--notrunclabels", "--qmask", "soft"],
                  dict(id=0.97, threads=2, relabel="OTU_", sizeout=1, xsize=1, clusterout_id=1, clusterout_sort=1, fasta_width=0,
                       notrunclabels=1, qmask="soft")),
    "i_fastq_both": ("fastq_symbols", "cluster_fast",
                     ["--id", "0.9", "--threads", "8", "--minseqlength", "50", "--maxseqlength", "600", "--strand", "both",
                      "--qmask", "none"],
                     dict(id=0.9, threads=8, minseqlength=50, maxseqlength=600, strand_both=1, qmask="none")),
    "j_all_discarded": ("all_short", "cluster_fast", ["--id", "0.97", "--threads", "2"], dict(id=0.97, threads=2)),
    "k_smallmem": ("length_sorted", "cluster_smallmem", ["--id", "0.97", "--threads", "4", "--qmask", "none"],
                   dict(id=0.97, threads=4, qmask="none")),
    "l_hardmask": ("unsorted_lower", "cluster_size", ["--id", "0.95", "--threads", "4", "--qmask", "soft", "--hardmask"],
                   dict(id=0.95, threads=4, qmask="soft", hardmask=1)),
    "m_indels": ("indels", "cluster_size", ["--id", "0.8", "--threads", "4", "--qmask", "none", "--sizeout"],
                 dict(id=0.8, threads=4, qmask="none", sizeout=1)),
    "n_big": ("big_cluster", "cluster_fast", ["--id", "0.9", "--threads", "8"], dict(id=0.9, threads=8)),
    "o_long": ("long_reads", "cluster_fast", ["--id", "0.95", "--threads", "8", "--fasta_width", "120"],
               dict(id=0.95, threads=8, fasta_width=120)),
    "p_singletons": ("singletons", "cluster_fast", ["--id", "0.97", "--threads", "4", "--qmask", "none"],
                     dict(id=0.97, threads=4, qmask="none")),
}

# the cases test_cluster_msa_cpu.py rebuilds from the reference's records (no DUST: no device)
CPU_CASES = ("b_fast_both", "c_size_sizes", "e_unoise", "f_relabel", "i_fastq_both", "k_smallmem", "l_hardmask", "m_indels",
             "p_singletons")
# the cases test_cluster_msa_gpu.py also checks array by array against restate()
ARRAY_CASES = ("m_indels", "n_big", "o_long")

sha256 = cc.sha256


def input_file(name, directory):
    fn, ext = INPUTS[name]
    path = os.path.join(directory, f"{name}.{ext}")
    if not os.path.exists(path):
        fn(path)
    return path


def output_files(directory, name):
    return {o: os.path.join(directory, f"{name}.{o}") for o in OUTPUTS}


def output_digests(paths):
    return {o: sha256(p) for o, p in paths.items()}


def reference_run(inp, command, cli, paths):
    args = [STOCK, "--" + command, inp, *cli]
    for o, p in paths.items():
        args += ["--" + o, p]
    r = subprocess.run(args, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def abundance(label):
    m = re.search(r"(?:^|;)size=(\d+)(?:;|$)", label)
    return int(m.group(1)) if m else 1


def processing_order(command, labels, seqs):
    """Database::sortbylength / sortbyabundance (core/db.cpp:433-485), or the input order for --cluster_smallmem"""
    key = {"cluster_fast": lambda i: (-len(seqs[i]), -abundance(labels[i]), labels[i].encode(), i),
           "cluster_size": lambda i: (-abundance(labels[i]), labels[i].encode(), i),
           "cluster_unoise": lambda i: (-abundance(labels[i]), labels[i].encode(), i),
           "cluster_smallmem": lambda i: i}[command]
    return sorted(range(len(labels)), key=key)


_COMP = bytes.maketrans(b"ACGTURYKMBVDHSWNacgturykmbvdhswn", b"TGCAAYRMKVBHDSWNtgcaayrmkvbhdswn")


def revcomp(s: bytes) -> bytes:
    """reverse_complement with the reference's complement map (IUPAC codes included)"""
    return bytes(s).translate(_COMP)[::-1]


_CLASS = np.full(256, 4, dtype=np.int64)
for _ch, _k in ((b"A", 0), (b"C", 1), (b"G", 2), (b"T", 3), (b"U", 3)):
    _CLASS[_ch[0]] = _CLASS[_ch[0] | 0x20] = _k


def _cigar_ops(cigar):
    return [(int(n) if n else 1, op) for n, op in re.findall(r"(\d*)([MDI])", cigar)]


def restate(seqs, results, weights, cigars):
    """msa() restated: seqs are the records in processing order (bytes, as clustered), results a cluster result array,
    weights per record, cigars the CIGAR of each H record.  Returns (insertions, col_first, profile [columns x 6: A, C,
    G, T, N, gap], consensus bytes), clusters in cluster-number order."""
    n = len(seqs)
    nclusters = int(results["cluster"].max()) + 1 if n else 0
    rows = [[] for _ in range(nclusters)]
    for i in range(n):
        rows[int(results["cluster"][i])].append(i)
    ins_all, first, prof_all, cons_all = [], [0], [], []
    for cl in range(nclusters):
        cent = rows[cl][0]
        assert results["centroid"][cent] < 0
        L = len(seqs[cent])
        ins = np.zeros(L + 1, dtype=np.int64)
        for i in rows[cl][1:]:
            q = 0
            for run, op in _cigar_ops(cigars[i]):
                if op == "D":
                    ins[q] = max(ins[q], run)
                else:
                    q += run
        block = np.concatenate(([0], np.cumsum(ins + 1)))[:-1] if L >= 0 else np.zeros(1, dtype=np.int64)
        block = block.astype(np.int64)            # block p begins at block[p]; centroid column of p: block[p] + ins[p]
        width = L + int(ins.sum())
        centcol = block[:L] + ins[:L]
        prof = np.zeros((width, 6), dtype=np.uint64)
        wsum = 0
        for i in rows[cl]:
            w = int(weights[i])
            wsum += w
            s = seqs[i]
            if results["centroid"][i] >= 0 and results["strand"][i]:
                s = revcomp(s)
            cls = _CLASS[np.frombuffer(s, dtype=np.uint8)] if len(s) else np.zeros(0, dtype=np.int64)
            if results["centroid"][i] < 0:
                cols = centcol
            else:
                parts, q = [], 0
                for run, op in _cigar_ops(cigars[i]):
                    if op == "M":
                        parts.append(centcol[q:q + run])
                        q += run
                    elif op == "I":
                        q += run
                    else:
                        parts.append(block[q] + np.arange(run, dtype=np.int64))
                cols = np.concatenate(parts) if parts else np.zeros(0, dtype=np.int64)
            assert cols.shape[0] == cls.shape[0]
            np.add.at(prof, (cols, cls), np.uint64(w))
        prof[:, 5] = np.uint64(wsum) - prof[:, :5].sum(axis=1)
        cons = bytearray(b"+" * width)
        for k in range(int(ins[0]), width - int(ins[L])):
            best, count = ord("-"), 0
            for j in range(4):
                if int(prof[k, j]) > count:
                    best, count = b"ACGT"[j], int(prof[k, j])
            if count == 0 and int(prof[k, 4]) > 0:
                best, count = ord("N"), int(prof[k, 4])
            cons[k] = best if count >= int(prof[k, 5]) else ord("-")
        ins_all.append(ins)
        first.append(first[-1] + width)
        prof_all.append(prof)
        cons_all.append(bytes(cons))
    return (np.concatenate(ins_all).astype(np.int32) if ins_all else np.zeros(0, dtype=np.int32),
            np.array(first, dtype=np.int64),
            np.concatenate(prof_all) if prof_all else np.zeros((0, 6), dtype=np.uint64),
            b"".join(cons_all))


if __name__ == "__main__":   # regenerate the golden file from oracle/_ref/vsearch
    import sys
    import tempfile
    d = tempfile.mkdtemp()
    out = {}
    for name, (inp, command, cli, kw) in CASES.items():
        p = input_file(inp, d)
        sub = os.path.join(d, name)
        os.makedirs(sub)
        paths = output_files(sub, name)
        reference_run(p, command, cli, paths)
        rec = {"input_sha256": sha256(p), "files": output_digests(paths)}
        if name in CPU_CASES:
            labels, _ = cc.read_input(p, kw.get("notrunclabels", 0))
            rec["records"] = cc.uc_records(open(paths["uc"]).read(), labels)
        out[name] = rec
        print(name, sum(1 for line in open(paths["uc"]) if line[0] == "C"), "clusters", file=sys.stderr)
    with open(GOLDEN, "w") as f:   # one case per line
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(out[k], separators=(",", ":"), sort_keys=True)
                                    for k in sorted(out)) + "\n}\n")
