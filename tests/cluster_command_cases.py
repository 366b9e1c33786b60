"""The clustering command cases shared by test_cluster_command_gpu.py, test_cluster_command_cpu.py and tools: the synthetic
inputs, the option sets and the reference CLI's results, stored in tests/golden/cluster_command_reference.json under the
case name with the sha256 of the input.  A record holds the sha256 of every file `vsearch --cluster_* ... --uc
--centroids --clusters` wrote and the counts of its summary.  The cases the CPU test rebuilds (CPU_CASES) also hold the
reference's S / H records in processing order: [input record, cluster, centroid's input record or -1, strand, id]."""
from __future__ import annotations

import functools
import hashlib
import json
import os
import re
import subprocess

import numpy as np

import checkers
from vsearch_b200 import synth

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "cluster_command_reference.json")
STOCK = os.path.join(checkers.ROOT, "oracle", "_ref", "vsearch")


def _family_reads(rng, n, nroots, rootlen=300, divs=(0.0, 0.01, 0.02, 0.035, 0.05)):
    """n reads from nroots random roots (a few roots own most reads), mutated and trimmed at both ends"""
    roots = synth.random_seqs(rng, nroots, rootlen)
    w = 1.0 / np.arange(1, nroots + 1)
    w /= w.sum()
    pick = rng.choice(nroots, size=n, p=w)
    out = []
    for i in range(n):
        m = synth.mutate(rng, roots[int(pick[i])], float(divs[int(rng.integers(0, len(divs)))]))
        a = int(rng.integers(0, 6))
        b = int(rng.integers(0, 6))
        out.append(bytearray(m[a: m.shape[0] - b].tobytes()))
    return out


_COMP = bytes.maketrans(b"ACGTUacgtu", b"TGCAAtgcaa")


def revcomp(s: bytes) -> bytes:
    return bytes(s).translate(_COMP)[::-1]


def _write_fasta(path, labels, seqs, width=70):
    with open(path, "w") as f:
        for lab, s in zip(labels, seqs):
            t = bytes(s).decode()
            f.write(">" + lab + "\n")
            for a in range(0, len(t), width):
                f.write(t[a:a + width] + "\n")


def dust_bait(path):
    """(a) 1 500 reads of 40 families; every 97th carries a 60-nt AT repeat that DUST masks"""
    rng = np.random.default_rng(21)
    seqs = _family_reads(rng, 1500, 40)
    for i in range(5, len(seqs), 97):
        seqs[i] = seqs[i][:100] + b"AT" * 30 + seqs[i][100:]
    _write_fasta(path, [f"a{i:05d}" for i in range(len(seqs))], seqs)


def mixed_strands(path):
    """(b) 1 200 reads of 30 families, about half of them reverse-complemented"""
    rng = np.random.default_rng(22)
    seqs = _family_reads(rng, 1200, 30)
    seqs = [revcomp(s) if rng.random() < 0.5 else bytes(s) for s in seqs]
    _write_fasta(path, [f"b{i:05d}" for i in range(len(seqs))], seqs)


def sized(path):
    """(c) 500 reads with ;size= annotations from a few values, so many abundances tie and only the label order breaks
    the tie; labels in scrambled order"""
    rng = np.random.default_rng(23)
    seqs = _family_reads(rng, 500, 25, rootlen=250)
    perm = rng.permutation(len(seqs))
    sizes = [int(x) for x in rng.choice([1, 2, 3, 5, 8], size=len(seqs))]
    _write_fasta(path, [f"c{int(perm[i]):04d};size={sizes[i]}" for i in range(len(seqs))], seqs)


def unsorted_lower(path):
    """(d) 400 reads of ragged lengths in no order, some with lower-case runs"""
    rng = np.random.default_rng(24)
    seqs = _family_reads(rng, 400, 20, rootlen=320)
    out = []
    for i, s in enumerate(seqs):
        s = s[: len(s) - int(rng.integers(0, 120))]
        if i % 4 == 0:
            a = int(rng.integers(0, len(s) - 40))
            s[a:a + 30] = bytes(s[a:a + 30]).lower()
        out.append(s)
    _write_fasta(path, [f"d{i:04d}" for i in range(len(out))], out)


def denoise(path):
    """(e) 700 amplicons: a few true sequences of high abundance and their one- and two-error variants of low abundance,
    many of them below the default --minsize 8"""
    rng = np.random.default_rng(25)
    roots = synth.random_seqs(rng, 12, 250)
    labels, seqs = [], []
    for i in range(700):
        r = int(rng.integers(0, len(roots)))
        s = bytearray(roots[r].tobytes())
        if i < len(roots):
            s = bytearray(roots[i].tobytes())
            size = int(rng.integers(200, 2000))
        else:
            for _ in range(int(rng.integers(1, 4))):
                p = int(rng.integers(0, len(s)))
                s[p] = b"ACGT"[(b"ACGT".index(s[p]) + int(rng.integers(1, 4))) % 4]
            size = int(rng.integers(1, 40))
        labels.append(f"e{i:04d};size={size}")
        seqs.append(s)
    _write_fasta(path, labels, seqs)


def described(path):
    """(f) 400 reads whose headers carry ;size= in the middle and a description after a blank"""
    rng = np.random.default_rng(26)
    seqs = _family_reads(rng, 400, 15, rootlen=200)
    labels = [f"f{i:04d};size={int(rng.integers(1, 9))};sample=s{i % 3} desc of {i} x" for i in range(len(seqs))]
    _write_fasta(path, labels, seqs, width=50)


def soft_sized(path):
    """(g) 500 reads with abundances and lower-case runs; many reads are prefixes or suffixes of their family's root, so
    identities of 100 without an identical alignment occur"""
    rng = np.random.default_rng(27)
    seqs = _family_reads(rng, 500, 20, rootlen=260, divs=(0.0, 0.0, 0.01, 0.03))
    out = []
    for i, s in enumerate(seqs):
        if i % 3 == 0:
            s = s[int(rng.integers(0, 15)):]
        if i % 5 == 0:
            a = int(rng.integers(0, len(s) - 30))
            s[a:a + 20] = bytes(s[a:a + 20]).lower()
        out.append(s)
    _write_fasta(path, [f"g{i:04d};size={int(rng.integers(1, 30))}" for i in range(len(out))], out)


def small(path):
    """(h) 150 reads of 6 families"""
    rng = np.random.default_rng(28)
    seqs = _family_reads(rng, 150, 6, rootlen=200)
    _write_fasta(path, [f"h{i:04d}" for i in range(len(seqs))], seqs)


def fastq_symbols(path):
    """(i) FASTQ: 300 reads of 10..600 nt (some below --minseqlength, some above --maxseqlength), with IUPAC codes and U"""
    rng = np.random.default_rng(29)
    seqs = _family_reads(rng, 300, 10, rootlen=500)
    with open(path, "w") as f:
        for i, s in enumerate(seqs):
            if i % 7 == 0:
                s = s[: int(rng.integers(10, 60))]
            elif i % 11 == 0:
                s = s + bytes(synth.random_seqs(rng, 1, 200)[0].tobytes())
            if i % 5 == 0:
                for c in b"NRYUKMBuSW":
                    s[int(rng.integers(0, len(s)))] = c
            q = bytes(33 + int(x) for x in rng.integers(0, 41, size=len(s)))
            f.write(f"@i{i:04d} read {i}\n{bytes(s).decode()}\n+\n{q.decode()}\n")


def all_short(path):
    """(j) every record shorter than 32 nt"""
    rng = np.random.default_rng(30)
    _write_fasta(path, [f"j{i}" for i in range(20)], [synth.random_seqs(rng, 1, int(rng.integers(5, 32)))[0].tobytes()
                                                     for _ in range(20)])


def length_sorted(path):
    """(k) 300 reads in decreasing length order, for --cluster_smallmem without --usersort"""
    rng = np.random.default_rng(31)
    seqs = sorted(_family_reads(rng, 300, 12, rootlen=280), key=len, reverse=True)
    _write_fasta(path, [f"k{i:04d}" for i in range(len(seqs))], seqs)


INPUTS = {"dust_bait": (dust_bait, "fasta"), "mixed_strands": (mixed_strands, "fasta"), "sized": (sized, "fasta"),
          "unsorted_lower": (unsorted_lower, "fasta"), "denoise": (denoise, "fasta"), "described": (described, "fasta"),
          "soft_sized": (soft_sized, "fasta"), "small": (small, "fasta"), "fastq_symbols": (fastq_symbols, "fastq"),
          "all_short": (all_short, "fasta"), "length_sorted": (length_sorted, "fasta")}

# name: (input, command, CLI options, the same as cluster_cmd_opts keywords, outputs); outputs: "uc", "centroids",
# "clusters"
CASES = {
    "a_fast_dust": ("dust_bait", "cluster_fast", ["--id", "0.97", "--threads", "8"], dict(id=0.97, threads=8),
                    ("uc", "centroids")),
    "b_fast_both": ("mixed_strands", "cluster_fast", ["--id", "0.95", "--threads", "16", "--strand", "both"],
                    dict(id=0.95, threads=16, strand_both=1), ("uc", "centroids", "clusters")),
    "c_size_sizes": ("sized", "cluster_size", ["--id", "0.97", "--threads", "4", "--sizein", "--sizeout", "--qmask", "none"],
                     dict(id=0.97, threads=4, sizein=1, sizeout=1, qmask="none"), ("uc", "centroids", "clusters")),
    "d_smallmem_usersort": ("unsorted_lower", "cluster_smallmem",
                            ["--id", "0.95", "--threads", "1", "--usersort", "--qmask", "none"],
                            dict(id=0.95, threads=1, usersort=1, qmask="none"), ("uc", "centroids", "clusters")),
    "e_unoise": ("denoise", "cluster_unoise", ["--threads", "4", "--sizein", "--sizeout"], dict(threads=4, sizein=1, sizeout=1),
                 ("uc", "centroids")),
    "f_relabel": ("described", "cluster_fast",
                  ["--id", "0.97", "--threads", "2", "--relabel", "OTU_", "--sizeout", "--xsize", "--clusterout_id",
                   "--clusterout_sort", "--fasta_width", "0", "--notrunclabels", "--qmask", "soft"],
                  dict(id=0.97, threads=2, relabel="OTU_", sizeout=1, xsize=1, clusterout_id=1, clusterout_sort=1, fasta_width=0,
                       notrunclabels=1, qmask="soft"), ("uc", "centroids", "clusters")),
    "g_iddef1_sizeorder": ("soft_sized", "cluster_size",
                           ["--id", "0.97", "--threads", "3", "--iddef", "1", "--maxaccepts", "4", "--maxrejects", "16",
                            "--sizeorder", "--qmask", "soft", "--sizein"],
                           dict(id=0.97, threads=3, iddef=1, maxaccepts=4, maxrejects=16, sizeorder=1, qmask="soft", sizein=1),
                           ("uc", "centroids", "clusters")),
    "h_exhaustive": ("small", "cluster_fast", ["--id", "0.97", "--threads", "4", "--maxaccepts", "0", "--maxrejects", "0"],
                     dict(id=0.97, threads=4, maxaccepts=0, maxrejects=0), ("uc", "centroids")),
    "i_fastq": ("fastq_symbols", "cluster_fast", ["--id", "0.9", "--threads", "8", "--minseqlength", "50", "--maxseqlength", "600"],
                dict(id=0.9, threads=8, minseqlength=50, maxseqlength=600), ("uc", "centroids", "clusters")),
    "j_all_discarded": ("all_short", "cluster_fast", ["--id", "0.97", "--threads", "2"], dict(id=0.97, threads=2),
                        ("uc", "centroids", "clusters")),
    "k_smallmem_sorted": ("length_sorted", "cluster_smallmem", ["--id", "0.97", "--threads", "4"], dict(id=0.97, threads=4),
                          ("uc", "centroids")),
}

# the cases test_cluster_command_cpu.py rebuilds from the reference's records (no DUST: no device)
CPU_CASES = ("c_size_sizes", "d_smallmem_usersort", "f_relabel", "g_iddef1_sizeorder")


def sha256_bytes(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def sha256(path):
    with open(path, "rb") as f:
        return sha256_bytes(f.read())


@functools.lru_cache(maxsize=None)
def input_file(name, directory):
    fn, ext = INPUTS[name]
    path = os.path.join(directory, f"{name}.{ext}")
    if not os.path.exists(path):
        fn(path)
    return path


def output_files(directory, name, outputs):
    """{output: path} for a run of case `name` in `directory`; "clusters" is the prefix"""
    return {o: os.path.join(directory, f"{name}.{o}" if o != "clusters" else f"{name}.cl_") for o in outputs}


def output_digests(paths):
    """{file name: sha256}: "uc", "centroids" and one "clusters<n>" per cluster file"""
    out = {}
    for o, p in paths.items():
        if o == "clusters":
            d, prefix = os.path.split(p)
            for f in os.listdir(d):
                if f.startswith(prefix) and f[len(prefix):].isdigit():
                    out["clusters" + f[len(prefix):]] = sha256(os.path.join(d, f))
        else:
            out[o] = sha256(p)
    return out


_SUMMARY = {"sequences": r"nt in (\d+) seqs", "discarded_short": r"minseqlength \d+: (\d+) seq",
            "discarded_long": r"maxseqlength \d+: (\d+) seq", "discarded_minsize": r"minsize \d+: (\d+) seq",
            "clusters": r"Clusters: (\d+)", "singletons": r"Singletons: (\d+)"}


def reference_run(inp, command, cli, paths):
    """runs the reference CLI; returns the counts of its stderr summary"""
    args = [STOCK, "--" + command, inp, *cli]
    flags = {"uc": "--uc", "centroids": "--centroids", "clusters": "--clusters"}
    for o, p in paths.items():
        args += [flags[o], p]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    counts = {}
    for k, pat in _SUMMARY.items():
        m = re.search(pat, r.stderr)
        counts[k] = int(m.group(1)) if m else 0
    return counts


def uc_records(uc_text: str, input_labels):
    """the S / H records of a --uc file in processing order: [input record, cluster, centroid's input record or -1, strand
    (0 / 1), id]; labels are matched on their first ';'- or blank-separated token, which is unique in every input"""
    key = {re.split(r"[; \t]", lab)[0]: i for i, lab in enumerate(input_labels)}
    out = []
    for line in uc_text.splitlines():
        f = line.split("\t")
        if f[0] == "S":
            out.append([key[re.split(r"[; \t]", f[8])[0]], int(f[1]), -1, 0, 0.0])
        elif f[0] == "H":
            out.append([key[re.split(r"[; \t]", f[8])[0]], int(f[1]), key[re.split(r"[; \t]", f[9])[0]],
                        int(f[4] == "-"), float(f[3])])
    return out


def read_input(path, notrunclabels=False):
    """(labels, sequences) of a FASTA / FASTQ input file, labels cut at the first blank unless notrunclabels"""
    labels, seqs = [], []
    with open(path) as f:
        text = f.read()
    if text.startswith("@"):
        lines = text.splitlines()
        for i in range(0, len(lines), 4):
            labels.append(lines[i][1:])
            seqs.append(lines[i + 1].encode())
    else:
        for rec in text.split(">")[1:]:
            h, _, body = rec.partition("\n")
            labels.append(h)
            seqs.append(body.replace("\n", "").encode())
    if not notrunclabels:
        labels = [re.split(r"[ \t]", h)[0] for h in labels]
    return labels, seqs


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


if __name__ == "__main__":   # regenerate the golden file from oracle/_ref/vsearch
    import sys
    import tempfile
    d = tempfile.mkdtemp()
    out = {}
    for name, (inp, command, cli, kw, outputs) in CASES.items():
        p = input_file(inp, d)
        sub = os.path.join(d, name)
        os.makedirs(sub)
        paths = output_files(sub, name, outputs)
        counts = reference_run(p, command, cli, paths)
        rec = {"input_sha256": sha256(p), "files": output_digests(paths), **counts}
        if name in CPU_CASES:
            labels, _ = read_input(p, kw.get("notrunclabels", 0))
            rec["records"] = uc_records(open(paths["uc"]).read(), labels)
        out[name] = rec
        print(name, {k: v for k, v in rec.items() if k not in ("files", "records")}, len(rec["files"]), file=sys.stderr)
    with open(GOLDEN, "w") as f:   # one case per line
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(out[k], separators=(",", ":"), sort_keys=True)
                                    for k in sorted(out)) + "\n}\n")
