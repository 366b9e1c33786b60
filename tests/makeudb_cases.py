"""The --makeudb_usearch parity cases shared by test_makeudb_gpu.py and tools: the synthetic inputs, the option sets and
the reference CLI's results, stored in tests/golden/makeudb_reference.json under the case name with the sha256 of the
input.  A record holds the sha256 and size of the file `vsearch --makeudb_usearch` wrote; the "search_*" records hold
the digest of the --blast6out of `vsearch --usearch_global` against the reference's own UDB file of the same FASTA
(test_udb_gpu.py's database, queries and options)."""
from __future__ import annotations

import functools
import hashlib
import json
import os
import subprocess

import numpy as np

import checkers
from vsearch_b200 import synth

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "makeudb_reference.json")
STOCK = os.path.join(checkers.ROOT, "oracle", "_ref", "vsearch")


def _random(rng, n):
    return synth.random_seqs(rng, 1, n)[0].tobytes()


def mixed(path):
    """400 ragged records: low-complexity stretches (DUST masks them), lower-case runs, IUPAC codes, U, a few records of
    fewer than k symbols; headers with descriptions"""
    rng = np.random.default_rng(11)
    with open(path, "w") as f:
        for i in range(400):
            s = bytearray(_random(rng, int(rng.integers(32, 1200))))
            if i % 5 == 0:
                a = int(rng.integers(0, max(1, len(s) - 80)))
                s[a:a + 64] = (b"ACACACACAC" * 7)[: len(s[a:a + 64])]
            if i % 7 == 0:
                a = int(rng.integers(0, max(1, len(s) - 40)))
                s[a:a + 30] = bytes(s[a:a + 30]).lower()
            if i % 9 == 0:
                for c in b"NRYUKMBu":
                    s[int(rng.integers(0, len(s)))] = c
            if i % 50 == 3:
                s = s[:34]
            f.write(f">r{i};size={i % 5 + 1} desc\tof {i}\n")
            t = s.decode()
            for a in range(0, len(t), 60):
                f.write(t[a:a + 60] + "\n")


def lengths(path):
    """records of 20, 31, 32, 50 000, 50 001 and 60 000 nt among ordinary ones"""
    rng = np.random.default_rng(12)
    with open(path, "w") as f:
        for i, n in enumerate([300, 20, 31, 32, 50000, 50001, 60000, 500, 20, 60000, 1000]):
            f.write(f">len{i}_{n}\n{_random(rng, n).decode()}\n")


def symbols(path):
    """lower case, IUPAC codes, U / u, and symbols the reference strips with a warning: digits, '*', blanks"""
    rng = np.random.default_rng(13)
    with open(path, "w") as f:
        for i in range(60):
            s = list(_random(rng, int(rng.integers(40, 400))).decode())
            for j in range(0, len(s), 17):
                s[j] = "acgtuRYSWKMBDHVNrysw*0123456789 "[(i + j) % 32]
            f.write(f">sym{i} x\n{''.join(s)}\n")


def fastq(path):
    rng = np.random.default_rng(14)
    with open(path, "w") as f:
        for i in range(300):
            s = bytearray(_random(rng, int(rng.integers(40, 700))))
            if i % 6 == 0:
                s[5:50] = b"T" * 45
            if i % 4 == 0:
                s[10:20] = bytes(s[10:20]).lower()
            q = bytes(33 + int(x) for x in rng.integers(0, 41, size=len(s)))
            f.write(f"@fq{i} read\n{s.decode()}\n+\n{q.decode()}\n")


def all_short(path):
    rng = np.random.default_rng(15)
    with open(path, "w") as f:
        for i in range(25):
            f.write(f">short{i}\n{_random(rng, int(rng.integers(1, 32))).decode()}\n")


def many(path):
    """72 000 records of 60..180 nt; every 100th is a 200-nt homopolymer (one word with more windows than a small
    scratch budget holds when --dbmask none leaves it unmasked)"""
    rng = np.random.default_rng(16)
    ls = rng.integers(60, 181, size=72000)
    with open(path, "w") as f:
        for i in range(72000):
            s = b"A" * 200 if i % 100 == 7 else _random(rng, int(ls[i]))
            f.write(f">m{i}\n{s.decode()}\n")


INPUTS = {"mixed": (mixed, "fasta"), "lengths": (lengths, "fasta"), "symbols": (symbols, "fasta"), "fastq": (fastq, "fastq"),
          "all_short": (all_short, "fasta"), "many": (many, "fasta")}

# name: (input, CLI options, the same as vsg_makeudb_opts fields)
CASES = {
    "defaults": ("mixed", [], {}),
    "dbmask_none": ("mixed", ["--dbmask", "none"], dict(dbmask="none")),
    "dbmask_soft": ("mixed", ["--dbmask", "soft"], dict(dbmask="soft")),
    "dust_hardmask": ("mixed", ["--dbmask", "dust", "--hardmask"], dict(dbmask="dust", hardmask=1)),
    "soft_hardmask": ("mixed", ["--dbmask", "soft", "--hardmask"], dict(dbmask="soft", hardmask=1)),
    "k3": ("mixed", ["--wordlength", "3"], dict(wordlength=3)),
    "k10": ("mixed", ["--wordlength", "10"], dict(wordlength=10)),
    "k11": ("mixed", ["--wordlength", "11"], dict(wordlength=11)),
    "k12": ("mixed", ["--wordlength", "12"], dict(wordlength=12)),
    "notrunclabels": ("mixed", ["--notrunclabels"], dict(notrunclabels=1)),
    "lengths_default": ("lengths", [], {}),
    "lengths_wide": ("lengths", ["--minseqlength", "1", "--maxseqlength", "100000"], dict(minseqlength=1, maxseqlength=100000)),
    "symbols": ("symbols", [], {}),
    "fastq": ("fastq", [], {}),
    "all_discarded": ("all_short", [], {}),
    "many": ("many", [], {}),
    "many_none_k12": ("many", ["--dbmask", "none", "--wordlength", "12"], dict(dbmask="none", wordlength=12)),
}


def sha256(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 20), b""):
            h.update(b)
    return h.hexdigest()


@functools.lru_cache(maxsize=None)
def input_file(name, directory):
    fn, ext = INPUTS[name]
    path = os.path.join(directory, f"{name}.{ext}")
    if not os.path.exists(path):
        fn(path)
    return path


def reference_makeudb(inp, out, cli):
    r = subprocess.run([STOCK, "--makeudb_usearch", inp, "--output", out, "--quiet", *cli], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]


SEARCH_MASKS = ("dust", "none")
SEARCH_CLI = ["--id", "0.9", "--threads", "1", "--quiet", "--qmask", "none", "--maxaccepts", "2", "--maxrejects", "16"]


def search_inputs(directory):
    """test_udb_gpu.py's database (600 records, seed 8) and 1 500 mutated 200-nt queries"""
    import pathlib
    from test_udb_cpu import make_db
    fasta, seqs = make_db(pathlib.Path(directory), n=600, seed=8)
    rng = np.random.default_rng(3)
    qf = os.path.join(directory, "q.fasta")
    with open(qf, "w") as f:
        for i in range(1500):
            s = seqs[int(rng.integers(0, len(seqs)))].upper()
            a = int(rng.integers(0, max(1, len(s) - 120)))
            q = synth.mutate(rng, np.frombuffer(s[a:a + 200], dtype=np.uint8), 0.04).tobytes()
            f.write(f">q{i}\n{q.decode()}\n")
    return fasta, qf


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


if __name__ == "__main__":   # regenerate the golden file from oracle/_ref/vsearch
    import sys
    import tempfile
    d = tempfile.mkdtemp()
    out = {}
    for name, (inp, cli, _) in CASES.items():
        p = input_file(inp, d)
        udb = os.path.join(d, name + ".udb")
        reference_makeudb(p, udb, cli)
        out[name] = {"input_sha256": sha256(p), "sha256": sha256(udb), "size": os.path.getsize(udb)}
        print(name, out[name], file=sys.stderr)
    fasta, qf = search_inputs(d)
    for m in SEARCH_MASKS:
        udb = os.path.join(d, f"search_{m}.udb")
        reference_makeudb(fasta, udb, ["--dbmask", m])
        b6 = os.path.join(d, f"search_{m}.b6")
        r = subprocess.run([STOCK, "--usearch_global", qf, "--db", udb, "--blast6out", b6, *SEARCH_CLI], capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        out[f"search_{m}"] = {"input_sha256": sha256(fasta) + sha256(qf), "sha256": sha256(b6), "size": os.path.getsize(b6)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
