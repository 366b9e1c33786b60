"""The --search_exact cases shared by test_search_exact_cpu.py, test_search_exact_gpu.py and tools: seeded synthetic
queries and databases, the option sets, and the reference CLI's results in tests/golden/search_exact_reference.json under
the case name: the sha256 of both inputs, of every file `vsearch --search_exact ... --threads 1` wrote, and the counts of
its summary.  Run as a script to regenerate the golden file from oracle/_ref/vsearch."""
from __future__ import annotations

import functools
import hashlib
import json
import os
import re
import subprocess

import numpy as np

import checkers

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "search_exact_reference.json")
STOCK = os.path.join(checkers.ROOT, "oracle", "_ref", "vsearch")
OUTPUTS = ("blast6out", "uc", "matched", "notmatched", "dbmatched", "dbnotmatched", "otutabout", "mothur_shared_out")

_COMP = bytes.maketrans(b"ACGTURYKMBVDHSWNacgturykmbvdhswn", b"TGCAAYRMKVBHDSWNtgcaayrmkvbhdswn")


def revcomp(s: bytes) -> bytes:
    return bytes(s).translate(_COMP)[::-1]


def _seq(rng, n):
    return bytes(rng.choice(list(b"ACGT"), size=n).astype(np.uint8).tobytes())


def _mutate(rng, s: bytes) -> bytes:
    b = bytearray(s)
    p = int(rng.integers(0, len(b)))
    b[p] = b"ACGT"[(b"ACGT".index(b[p]) + 1) % 4]
    return bytes(b)


def _write_fasta(path, labels, seqs, width=70):
    with open(path, "w") as f:
        for lab, s in zip(labels, seqs):
            t = bytes(s).decode()
            f.write(">" + lab + "\n")
            for a in range(0, len(t), width):
                f.write(t[a:a + width] + "\n")


def _zotus(rng, n, lo=200, hi=260):
    return [_seq(rng, int(rng.integers(lo, hi))) for _ in range(n)]


def _reads(rng, zotus, n, rc=0.0):
    """n reads: 60 % exact copies of a ZOTU (a share rc of them reverse-complemented), 25 % one mutation, the rest random"""
    out = []
    for _ in range(n):
        z = zotus[int(rng.integers(0, len(zotus)))]
        u = rng.random()
        if u < 0.6:
            out.append(revcomp(z) if rng.random() < rc else z)
        elif u < 0.85:
            out.append(_mutate(rng, z))
        else:
            out.append(_seq(rng, len(z)))
    return out


def amplicons(d):
    """ZOTUs with ;size= on most, otu= / tax= on some; reads with ;sample= in 7 samples"""
    rng = np.random.default_rng(41)
    zotus = _zotus(rng, 60)
    labels = []
    for i in range(len(zotus)):
        lab = f"Zotu{i + 1}"
        if i % 4 != 3:
            lab += f";size={int(rng.integers(1, 50))}"
        if i % 5 == 0:
            lab += f";otu=OTU_{i // 10}"
        if i % 3 == 0:
            lab += f";tax=d:Bacteria,p:P{i % 4},g:G{i % 7}"
        labels.append(lab)
    reads = _reads(rng, zotus, 700)
    _write_fasta(os.path.join(d, "amplicons.db.fasta"), labels, zotus)
    _write_fasta(os.path.join(d, "amplicons.q.fasta"), [f"r{i};sample=S{i % 7}" for i in range(len(reads))], reads)


def strands(d):
    """a tenth of the reads reverse-complemented; palindromic sequences (s + revcomp(s)) in the database and the reads"""
    rng = np.random.default_rng(42)
    zotus = _zotus(rng, 40)
    pal = [(lambda h: h + revcomp(h))(_seq(rng, int(rng.integers(60, 130)))) for _ in range(8)]
    db = zotus + pal + [pal[0], revcomp(zotus[3])]
    reads = _reads(rng, zotus, 400, rc=0.1) + pal + [revcomp(p) for p in pal[:3]]
    _write_fasta(os.path.join(d, "strands.db.fasta"), [f"t{i}" for i in range(len(db))], db)
    _write_fasta(os.path.join(d, "strands.q.fasta"), [f"q{i};sample=A{i % 3}" for i in range(len(reads))], reads)


def duplicates(d):
    """one sequence 3 000 times in the database, others under several labels; reads hit them and miss"""
    rng = np.random.default_rng(43)
    zotus = _zotus(rng, 20)
    db, labels = [], []
    for i in range(3000):
        db.append(zotus[0])
        labels.append(f"dup{i}")
    for i, z in enumerate(zotus[1:]):
        for k in range(1 + i % 4):
            db.append(z)
            labels.append(f"z{i}_{k};otu=Z{i}")
    order = rng.permutation(len(db))
    db = [db[int(k)] for k in order]
    labels = [labels[int(k)] for k in order]
    reads = _reads(rng, zotus, 120, rc=0.2)
    _write_fasta(os.path.join(d, "duplicates.db.fasta"), labels, db)
    _write_fasta(os.path.join(d, "duplicates.q.fasta"), [f"d{i}" for i in range(len(reads))], reads)


def _mixed_case(rng, s: bytes) -> bytes:
    b = bytearray(s)
    a = int(rng.integers(0, len(b) - 30))
    b[a:a + 25] = bytes(b[a:a + 25]).lower()
    return bytes(b)


def symbols(d):
    """lower and mixed case, U for T, N / R / Y on both sides; some matches exist only up to case and U / T"""
    rng = np.random.default_rng(44)
    zotus = _zotus(rng, 40)
    db = []
    for i, z in enumerate(zotus):
        b = bytearray(z)
        if i % 5 == 0:
            for c in b"NRY":
                b[int(rng.integers(0, len(b)))] = c
        if i % 3 == 0:
            b = bytearray(_mixed_case(rng, bytes(b)))
        db.append(bytes(b))
    reads = []
    for i in range(300):
        z = db[int(rng.integers(0, len(db)))]
        u = rng.random()
        if u < 0.3:
            reads.append(z.lower())
        elif u < 0.5:
            reads.append(z.upper().replace(b"T", b"U"))
        elif u < 0.7:
            reads.append(_mixed_case(rng, z.upper()))
        elif u < 0.8:
            b = bytearray(z.upper())
            b[int(rng.integers(0, len(b)))] = ord("N")
            reads.append(bytes(b))
        else:
            reads.append(z)
    _write_fasta(os.path.join(d, "symbols.db.fasta"), [f"s{i}" for i in range(len(db))], db)
    _write_fasta(os.path.join(d, "symbols.q.fasta"), [f"y{i}" for i in range(len(reads))], reads)


def sizes(d):
    """;size= on some reads and targets, barcodelabel= and prefix-only samples"""
    rng = np.random.default_rng(45)
    zotus = _zotus(rng, 30)
    labels = [f"Z{i}" + (f";size={int(rng.integers(1, 30))}" if i % 3 else "") for i in range(len(zotus))]
    reads = _reads(rng, zotus, 300)
    rl = []
    for i in range(len(reads)):
        size = f";size={int(rng.integers(1, 20))}" if i % 4 else ""
        if i % 3 == 0:
            rl.append(f"r{i};barcodelabel=B{i % 5}{size}")
        elif i % 3 == 1:
            rl.append(f"Sam{i % 4}.r{i}{size}")
        else:
            rl.append(f"x{i}{size};sample=P{i % 2}")
    _write_fasta(os.path.join(d, "sizes.db.fasta"), labels, zotus)
    _write_fasta(os.path.join(d, "sizes.q.fasta"), rl, reads)


def selfish(d):
    """queries that are database records under the same label, and under other labels"""
    rng = np.random.default_rng(46)
    zotus = _zotus(rng, 30)
    labels = [f"L{i};size={int(rng.integers(1, 9))}" for i in range(len(zotus))] + ["L0;size=2", "M1"]
    db = zotus + [zotus[0], zotus[1]]
    reads, rl = [], []
    for i in range(200):
        k = int(rng.integers(0, len(zotus)))
        reads.append(zotus[k])
        rl.append(labels[k] if i % 2 else f"Q{i};size={int(rng.integers(1, 12))}")
    _write_fasta(os.path.join(d, "selfish.db.fasta"), labels, db)
    _write_fasta(os.path.join(d, "selfish.q.fasta"), rl, reads)


def described(d):
    """headers with a description after a blank"""
    rng = np.random.default_rng(47)
    zotus = _zotus(rng, 25)
    reads = _reads(rng, zotus, 150)
    _write_fasta(os.path.join(d, "described.db.fasta"), [f"D{i};size={i + 1} the target {i}" for i in range(len(zotus))], zotus)
    _write_fasta(os.path.join(d, "described.q.fasta"), [f"q{i};sample=s{i % 2} read {i} of x" for i in range(len(reads))],
                 reads, width=50)


def edges(d):
    """empty query records, queries longer than every target, database records of 10..400 nt"""
    rng = np.random.default_rng(48)
    db = [_seq(rng, int(rng.integers(10, 400))) for _ in range(60)]
    reads, rl = [], []
    for i in range(120):
        u = i % 6
        if u == 0:
            reads.append(b"")
        elif u == 1:
            reads.append(_seq(rng, 500))
        else:
            reads.append(db[int(rng.integers(0, len(db)))])
        rl.append(f"e{i}")
    _write_fasta(os.path.join(d, "edges.db.fasta"), [f"E{i}" for i in range(len(db))], db)
    _write_fasta(os.path.join(d, "edges.q.fasta"), rl, reads)


def fastq(d):
    """FASTQ queries against FASTA targets"""
    rng = np.random.default_rng(49)
    zotus = _zotus(rng, 30)
    reads = _reads(rng, zotus, 200, rc=0.1)
    _write_fasta(os.path.join(d, "fastq.db.fasta"), [f"F{i};size={i + 2}" for i in range(len(zotus))], zotus)
    with open(os.path.join(d, "fastq.q.fastq"), "w") as f:
        for i, s in enumerate(reads):
            q = bytes(33 + int(x) for x in rng.integers(0, 41, size=len(s)))
            f.write(f"@fq{i};sample=F{i % 3} x\n{s.decode()}\n+\n{q.decode()}\n")


def dusty(d):
    """ZOTUs and reads with a 60-nt AT repeat that DUST masks, for the printed case of the masked files"""
    rng = np.random.default_rng(50)
    zotus = _zotus(rng, 30)
    zotus = [z[:80] + b"AT" * 30 + z[80:] if i % 3 == 0 else z for i, z in enumerate(zotus)]
    reads = _reads(rng, zotus, 200)
    _write_fasta(os.path.join(d, "dusty.db.fasta"), [f"U{i}" for i in range(len(zotus))], zotus)
    _write_fasta(os.path.join(d, "dusty.q.fasta"), [f"u{i};sample=K{i % 2}" for i in range(len(reads))], reads)


INPUTS = {"amplicons": (amplicons, "fasta"), "strands": (strands, "fasta"), "duplicates": (duplicates, "fasta"),
          "symbols": (symbols, "fasta"), "sizes": (sizes, "fasta"), "selfish": (selfish, "fasta"),
          "described": (described, "fasta"), "edges": (edges, "fasta"), "fastq": (fastq, "fastq"), "dusty": (dusty, "fasta")}

ALL = OUTPUTS
# name: (input, CLI options, the same as search_exact_command keywords, outputs)
CASES = {
    "a_default": ("amplicons", [], {}, ALL),
    "b_strand_both": ("strands", ["--strand", "both", "--uc_allhits"], dict(strand_both=1, uc_allhits=1), ALL),
    "c_dups_all": ("duplicates", ["--strand", "both", "--output_no_hits"], dict(strand_both=1, output_no_hits=1),
                   ("blast6out", "uc", "dbmatched", "otutabout")),
    "d_dups_maxhits5": ("duplicates", ["--maxhits", "5", "--uc_allhits", "--output_no_hits", "--sizeout"],
                        dict(maxhits=5, uc_allhits=1, output_no_hits=1, sizeout=1), ALL),
    "e_symbols_none": ("symbols", ["--qmask", "none", "--dbmask", "none"], dict(qmask="none", dbmask="none"), ALL),
    "f_symbols_soft": ("symbols", ["--qmask", "soft", "--dbmask", "none", "--strand", "both"],
                       dict(qmask="soft", dbmask="none", strand_both=1), ALL),
    "g_hardmask": ("symbols", ["--qmask", "soft", "--dbmask", "soft", "--hardmask"], dict(qmask="soft", dbmask="soft", hardmask=1),
                   ALL),
    "h_sizes": ("sizes", ["--sizein", "--sizeout"], dict(sizein=1, sizeout=1), ALL),
    "i_xsize": ("sizes", ["--sizeout", "--xsize"], dict(sizeout=1, xsize=1), ALL),
    "j_self": ("selfish", ["--self", "--sizein"], dict(self=1, sizein=1), ALL),
    "k_tsize": ("selfish", ["--mintsize", "3", "--maxqsize", "8"], dict(mintsize=3, maxqsize=8), ("blast6out", "uc", "otutabout")),
    "l_ratio": ("selfish", ["--minsizeratio", "0.5", "--maxsizeratio", "2"], dict(minsizeratio=0.5, maxsizeratio=2.0),
                ("blast6out", "uc", "dbmatched")),
    "m_notrunc_w0": ("described", ["--notrunclabels", "--fasta_width", "0", "--sizeout"], dict(notrunclabels=1, fasta_width=0, sizeout=1),
                     ALL),
    "n_width60": ("described", ["--fasta_width", "60"], dict(fasta_width=60), ALL),
    "o_edges": ("edges", ["--minseqlength", "50", "--maxseqlength", "300", "--output_no_hits"],
                dict(minseqlength=50, maxseqlength=300, output_no_hits=1), ALL),
    "p_fastq": ("fastq", ["--strand", "both", "--sizein", "--sizeout"], dict(strand_both=1, sizein=1, sizeout=1), ALL),
    "q_dust": ("dusty", ["--strand", "both"], dict(strand_both=1), ALL),
}

# the case built to exercise DUST's masked regions; the CPU oracle, which does not restate DUST, skips it
DUST_CASES = ("q_dust",)

_FLAGS = {"blast6out": "--blast6out", "uc": "--uc", "matched": "--matched", "notmatched": "--notmatched",
          "dbmatched": "--dbmatched", "dbnotmatched": "--dbnotmatched", "otutabout": "--otutabout",
          "mothur_shared_out": "--mothur_shared_out"}


def sha256_bytes(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def sha256(path):
    with open(path, "rb") as f:
        return sha256_bytes(f.read())


@functools.lru_cache(maxsize=None)
def input_files(name, directory):
    """(query path, database path) of input `name` in `directory`, made on first use"""
    fn, ext = INPUTS[name]
    q = os.path.join(directory, f"{name}.q.{ext}")
    db = os.path.join(directory, f"{name}.db.fasta")
    if not os.path.exists(q):
        fn(directory)
    return q, db


def output_files(directory, name, outputs):
    return {o: os.path.join(directory, f"{name}.{o}") for o in outputs}


def output_digests(paths):
    return {o: sha256(p) for o, p in paths.items()}


def reference_run(q, db, cli, paths):
    """runs the reference CLI; returns the counts of its summary"""
    args = [STOCK, "--search_exact", q, "--db", db, "--threads", "1", *cli]
    for o, p in paths.items():
        args += [_FLAGS[o], p]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    m = re.search(r"Matching unique query sequences: (\d+) of (\d+)", r.stderr)
    return {"matched": int(m.group(1)), "queries": int(m.group(2))}


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


if __name__ == "__main__":   # regenerate the golden file from oracle/_ref/vsearch
    import sys
    import tempfile
    d = tempfile.mkdtemp()
    out = {}
    for name, (inp, cli, kw, outputs) in CASES.items():
        q, db = input_files(inp, d)
        sub = os.path.join(d, name)
        os.makedirs(sub)
        paths = output_files(sub, name, outputs)
        counts = reference_run(q, db, cli, paths)
        out[name] = {"query_sha256": sha256(q), "db_sha256": sha256(db), "files": output_digests(paths), **counts}
        print(name, counts, file=sys.stderr)
    with open(GOLDEN, "w") as f:   # one case per line
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(out[k], separators=(",", ":"), sort_keys=True)
                                    for k in sorted(out)) + "\n}\n")
