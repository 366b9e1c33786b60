"""The --usearch_global cases shared by test_usearch_global_cpu.py, test_usearch_global_gpu.py and tools: seeded synthetic
queries and databases, the option sets, and the reference CLI's results in tests/golden/usearch_global_reference.json
under the case name: the sha256 of both inputs, of every file `vsearch --usearch_global ... --threads 1` wrote, the counts
of its summary, and every query's full hit list (target number, strand, identity as printed, CIGAR or "=") from a second
run with every hit in --uc (no --maxhits, --uc_allhits, no --top_hits_only).  A case whose database is "udb" searches the
UDB file `vsearch --makeudb_usearch` makes of the input's database; its sha256 is recorded as "udb_sha256".  Run as a
script to regenerate the golden file from oracle/_ref/vsearch."""
from __future__ import annotations

import functools
import hashlib
import json
import os
import re
import subprocess

import numpy as np

import checkers

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "usearch_global_reference.json")
STOCK = os.path.join(checkers.ROOT, "oracle", "_ref", "vsearch")
OUTPUTS = ("blast6out", "uc", "matched", "notmatched", "dbmatched", "dbnotmatched", "otutabout", "mothur_shared_out")

_COMP = bytes.maketrans(b"ACGTURYKMBVDHSWNacgturykmbvdhswn", b"TGCAAYRMKVBHDSWNtgcaayrmkvbhdswn")


def revcomp(s: bytes) -> bytes:
    return bytes(s).translate(_COMP)[::-1]


def _seq(rng, n):
    return bytes(rng.choice(list(b"ACGT"), size=n).astype(np.uint8).tobytes())


def _mutate(rng, s: bytes, k: int) -> bytes:
    """k random edits: substitutions, single-base insertions and deletions"""
    b = bytearray(s)
    for _ in range(k):
        p = int(rng.integers(1, len(b) - 1))
        u = rng.random()
        if u < 0.6:
            b[p] = b"ACGT"[(b"ACGT".index(b[p]) + 1 + int(rng.integers(0, 3))) % 4]
        elif u < 0.8:
            b.insert(p, b"ACGT"[int(rng.integers(0, 4))])
        else:
            del b[p]
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


def _reads(rng, zotus, n, rc=0.0, edits=(0, 1, 2, 4, 9, 20)):
    """n reads from the ZOTUs with a number of edits drawn from `edits` (a share rc reverse-complemented), one in eight random"""
    out = []
    for _ in range(n):
        z = zotus[int(rng.integers(0, len(zotus)))]
        if rng.random() < 0.125:
            out.append(_seq(rng, len(z)))
            continue
        r = _mutate(rng, z, int(edits[int(rng.integers(0, len(edits)))]))
        out.append(revcomp(r) if rng.random() < rc else r)
    return out


def amplicons(d):
    """ZOTUs with ;size= on most, otu= / tax= on some, a few near-identical pairs; reads with ;sample= in 7 samples"""
    rng = np.random.default_rng(61)
    zotus = _zotus(rng, 70)
    zotus += [_mutate(rng, zotus[i], 2) for i in range(0, 10)]
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
    reads = _reads(rng, zotus, 600)
    _write_fasta(os.path.join(d, "amplicons.db.fasta"), labels, zotus)
    _write_fasta(os.path.join(d, "amplicons.q.fasta"), [f"r{i};sample=S{i % 7}" for i in range(len(reads))], reads)


def strands(d):
    """a third of the reads reverse-complemented"""
    rng = np.random.default_rng(62)
    zotus = _zotus(rng, 50)
    reads = _reads(rng, zotus, 400, rc=0.33)
    _write_fasta(os.path.join(d, "strands.db.fasta"), [f"t{i};size={i + 1}" for i in range(len(zotus))], zotus)
    _write_fasta(os.path.join(d, "strands.q.fasta"), [f"q{i};sample=A{i % 3}" for i in range(len(reads))], reads)


def ties(d):
    """identical ZOTUs under several labels and families of close variants, so hits tie and top hits differ"""
    rng = np.random.default_rng(63)
    base = _zotus(rng, 20)
    db, labels = [], []
    for i, z in enumerate(base):
        for k in range(1 + i % 3):
            db.append(z)
            labels.append(f"z{i}_{k};size={k + 1}")
        for k in range(i % 4):
            db.append(_mutate(rng, z, 1 + k))
            labels.append(f"v{i}_{k}")
    order = rng.permutation(len(db))
    db = [db[int(k)] for k in order]
    labels = [labels[int(k)] for k in order]
    reads = _reads(rng, base, 300, rc=0.2, edits=(0, 1, 3, 6))
    _write_fasta(os.path.join(d, "ties.db.fasta"), labels, db)
    _write_fasta(os.path.join(d, "ties.q.fasta"), [f"t{i};sample=T{i % 4}" for i in range(len(reads))], reads)


def _mixed_case(rng, s: bytes) -> bytes:
    b = bytearray(s)
    a = int(rng.integers(0, len(b) - 40))
    b[a:a + 30] = bytes(b[a:a + 30]).lower()
    return bytes(b)


def symbols(d):
    """lower-case stretches and N / R / Y on both sides"""
    rng = np.random.default_rng(64)
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
        z = _mutate(rng, zotus[int(rng.integers(0, len(zotus)))], int(rng.integers(0, 5)))
        u = rng.random()
        if u < 0.3:
            z = _mixed_case(rng, z)
        elif u < 0.4:
            z = z.lower()
        reads.append(z)
    _write_fasta(os.path.join(d, "symbols.db.fasta"), [f"s{i}" for i in range(len(db))], db)
    _write_fasta(os.path.join(d, "symbols.q.fasta"), [f"y{i};sample=Y{i % 2}" for i in range(len(reads))], reads)


def sizes(d):
    """;size= on some reads and targets, barcodelabel= and prefix-only samples, a description after a blank"""
    rng = np.random.default_rng(65)
    zotus = _zotus(rng, 30)
    labels = [f"Z{i}" + (f";size={int(rng.integers(1, 30))}" if i % 3 else "") + " desc" for i in range(len(zotus))]
    reads = _reads(rng, zotus, 300)
    rl = []
    for i in range(len(reads)):
        size = f";size={int(rng.integers(1, 20))}" if i % 4 else ""
        if i % 3 == 0:
            rl.append(f"r{i};barcodelabel=B{i % 5}{size}")
        elif i % 3 == 1:
            rl.append(f"Sam{i % 4}.r{i}{size}")
        else:
            rl.append(f"x{i}{size};sample=P{i % 2} read {i}")
    _write_fasta(os.path.join(d, "sizes.db.fasta"), labels, zotus)
    _write_fasta(os.path.join(d, "sizes.q.fasta"), rl, reads)


def selfish(d):
    """queries that are database records under the same label, and under other labels"""
    rng = np.random.default_rng(66)
    zotus = _zotus(rng, 30)
    zotus += [_mutate(rng, z, 1) for z in zotus[:10]]
    labels = [f"L{i};size={int(rng.integers(1, 9))}" for i in range(len(zotus))]
    reads, rl = [], []
    for i in range(200):
        k = int(rng.integers(0, len(zotus)))
        reads.append(zotus[k] if i % 3 else _mutate(rng, zotus[k], 1))
        rl.append(labels[k] if i % 2 else f"Q{i};size={int(rng.integers(1, 12))}")
    _write_fasta(os.path.join(d, "selfish.db.fasta"), labels, zotus)
    _write_fasta(os.path.join(d, "selfish.q.fasta"), rl, reads)


def edges(d):
    """database records of 10..400 nt (those under 32 discarded by default), queries shorter and longer than the targets"""
    rng = np.random.default_rng(67)
    db = [_seq(rng, int(rng.integers(10, 400))) for _ in range(80)]
    reads = []
    for i in range(200):
        t = db[int(rng.integers(0, len(db)))]
        u = i % 5
        if u == 0:
            reads.append(t[: max(20, len(t) * 2 // 3)])
        elif u == 1:
            reads.append(t + _seq(rng, 30))
        else:
            reads.append(_mutate(rng, t, int(rng.integers(0, 3))) if len(t) > 3 else t)
    _write_fasta(os.path.join(d, "edges.db.fasta"), [f"E{i}" for i in range(len(db))], db)
    _write_fasta(os.path.join(d, "edges.q.fasta"), [f"e{i}" for i in range(len(reads))], reads)


def fastq(d):
    """FASTQ queries against FASTA targets"""
    rng = np.random.default_rng(68)
    zotus = _zotus(rng, 30)
    reads = _reads(rng, zotus, 200, rc=0.2)
    _write_fasta(os.path.join(d, "fastq.db.fasta"), [f"F{i};size={i + 2}" for i in range(len(zotus))], zotus)
    with open(os.path.join(d, "fastq.q.fastq"), "w") as f:
        for i, s in enumerate(reads):
            q = bytes(33 + int(x) for x in rng.integers(0, 41, size=len(s)))
            f.write(f"@fq{i};sample=F{i % 3} x\n{s.decode()}\n+\n{q.decode()}\n")


def dusty(d):
    """ZOTUs and reads with a 60-nt AT repeat that DUST masks"""
    rng = np.random.default_rng(69)
    zotus = _zotus(rng, 30)
    zotus = [z[:80] + b"AT" * 30 + z[80:] if i % 3 == 0 else z for i, z in enumerate(zotus)]
    reads = _reads(rng, zotus, 200, rc=0.2)
    _write_fasta(os.path.join(d, "dusty.db.fasta"), [f"U{i};size={i + 1}" for i in range(len(zotus))], zotus)
    _write_fasta(os.path.join(d, "dusty.q.fasta"), [f"u{i};sample=K{i % 2}" for i in range(len(reads))], reads)


INPUTS = {"amplicons": (amplicons, "fasta"), "strands": (strands, "fasta"), "ties": (ties, "fasta"), "symbols": (symbols, "fasta"),
          "sizes": (sizes, "fasta"), "selfish": (selfish, "fasta"), "edges": (edges, "fasta"), "fastq": (fastq, "fastq"),
          "dusty": (dusty, "fasta")}

ALL = OUTPUTS
ID97 = (["--id", "0.97"], dict(id=0.97))
ID90 = (["--id", "0.9"], dict(id=0.9))


def _case(inp, idopt, cli, kw, outputs=ALL, db="fasta"):
    return (inp, idopt[0] + cli, {**idopt[1], **kw}, outputs, db)


# name: (input, CLI options, the same as usearch_global_command keywords, outputs, "fasta" or "udb" database)
CASES = {
    "a_default": _case("amplicons", ID97, [], {}),
    "b_strand_both": _case("strands", ID90, ["--strand", "both"], dict(strand_both=1)),
    "c_weak": _case("amplicons", ID97, ["--weak_id", "0.9", "--maxaccepts", "4"], dict(weak_id=0.9, maxaccepts=4)),
    "d_top_hits": _case("ties", ID90, ["--maxaccepts", "8", "--top_hits_only", "--uc_allhits", "--strand", "both"],
                        dict(maxaccepts=8, top_hits_only=1, uc_allhits=1, strand_both=1)),
    "e_maxhits2": _case("ties", ID90, ["--maxaccepts", "6", "--maxhits", "2", "--uc_allhits", "--output_no_hits"],
                        dict(maxaccepts=6, maxhits=2, uc_allhits=1, output_no_hits=1)),
    "f_exhaustive": _case("ties", ID90, ["--maxaccepts", "0", "--maxrejects", "0", "--uc_allhits"],
                          dict(maxaccepts=0, maxrejects=0, uc_allhits=1)),
    "g_mask_none": _case("symbols", ID90, ["--qmask", "none", "--dbmask", "none"], dict(qmask="none", dbmask="none")),
    "h_mask_soft": _case("symbols", ID90, ["--qmask", "soft", "--dbmask", "soft", "--strand", "both"],
                         dict(qmask="soft", dbmask="soft", strand_both=1)),
    "i_hardmask": _case("symbols", ID90, ["--qmask", "soft", "--dbmask", "soft", "--hardmask"],
                        dict(qmask="soft", dbmask="soft", hardmask=1)),
    "j_sizes": _case("sizes", ID90, ["--sizein", "--sizeout", "--xsize"], dict(sizein=1, sizeout=1, xsize=1)),
    "k_sizeout": _case("sizes", ID90, ["--sizeout", "--notrunclabels", "--fasta_width", "0"], dict(sizeout=1, notrunclabels=1, fasta_width=0)),
    "l_self": _case("selfish", ID90, ["--self", "--sizein", "--maxaccepts", "3"], dict(self=1, sizein=1, maxaccepts=3)),
    "m_selfid": _case("selfish", ID90, ["--selfid", "--maxaccepts", "3"], dict(selfid=1, maxaccepts=3)),
    "n_cov": _case("edges", ID90, ["--query_cov", "0.9", "--target_cov", "0.8", "--minqt", "0.8", "--maxqt", "1.2", "--output_no_hits"],
                   dict(query_cov=0.9, target_cov=0.8, minqt=0.8, maxqt=1.2, output_no_hits=1)),
    "o_edges": _case("edges", ID90, ["--minseqlength", "50", "--maxseqlength", "300", "--minsl", "0.7", "--maxdiffs", "3"],
                     dict(minseqlength=50, maxseqlength=300, minsl=0.7, maxdiffs=3)),
    "p_short_db": _case("edges", ID90, ["--strand", "both", "--uc_allhits", "--maxaccepts", "2"], dict(strand_both=1, uc_allhits=1, maxaccepts=2)),
    "q_fastq": _case("fastq", ID90, ["--strand", "both", "--sizein", "--sizeout"], dict(strand_both=1, sizein=1, sizeout=1)),
    "r_wordlength12": _case("amplicons", ID90, ["--wordlength", "12", "--maxaccepts", "2", "--uc_allhits"],
                            dict(wordlength=12, maxaccepts=2, uc_allhits=1)),
    "s_dust": _case("dusty", ID90, ["--strand", "both"], dict(strand_both=1)),
    "t_dust_soft": _case("dusty", ID90, ["--qmask", "dust", "--dbmask", "soft", "--sizeout"], dict(dbmask="soft", sizeout=1)),
    "u_udb": _case("amplicons", ID97, ["--strand", "both", "--weak_id", "0.9", "--maxaccepts", "2"],
                   dict(strand_both=1, weak_id=0.9, maxaccepts=2), db="udb"),
}



def dusted(name):
    """the files of case `name` that print DUST-masked sequences (a restatement without DUST cannot make them)"""
    inp, cli, kw, outputs, dbkind = CASES[name]
    return {o for o in outputs if (o in ("matched", "notmatched") and kw.get("qmask", "dust") == "dust")
            or (o in ("dbmatched", "dbnotmatched") and (kw.get("dbmask", "dust") == "dust" or dbkind == "udb"))}


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


def reference_makeudb(db, udb):
    r = subprocess.run([STOCK, "--makeudb_usearch", db, "--output", udb, "--threads", "1"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]


def reference_run(q, db, cli, paths):
    """runs the reference CLI; returns the counts of its summary"""
    args = [STOCK, "--usearch_global", q, "--db", db, "--threads", "1", *cli]
    for o, p in paths.items():
        args += [_FLAGS[o], p]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    m = re.search(r"Matching unique query sequences: (\d+) of (\d+)", r.stderr)
    return {"matched": int(m.group(1)), "queries": int(m.group(2))}


def hit_cli(cli):
    """the case's options with every hit shown in --uc"""
    out, i = [], 0
    while i < len(cli):
        if cli[i] == "--maxhits":
            i += 2
            continue
        if cli[i] not in ("--top_hits_only", "--uc_allhits", "--output_no_hits"):
            out.append(cli[i])
        i += 1
    return out + ["--uc_allhits"]


def parse_hits(uc_text):
    """every query's hits from an --uc_allhits file, in order: [[target, strand, id text, CIGAR or "="], ...] per query"""
    out = []
    prev = None
    for line in uc_text.splitlines():
        f = line.split("\t")
        if f[0] == "N":
            out.append([])
            prev = None
            continue
        key = f[8]
        h = [int(f[1]), 1 if f[4] == "-" else 0, f[3], f[7]]
        if prev is not None and prev == key and out:
            out[-1].append(h)
        else:
            out.append([h])
        prev = key
    return out


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


if __name__ == "__main__":   # regenerate the golden file from oracle/_ref/vsearch
    import sys
    import tempfile
    d = tempfile.mkdtemp()
    out = {}
    for name, (inp, cli, kw, outputs, dbkind) in CASES.items():
        q, db = input_files(inp, d)
        sub = os.path.join(d, name)
        os.makedirs(sub)
        entry = {"query_sha256": sha256(q), "db_sha256": sha256(db)}
        if dbkind == "udb":
            udb = os.path.join(sub, "db.udb")
            reference_makeudb(db, udb)
            entry["udb_sha256"] = sha256(udb)
            db = udb
        paths = output_files(sub, name, outputs)
        counts = reference_run(q, db, cli, paths)
        hp = os.path.join(sub, "hits.uc")
        reference_run(q, db, hit_cli(cli), {"uc": hp})
        hits = parse_hits(open(hp).read())
        assert len(hits) == counts["queries"], name
        out[name] = {**entry, "files": output_digests(paths), **counts, "hits": hits}
        print(name, counts, sum(len(h) for h in hits), file=sys.stderr)
    with open(GOLDEN, "w") as f:   # one case per line
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(out[k], separators=(",", ":"), sort_keys=True)
                                    for k in sorted(out)) + "\n}\n")
