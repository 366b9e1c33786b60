"""The --uchime_ref cases shared by test_uchime_cpu.py, test_uchime_gpu.py and tools/make_uchime_golden.py: seeded synthetic
references and queries (two- and three-segment chimeras of the references, point-mutated non-chimeras, unrelated and
very short queries), the option sets, and the reference CLI's results in tests/golden/uchime_reference.json under the
case name: the sha256 of both inputs, of every file `vsearch --uchime_ref ... --threads 1` wrote, and the counts of its
summary.  The reference's own api_examples chimera data are fixtures under tests/golden/uchime/ (case "api_example").
tools/make_uchime_golden.py regenerates the golden file from oracle/_ref/vsearch."""
from __future__ import annotations

import hashlib
import json
import os
import re
import subprocess

import numpy as np

import checkers

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "uchime_reference.json")
FIXTURES = os.path.join(checkers.ROOT, "tests", "golden", "uchime")
STOCK = os.path.join(checkers.ROOT, "oracle", "_ref", "vsearch")
OUTPUTS = ("chimeras", "nonchimeras", "borderline", "uchimeout", "uchimealns")


def _seq(rng, n):
    return bytes(rng.choice(list(b"ACGT"), size=n).astype(np.uint8).tobytes())


def _mutate(rng, s: bytes, k: int) -> bytes:
    """k random point substitutions"""
    b = bytearray(s)
    for _ in range(k):
        p = int(rng.integers(0, len(b)))
        b[p] = b"ACGT"[(b"ACGT".index(b[p] & ~0x20 if b[p] >= 97 else b[p]) + 1 + int(rng.integers(0, 3))) % 4]
    return bytes(b)


def _write_fasta(path, labels, seqs, width=70):
    with open(path, "w") as f:
        for lab, s in zip(labels, seqs):
            t = bytes(s).decode()
            f.write(">" + lab + "\n")
            for a in range(0, max(len(t), 1), width):
                f.write(t[a:a + width] + "\n")


def _family(rng, n, length):
    """n references of about `length` nt: a few roots, each with diverged members (5-15 % apart)"""
    roots = [_seq(rng, length + int(rng.integers(-10, 10))) for _ in range(max(1, n // 5))]
    refs = []
    for i in range(n):
        r = roots[i % len(roots)]
        refs.append(_mutate(rng, r, int(len(r) * rng.uniform(0.05, 0.15))) if i >= len(roots) else r)
    return refs


def _queries(rng, refs, n, three=0.3, clean=0.3, junk=0.1):
    """chimeras of two or three references (cut at random points), mutated copies of one reference, unrelated sequences"""
    out, kinds = [], []
    for _ in range(n):
        u = rng.random()
        if u < junk:
            out.append(_seq(rng, int(rng.integers(150, 260)))); kinds.append("junk")
        elif u < junk + clean:
            r = refs[int(rng.integers(0, len(refs)))]
            out.append(_mutate(rng, r, int(rng.integers(0, 6)))); kinds.append("clean")
        else:
            k = 3 if rng.random() < three else 2
            pick = rng.choice(len(refs), size=k, replace=False)
            L = min(len(refs[int(p)]) for p in pick)
            cuts = sorted(int(c) for c in rng.choice(np.arange(30, L - 30), size=k - 1, replace=False))
            bounds = [0] + cuts + [None]
            s = b"".join(refs[int(pick[j])][bounds[j]:bounds[j + 1]] for j in range(k))
            out.append(_mutate(rng, s, int(rng.integers(0, 3)))); kinds.append(f"chim{k}")
    return out, kinds


def _soft(rng, s: bytes, share=0.15) -> bytes:
    """lower-case a few stretches"""
    b = bytearray(s)
    for _ in range(int(len(b) * share / 12) + 1):
        p = int(rng.integers(0, max(1, len(b) - 12)))
        b[p:p + 12] = bytes(b[p:p + 12]).lower()
    return bytes(b)


def _sizes(rng, n):
    return [int(x) for x in np.clip(rng.pareto(1.2, size=n) * 5 + 1, 1, 100000).astype(np.int64)]


def amplicons(d, seed=5, nref=60, nq=150, length=250, soft=False, iupac=False, short=False, selfq=False):
    rng = np.random.default_rng(seed)
    refs = _family(rng, nref, length)
    qs, kinds = _queries(rng, refs, nq)
    if soft:
        refs = [_soft(rng, r) for r in refs]
        qs = [_soft(rng, q) for q in qs]
    if iupac:
        for i in range(0, len(qs), 7):
            b = bytearray(qs[i])
            for _ in range(3):
                b[int(rng.integers(0, len(b)))] = b"RYKMSWNBDHV"[int(rng.integers(0, 11))]
            qs[i] = bytes(b).replace(b"T", b"U", 1)
    qlab = [f"q{i};size={s}" for i, s in enumerate(_sizes(rng, len(qs)))]
    rlab = [f"r{i};size={s}" for i, s in enumerate(_sizes(rng, len(refs)))]
    if short:
        qs += [b"", b"A", b"ACG", b"ACGT", b"ACGTACGTAC"]
        qlab += ["short0", "short1", "short3", "short4", "short10"]
    if selfq:
        for i in range(0, len(refs), 5):
            qs.append(refs[i]); qlab.append(rlab[i])
    q = os.path.join(d, "queries.fasta")
    r = os.path.join(d, "db.fasta")
    _write_fasta(q, qlab, qs)
    _write_fasta(r, rlab, refs)
    return q, r


def api_example(d):
    return os.path.join(FIXTURES, "chimera_queries.fasta"), os.path.join(FIXTURES, "chimera_ref.fasta")


def empty(d):
    q, r = amplicons(d, seed=9, nref=20, nq=1)
    open(q, "w").close()
    return q, r


def _write_fastq(path, labels, seqs):
    with open(path, "w") as f:
        for lab, s in zip(labels, seqs):
            f.write("@" + lab + "\n" + bytes(s).decode() + "\n+\n" + "I" * len(s) + "\n")


def zotus(d, seed=21, nparent=40, nchim=60, nclean=40, length=250, soft=False, iupac=False, fastq=False, short=False,
          equal=False, collision=0):
    """a de novo input: parents at high abundance, two- and three-segment chimeras and point-mutated copies at low
    abundance; `equal`: every abundance 1 (ordered by label); `collision`: that many near-identical copies of one
    parent at abundance 2, among which chimeras of that parent sit"""
    rng = np.random.default_rng(seed)
    parents = _family(rng, nparent, length)
    seqs, sizes = list(parents), [int(x) for x in rng.integers(200, 2000, size=nparent)]
    chims, _ = _queries(rng, parents, nchim, clean=0.0, junk=0.0)
    seqs += chims; sizes += [int(x) for x in rng.integers(1, 30, size=nchim)]
    seqs += [_mutate(rng, parents[int(rng.integers(0, nparent))], int(rng.integers(1, 4))) for _ in range(nclean)]
    sizes += [int(x) for x in rng.integers(1, 60, size=nclean)]
    if collision:
        base = parents[0]
        for i in range(collision):
            seqs.append(_mutate(rng, base, 1 + i % 3)); sizes.append(2)
            if i % 4 == 3:
                other = parents[1 + int(rng.integers(0, nparent - 1))]
                cut = int(rng.integers(60, length - 60))
                seqs.append(base[:cut] + other[cut:]); sizes.append(2)
    if soft:
        seqs = [_soft(rng, x) for x in seqs]
    if iupac:
        for i in range(0, len(seqs), 9):
            b = bytearray(seqs[i])
            b[int(rng.integers(0, len(b)))] = b"RYKMSWNBDHV"[int(rng.integers(0, 11))]
            seqs[i] = bytes(b).replace(b"T", b"U", 1)
    if equal:
        sizes = [1] * len(seqs)
    if short:
        seqs += [b"A", b"ACG", b"ACGT", b"ACGTACGTAC"]; sizes += [5, 5, 5, 5]
    order = rng.permutation(len(seqs))
    labels = [f"z{int(i)};size={sizes[int(i)]}" for i in order]
    seqs = [seqs[int(i)] for i in order]
    q = os.path.join(d, "input.fastq" if fastq else "input.fasta")
    (_write_fastq if fastq else _write_fasta)(q, labels, seqs)
    return q, None


# name -> (input maker, keyword options as vsg_uchime_opts fields / CLI options; "command" names a de novo command)
CASES = {
    "a_default": (lambda d: amplicons(d), {}),
    "a_minh_mindiv": (lambda d: amplicons(d, seed=6), {"minh": 0.1, "mindiv": 0.3, "mindiffs": 2, "xn": 6.0, "dn": 1.0}),
    "a_outputs": (lambda d: amplicons(d, seed=7), {"uchimeout5": 1, "alignwidth": 60, "fasta_score": 1, "sizeout": 1, "xsize": 1,
                                                    "fasta_width": 0}),
    "a_alignwidth0": (lambda d: amplicons(d, seed=8), {"alignwidth": 0}),
    "dbmask_none": (lambda d: amplicons(d, seed=10, soft=True), {"dbmask": "none", "qmask": "none"}),
    "dbmask_soft": (lambda d: amplicons(d, seed=11, soft=True), {"dbmask": "soft", "qmask": "soft"}),
    "soft_hardmask": (lambda d: amplicons(d, seed=12, soft=True), {"dbmask": "soft", "qmask": "soft", "hardmask": 1}),
    "dust_soft_input": (lambda d: amplicons(d, seed=13, soft=True), {}),
    "iupac_short": (lambda d: amplicons(d, seed=14, iupac=True, short=True), {}),
    "self": (lambda d: amplicons(d, seed=15, selfq=True), {"self": 1}),
    "selfid": (lambda d: amplicons(d, seed=16, selfq=True), {"selfid": 1}),
    "long_refs": (lambda d: amplicons(d, seed=17, nref=30, nq=60, length=1400), {}),
    "empty": (empty, {}),
    "api_example": (api_example, {}),
    "dn_uchime": (lambda d: zotus(d), {"command": "uchime_denovo"}),
    "dn_uchime2": (lambda d: zotus(d, seed=22), {"command": "uchime2_denovo"}),
    "dn_uchime3": (lambda d: zotus(d, seed=23), {"command": "uchime3_denovo"}),
    "dn_params": (lambda d: zotus(d, seed=24), {"command": "uchime_denovo", "abskew": 1.5, "xn": 7.0, "dn": 1.2, "minh": 0.2,
                                               "mindiv": 0.5, "mindiffs": 2}),
    "dn_abskew1": (lambda d: zotus(d, seed=25), {"command": "uchime_denovo", "abskew": 1.0}),
    "dn_equal": (lambda d: zotus(d, seed=26, equal=True), {"command": "uchime_denovo", "abskew": 1.0}),
    "dn_equal3": (lambda d: zotus(d, seed=27, equal=True), {"command": "uchime3_denovo"}),
    "dn_collision": (lambda d: zotus(d, seed=28, collision=80), {"command": "uchime3_denovo"}),
    "dn_collision1": (lambda d: zotus(d, seed=29, collision=60), {"command": "uchime_denovo"}),
    "dn_soft": (lambda d: zotus(d, seed=30, soft=True), {"command": "uchime_denovo", "qmask": "soft"}),
    "dn_none": (lambda d: zotus(d, seed=31, soft=True), {"command": "uchime2_denovo", "qmask": "none"}),
    "dn_hardmask": (lambda d: zotus(d, seed=32, soft=True), {"command": "uchime_denovo", "qmask": "soft", "hardmask": 1}),
    "dn_dust_soft": (lambda d: zotus(d, seed=33, soft=True), {"command": "uchime3_denovo"}),
    "dn_fastq_iupac": (lambda d: zotus(d, seed=34, fastq=True, iupac=True, short=True), {"command": "uchime_denovo"}),
    "dn_outputs": (lambda d: zotus(d, seed=35), {"command": "uchime_denovo", "uchimeout5": 1, "alignwidth": 60, "fasta_score": 1,
                                                "sizeout": 1, "xsize": 1, "fasta_width": 0}),
    "dn_alignwidth0": (lambda d: zotus(d, seed=36), {"command": "uchime2_denovo", "alignwidth": 0, "fasta_score": 1}),
    "dn_discarded": (lambda d: zotus(d, seed=37), {"command": "uchime_denovo", "minseqlength": 1000}),
}

DENOVO = sorted(k for k, v in CASES.items() if "command" in v[1])

def cli_args(opts):
    """the reference CLI's options for a case's option set"""
    a = []
    for k, v in opts.items():
        if k == "command":
            continue
        if k in ("qmask", "dbmask"):
            a += [f"--{k}", v]
        elif k in ("hardmask", "self", "selfid", "uchimeout5", "fasta_score", "sizeout", "xsize"):
            if v:
                a.append(f"--{k}")
        else:
            a += [f"--{k}", str(v)]
    return a


def sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def run_reference(name, d):
    """run the reference CLI on case `name` in directory d: (record, {output: path})"""
    make, opts = CASES[name]
    q, r = make(d)
    paths = {k: os.path.join(d, "ref." + k) for k in OUTPUTS}
    if "command" in opts:
        cmd = [STOCK, "--" + opts["command"], q, "--threads", "1"] + cli_args(opts)
    else:
        cmd = [STOCK, "--uchime_ref", q, "--db", r, "--threads", "1"] + cli_args(opts)
    for k, p in paths.items():
        cmd += [f"--{k}", p]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(p.stderr)
    counts = summary(p.stderr)
    rec = {"query_sha256": sha(q), "db_sha256": sha(r) if r else None, "files": {k: sha(v) for k, v in paths.items()}, "counts": counts}
    return rec, paths


def summary(stderr):
    """the counts of the reference's 'Found ... chimeras' summary"""
    m = re.search(r"Found (\d+)(?: \([\d.]+%\))? chimeras, (\d+)(?: \([\d.]+%\))? non-chimeras,\s*and (\d+)(?: \([\d.]+%\))? "
                  r"borderline sequences in (\d+) unique", stderr)
    a = re.search(r"this corresponds to\s*(\d+)(?: \([\d.]+%\))? chimeras, (\d+)(?: \([\d.]+%\))? non-chimeras,\s*and (\d+)"
                  r"(?: \([\d.]+%\))? borderline sequences in (\d+) total", stderr)
    return {"chimeras": int(m.group(1)), "nonchimeras": int(m.group(2)), "borderline": int(m.group(3)), "queries": int(m.group(4)),
            "chimeras_abundance": int(a.group(1)), "nonchimeras_abundance": int(a.group(2)),
            "borderline_abundance": int(a.group(3)), "queries_abundance": int(a.group(4))}


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def make_golden():
    import tempfile
    out = {}
    for name in CASES:
        with tempfile.TemporaryDirectory() as d:
            out[name], _ = run_reference(name, d)
            print(name, out[name]["counts"])
    with open(GOLDEN, "w") as f:
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, sort_keys=True, separators=(',', ':'))}" for k, v in out.items()) + "\n}\n")
