"""The --chimeras_denovo cases shared by test_chimeras_denovo_cpu.py, test_chimeras_denovo_gpu.py and
tools/make_chimeras_denovo_golden.py: seeded long reads (800 to 3 000 nt, in families whose members are 3 to 15 % apart,
with a few indels), chimeras of 2 to 6 segments of one family, point-mutated copies, unrelated reads, and the option
sets.  tests/golden/chimeras_denovo_reference.json holds, under the case name, the sha256 of the input and of every file
`vsearch --chimeras_denovo ... --threads 1` wrote, and the counts of its summary."""
from __future__ import annotations

import json
import os
import re
import subprocess

import numpy as np

import checkers
import uchime_cases as U

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "chimeras_denovo_reference.json")
STOCK = U.STOCK
# vsg_uchime_outputs slot -> the reference CLI's option
OUTPUTS = {"chimeras": "chimeras", "nonchimeras": "nonchimeras", "uchimeout": "tabbedout", "uchimealns": "alnout"}
CLI_ONLY = ("sizein",)   # options of the reference CLI that vsg_uchime_opts has no field for (abundances are always read)


def _indels(rng, s: bytes, k: int) -> bytes:
    """k random insertions or deletions of 1 to 4 nt"""
    b = bytearray(s)
    for _ in range(k):
        p = int(rng.integers(0, len(b)))
        n = int(rng.integers(1, 5))
        if rng.random() < 0.5:
            b[p:p] = U._seq(rng, n)
        else:
            del b[p:p + n]
    return bytes(b)


def _families(rng, nfam, per, lo, hi):
    """nfam roots of lo..hi nt, each with `per` members 3 to 15 % apart from it (the root is the first member)"""
    fams = []
    for _ in range(nfam):
        root = U._seq(rng, int(rng.integers(lo, hi + 1)))
        mem = [root]
        for _ in range(per - 1):
            m = U._mutate(rng, root, int(len(root) * rng.uniform(0.03, 0.15)))
            mem.append(_indels(rng, m, int(rng.integers(0, 4))))
        fams.append(mem)
    return fams


def _chimera(rng, fam, k, minseg):
    """k segments of k different members of a family, cut at common fractions of their lengths, each at least minseg"""
    pick = [fam[int(i)] for i in rng.choice(len(fam), size=min(k, len(fam)), replace=False)]
    k = len(pick)
    L = min(len(p) for p in pick)
    minseg = min(minseg, L // (2 * k))
    while True:
        cuts = sorted(int(c) for c in rng.choice(np.arange(1, L), size=k - 1, replace=False))
        b = [0] + cuts + [L]
        if min(b[i + 1] - b[i] for i in range(k)) >= minseg:
            break
    frac = [c / L for c in b]
    return b"".join(p[int(frac[i] * len(p)):int(frac[i + 1] * len(p))] for i, p in enumerate(pick))


def reads(d, seed=1, nfam=4, per=5, nchim=24, nclean=10, njunk=3, lo=800, hi=3000, maxseg=6, minseg=10, identical=0,
          equal=False, soft=False, iupac=False, fastq=False, short=False):
    """a long-read input: family members at high abundance, chimeras of 2..maxseg segments and mutated copies at low
    abundance, unrelated reads; `identical`: that many families get a copy of one member under another label, at the same
    abundance; `equal`: every abundance 2"""
    rng = np.random.default_rng(seed)
    fams = _families(rng, nfam, per, lo, hi)
    seqs, sizes = [], []
    for f in fams:
        for m in f:
            seqs.append(m); sizes.append(int(rng.integers(200, 2000)))
    for i in range(identical):
        seqs.append(fams[i % nfam][1]); sizes.append(sizes[(i % nfam) * per + 1])
    for _ in range(nchim):
        k = int(rng.integers(2, maxseg + 1))
        ms = minseg if rng.random() < 0.3 else 150
        c = _chimera(rng, fams[int(rng.integers(0, nfam))], k, ms)
        seqs.append(U._mutate(rng, c, int(rng.integers(0, 3)))); sizes.append(int(rng.integers(1, 30)))
    for _ in range(nclean):
        f = fams[int(rng.integers(0, nfam))]
        seqs.append(U._mutate(rng, f[int(rng.integers(0, per))], int(rng.integers(1, 6)))); sizes.append(int(rng.integers(1, 60)))
    for _ in range(njunk):
        seqs.append(U._seq(rng, int(rng.integers(lo, hi + 1)))); sizes.append(int(rng.integers(1, 10)))
    if soft:
        seqs = [U._soft(rng, x, 0.05) for x in seqs]
    if iupac:
        for i in range(0, len(seqs), 5):
            b = bytearray(seqs[i])
            for _ in range(4):
                b[int(rng.integers(0, len(b)))] = b"RYKMSWNBDHV"[int(rng.integers(0, 11))]
            seqs[i] = bytes(b).replace(b"T", b"U", 1)
    if equal:
        sizes = [2] * len(seqs)
    if short:
        seqs += [b"A", b"ACGTA", b"ACGTACG", b"ACGTACGTACGTACGTACGT"]; sizes += [5, 5, 5, 5]
    order = rng.permutation(len(seqs))
    labels = [f"r{int(i)};size={sizes[int(i)]}" for i in order]
    if identical:
        # the copies carry labels that sort before their originals', so the tie order decides which one is the parent
        labels = [("a" + lab if int(i) >= nfam * per and int(i) < nfam * per + identical else lab) for lab, i in zip(labels, order)]
    seqs = [seqs[int(i)] for i in order]
    q = os.path.join(d, "input.fastq" if fastq else "input.fasta")
    (U._write_fastq if fastq else U._write_fasta)(q, labels, seqs)
    return q


def empty(d):
    q = os.path.join(d, "input.fasta")
    open(q, "w").close()
    return q


C = "chimeras_denovo"
# name -> (input maker, keyword options as vsg_uchime_opts fields / CLI options)
CASES = {
    "cd_default": (lambda d: reads(d), {}),
    "cd_parents2": (lambda d: reads(d, seed=2), {"chimeras_parents_max": 2}),
    "cd_parents5": (lambda d: reads(d, seed=3), {"chimeras_parents_max": 5}),
    "cd_parents20": (lambda d: reads(d, seed=4, per=8), {"chimeras_parents_max": 20, "chimeras_length_min": 1}),
    "cd_diff03": (lambda d: reads(d, seed=5), {"chimeras_diff_pct": 0.3}),
    "cd_diff15": (lambda d: reads(d, seed=6), {"chimeras_diff_pct": 1.5, "chimeras_parents_max": 5}),
    "cd_diff50": (lambda d: reads(d, seed=7), {"chimeras_diff_pct": 50.0}),
    "cd_lenmin1": (lambda d: reads(d, seed=8), {"chimeras_length_min": 1}),
    "cd_lenmin200": (lambda d: reads(d, seed=9), {"chimeras_length_min": 200}),
    "cd_parts2": (lambda d: reads(d, seed=10), {"chimeras_parts": 2}),
    "cd_parts7": (lambda d: reads(d, seed=11), {"chimeras_parts": 7}),
    "cd_parts100": (lambda d: reads(d, seed=12), {"chimeras_parts": 100}),
    "cd_abskew2": (lambda d: reads(d, seed=13), {"abskew": 2.0}),
    "cd_qmask_none": (lambda d: reads(d, seed=14, soft=True), {"qmask": "none"}),
    "cd_qmask_soft": (lambda d: reads(d, seed=15, soft=True), {"qmask": "soft"}),
    "cd_qmask_dust": (lambda d: reads(d, seed=16, soft=True), {"qmask": "dust"}),
    "cd_hardmask": (lambda d: reads(d, seed=17, soft=True), {"qmask": "soft", "hardmask": 1}),
    "cd_outputs": (lambda d: reads(d, seed=18), {"sizein": 1, "sizeout": 1, "xsize": 1, "notrunclabels": 1, "fasta_width": 0,
                                                 "alignwidth": 0}),
    "cd_identical": (lambda d: reads(d, seed=19, identical=4), {"chimeras_parents_max": 4}),
    "cd_equal": (lambda d: reads(d, seed=20, equal=True, nchim=30), {"abskew": 2.0}),
    "cd_short_iupac_fastq": (lambda d: reads(d, seed=21, iupac=True, fastq=True, short=True), {"chimeras_parts": 7}),
    "cd_empty": (empty, {}),
    "cd_collision": (lambda d: reads(d, seed=22, equal=True, nchim=30), {"chimeras_diff_pct": 1.5}),
    "cd_iupac_soft_chimeras": (lambda d: reads(d, seed=23, iupac=True, soft=True), {"chimeras_diff_pct": 1.5, "qmask": "soft"}),
}


def cli_args(opts):
    """the reference CLI's options for a case's option set"""
    a = []
    for k, v in opts.items():
        if k == "qmask":
            a += ["--qmask", v]
        elif k in ("hardmask", "sizein", "sizeout", "xsize", "notrunclabels"):
            if v:
                a.append(f"--{k}")
        else:
            a += [f"--{k}", str(v)]
    return a


def api_opts(opts):
    """a case's options as vsg_uchime_opts fields"""
    return {k: v for k, v in opts.items() if k not in CLI_ONLY}


def run_reference(name, d):
    """run the reference CLI on case `name` in directory d: (record, {output slot: path})"""
    make, opts = CASES[name]
    q = make(d)
    paths = {k: os.path.join(d, "ref." + k) for k in OUTPUTS}
    cmd = [STOCK, "--chimeras_denovo", q, "--threads", "1"] + cli_args(opts)
    for k, p in paths.items():
        cmd += [f"--{OUTPUTS[k]}", p]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(p.stderr)
    rec = {"query_sha256": U.sha(q), "files": {k: U.sha(v) for k, v in paths.items()}, "counts": summary(p.stderr)}
    return rec, paths


def summary(stderr):
    """the counts of the reference's 'Found ... chimeras and ... non-chimeras' summary (all zero when it has none)"""
    m = re.search(r"Found (\d+)(?: \([\d.]+%\))? chimeras and (\d+)(?: \([\d.]+%\))? non-chimeras\s*in (\d+) unique", stderr)
    a = re.search(r"this corresponds to\s*(\d+)(?: \([\d.]+%\))? chimeras(?:,| and) (\d+)(?: \([\d.]+%\))? non-chimeras\s*"
                  r"in (\d+) total", stderr)
    if m is None or a is None:
        return {"chimeras": 0, "nonchimeras": 0, "queries": 0, "chimeras_abundance": 0, "nonchimeras_abundance": 0,
                "queries_abundance": 0, "borderline": 0}
    return {"chimeras": int(m.group(1)), "nonchimeras": int(m.group(2)), "queries": int(m.group(3)),
            "chimeras_abundance": int(a.group(1)), "nonchimeras_abundance": int(a.group(2)),
            "queries_abundance": int(a.group(3)), "borderline": 0}


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
