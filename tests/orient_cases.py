"""The --orient parity cases shared by test_orient_cpu.py and test_orient_gpu.py: the synthetic reads and database
(synth.orient_data), the option sets (a)-(i), their input files, a numpy restatement of the vote, and the reference
CLI's results, stored in tests/golden/orient_reference.json under a name and a hash of the inputs (as
sintax_cases.reference keys its records).  A record holds the digest of every output file, the (strand, count_fwd,
count_rev) rows of --tabbedout and the three summary counts; for the --dbmask dust cases also the DUST mask of the
database, as `vsearch --maskfasta --qmask dust` writes it."""
from __future__ import annotations

import functools
import gzip
import hashlib
import json
import os
import re
import subprocess

import numpy as np

import checkers
from vsearch_b200 import synth

GOLDEN = os.path.join(checkers.ROOT, "tests", "golden", "orient_reference.json")
UDB_GZ = os.path.join(checkers.ROOT, "tests", "golden", "orient_db8.udb.gz")
UDB_SEQS = 200   # the UDB file holds the first 200 database sequences (four families)

OUTS = ("fastaout", "fastqout", "notmatched", "tabbedout")
# name: CLI options; k = the index's word length; dbmask / qmask / hardmask as given to the CLI; fastq: FASTQ reads;
# udb: the database is the UDB file (made with --wordlength 8); outs: the output files
CASES = {
    "a_defaults": dict(k=12, dbmask="dust", qmask="dust", hardmask=False, fastq=False, udb=False, width=80, notrunc=False,
                       outs=("fastaout", "notmatched", "tabbedout"), opts=[]),
    "b_fastq": dict(k=12, dbmask="dust", qmask="dust", hardmask=False, fastq=True, udb=False, width=80, notrunc=False,
                    outs=OUTS, opts=[]),
    "c_k8_nomask": dict(k=8, dbmask="none", qmask="none", hardmask=False, fastq=False, udb=False, width=80, notrunc=False,
                        outs=("fastaout", "notmatched", "tabbedout"),
                        opts=["--wordlength", "8", "--dbmask", "none", "--qmask", "none"]),
    "d_soft_hardmask": dict(k=12, dbmask="soft", qmask="soft", hardmask=True, fastq=False, udb=False, width=80, notrunc=False,
                            outs=("fastaout", "notmatched", "tabbedout"),
                            opts=["--dbmask", "soft", "--hardmask", "--qmask", "soft"]),
    "e_k13": dict(k=13, dbmask="dust", qmask="dust", hardmask=False, fastq=False, udb=False, width=80, notrunc=False,
                  outs=("fastaout", "notmatched", "tabbedout"), opts=["--wordlength", "13"]),
    "f_udb8": dict(k=8, dbmask="udb", qmask="dust", hardmask=False, fastq=False, udb=True, width=80, notrunc=False,
                   outs=("fastaout", "notmatched", "tabbedout"), opts=[]),
    "g_width0_notrunc": dict(k=12, dbmask="dust", qmask="dust", hardmask=False, fastq=False, udb=False, width=0, notrunc=True,
                             outs=("fastaout", "notmatched", "tabbedout"), opts=["--fasta_width", "0", "--notrunclabels"]),
    # the small and the large end of the dense index.  At k = 4 every k-mer of data()'s database is about as common as its
    # reverse complement, so h_k4 pins only the outcome "no read is oriented" (and the output files); the votes at
    # k = 3..6 are pinned on biased_data() by biased_reference below
    "h_k4": dict(k=4, dbmask="dust", qmask="dust", hardmask=False, fastq=False, udb=False, width=80, notrunc=False,
                 outs=("fastaout", "notmatched", "tabbedout"), opts=["--wordlength", "4"]),
    "i_k10": dict(k=10, dbmask="dust", qmask="dust", hardmask=False, fastq=False, udb=False, width=80, notrunc=False,
                  outs=("fastaout", "notmatched", "tabbedout"), opts=["--wordlength", "10"]),
}


@functools.lru_cache(maxsize=None)
def data():
    return synth.orient_data()


@functools.lru_cache(maxsize=None)
def biased_data():
    """A database whose k-mers are strand-biased at every word length, so that reads are oriented even at k = 3..6: 300
    targets of 60 nt drawn 45 % A, 45 % C, 5 % G, 5 % T (an A/C-rich k-mer is common, its G/T-rich reverse complement
    rare), every 7th with a lower-case stretch and every 11th with an N.  Reads: mutated 40-nt windows of the targets on
    either strand, joins of a forward and a reverse-complemented window, A/C-rich and uniform random reads, reads with a
    lower-case stretch, and two reads shorter than 3 nt.  Returns dict(db (a (300, 60) ASCII matrix), db_heads, db_seqs,
    q_heads, q_seqs)."""
    rng = np.random.default_rng(97)
    m = synth.ACGT[rng.choice(4, size=(300, 60), p=[0.45, 0.45, 0.05, 0.05])]
    m[::7, 20:35] += ord("a") - ord("A")
    m[3::11, 30] = ord("N")

    def window():
        s = m[int(rng.integers(0, 300))]
        a = int(rng.integers(0, 21))
        return synth.mutate(rng, s[a:a + 40], 0.02).tobytes()
    q = []
    for i in range(150):
        kind = i % 6
        if kind in (0, 1):
            q.append(window())
        elif kind == 2:
            q.append(synth.revcomp(window()))
        elif kind == 3:
            a, b = window(), synth.revcomp(window())
            q.append(a[:24] + b[:16] if i % 12 == 3 else b[:24] + a[:16])
        elif kind == 4:
            r = synth.ACGT[rng.choice(4, size=40, p=[0.45, 0.45, 0.05, 0.05])].tobytes()
            q.append(synth.revcomp(r) if i % 12 == 4 else r)
        else:
            r = bytearray(synth.random_seqs(rng, 1, 40)[0].tobytes() if i % 12 == 5 else window())
            r[10:25] = bytes(r[10:25]).lower()
            q.append(bytes(r))
    q += [b"AC", b"A"]
    return dict(db=m, db_heads=[f"b{i}" for i in range(300)], db_seqs=[r.tobytes() for r in m],
                q_heads=[f"q{i}" for i in range(len(q))], q_seqs=q)


def run_biased_cli(k, mask, tmp):
    """(reference CLI) the --tabbedout rows of `vsearch --orient` on biased_data() with --dbmask and --qmask `mask`"""
    d = biased_data()
    dbf, qf, tab = os.path.join(tmp, "bdb.fa"), os.path.join(tmp, "bq.fa"), os.path.join(tmp, "b.tsv")
    synth.write_records(dbf, d["db_heads"], d["db_seqs"])
    synth.write_records(qf, d["q_heads"], d["q_seqs"])
    p = subprocess.run([checkers.STOCK, "--orient", qf, "--db", dbf, "--threads", "1", "--wordlength", str(k),
                        "--dbmask", mask, "--qmask", mask, "--tabbedout", tab, "--quiet"],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    return parse_rows(open(tab, "rb").read())


def biased_reference(k, mask, compute=None):
    """the stored rows of run_biased_cli(k, mask)"""
    d = biased_data()
    h = hashlib.sha256()
    checkers._feed(h, [k, mask, d["db_heads"], d["db_seqs"], d["q_heads"], d["q_seqs"]])
    return _record(f"orient_biased:k{k}_{mask}:{h.hexdigest()[:24]}", compute)


def write_inputs(tmp):
    """(database FASTA, reads FASTA, reads FASTQ)"""
    d = data()
    dbf, qa, qq = os.path.join(tmp, "db.fa"), os.path.join(tmp, "reads.fa"), os.path.join(tmp, "reads.fq")
    synth.write_records(dbf, d["db_heads"], d["db_seqs"])
    synth.write_records(qa, d["q_heads"], d["q_seqs"])
    synth.write_fastq(qq, d["q_heads"], d["q_seqs"], d["q_quals"])
    return dbf, qa, qq


def udb_path(tmp):
    """the first UDB_SEQS database sequences as `vsearch --makeudb_usearch --wordlength 8` wrote them (stored gzipped)"""
    out = os.path.join(tmp, "db8.udb")
    with gzip.open(UDB_GZ, "rb") as f, open(out, "wb") as g:
        g.write(f.read())
    return out


def make_udb(tmp):
    """(reference CLI) the UDB file of the first UDB_SEQS database sequences, gzipped into tests/golden"""
    d = data()
    fa, out = os.path.join(tmp, "db_udb.fa"), os.path.join(tmp, "db8.udb")
    synth.write_records(fa, d["db_heads"][:UDB_SEQS], d["db_seqs"][:UDB_SEQS])
    p = subprocess.run([checkers.STOCK, "--makeudb_usearch", fa, "--output", out, "--wordlength", "8", "--quiet"],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    with open(out, "rb") as f, gzip.GzipFile(UDB_GZ, "wb", mtime=0) as g:
        g.write(f.read())


def reference_available():
    return os.path.exists(checkers.STOCK)


def cli_args(case, dbf, qf, outs):
    c = CASES[case]
    a = ["--orient", qf, "--db", dbf, "--threads", "1"] + c["opts"]
    for o in c["outs"]:
        a += ["--" + o, outs[o]]
    return a


def parse_rows(tsv: bytes):
    """--tabbedout -> [[strand 0/1/2, count_fwd, count_rev], ...]"""
    rows = []
    for line in tsv.decode().splitlines():
        f = line.split("\t")
        rows.append(["+-?".index(f[-3]), int(f[-2]), int(f[-1])])
    return rows


def run_cli(case, tmp):
    """the reference CLI on the case: the record stored for it"""
    dbf, qa, qq = write_inputs(tmp)
    c = CASES[case]
    if c["udb"]:
        dbf = udb_path(tmp)
    outs = {o: os.path.join(tmp, f"{case}.ref.{o}") for o in c["outs"]}
    p = subprocess.run([checkers.STOCK] + cli_args(case, dbf, qq if c["fastq"] else qa, outs), capture_output=True,
                       text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-2000:]
    summary = [int(re.search(pat + r"\s+(\d+)", p.stderr).group(1))
               for pat in ("Forward oriented sequences:", "Reverse oriented sequences:", "Not oriented sequences:")]
    files = {o: checkers.digest(open(outs[o], "rb").read()) for o in c["outs"]}
    rec = {"files": files, "rows": parse_rows(open(outs["tabbedout"], "rb").read()), "summary": summary}
    if c["dbmask"] == "dust":
        rec["dust"] = dust_intervals(tmp, dbf)
    return rec


def dust_intervals(tmp, dbf):
    """(reference CLI) the database's DUST mask as [sequence, start, end) intervals"""
    out = os.path.join(tmp, "db.dust.fa")
    p = subprocess.run([checkers.STOCK, "--maskfasta", dbf, "--qmask", "dust", "--output", out, "--fasta_width", "0",
                        "--quiet"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    seqs = open(out, "rb").read().split(b"\n")[1::2]
    iv = []
    for i, s in enumerate(seqs):
        for m in re.finditer(rb"[a-z]+", s):
            iv.append([i, m.start(), m.end()])
    return iv


def _inputs(case):
    d = data()
    return [case, sorted(CASES[case].items()), d["db_heads"], d["db_seqs"], d["q_heads"], d["q_seqs"], d["q_quals"]]


_stored = None


def reference(case, compute=None):
    """the stored reference record of `case`; VSG_RECORD_REFERENCE=1 with the compiled reference present recomputes it
    (compute()) and writes it to tests/golden/orient_reference.json"""
    h = hashlib.sha256()
    checkers._feed(h, _inputs(case))
    return _record(f"orient:{case}:{h.hexdigest()[:24]}", compute)


def _record(key, compute):
    global _stored
    if os.environ.get("VSG_RECORD_REFERENCE") and reference_available() and compute is not None:
        val = compute()
        rec = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
        rec[key] = val
        with open(GOLDEN, "w") as f:
            json.dump(rec, f, indent=0, sort_keys=True)
            f.write("\n")
        _stored = rec
        return val
    if _stored is None:
        _stored = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
    assert key in _stored, f"no stored reference result {key} in {GOLDEN}"
    return _stored[key]


# ---- a numpy restatement of the vote (orient.cpp:224-312), for the CPU tests ----------------------------------------------
_CODE = np.full(256, -1, dtype=np.int64)
for _ch, _v in zip(b"ACGTUacgtu", (0, 1, 2, 3, 3, 0, 1, 2, 3, 3)):
    _CODE[_ch] = _v


def kmers(seq: bytes, k: int, skip_lower: bool) -> np.ndarray:
    """the k-mers of the windows with only ACGTU symbols (and no lower-case one when skip_lower), as unique_count keeps
    them (the set: the vote does not depend on the order)"""
    a = np.frombuffer(seq, dtype=np.uint8)
    n = a.shape[0] - k + 1
    if n <= 0:
        return np.zeros(0, dtype=np.int64)
    code = _CODE[a]
    bad = code < 0
    if skip_lower:
        bad |= (a >= ord("a")) & (a <= ord("z"))
    v = np.zeros(n, dtype=np.int64)
    nbad = np.zeros(n, dtype=np.int64)
    for j in range(k):
        v = (v << 2) | np.maximum(code[j:j + n], 0)
        nbad += bad[j:j + n]
    return np.unique(v[nbad == 0])


def rc_kmers(v: np.ndarray, k: int) -> np.ndarray:
    r = np.zeros_like(v)
    x = v.copy()
    for _ in range(k):
        r = (r << 2) | ((x & 3) ^ 3)
        x >>= 2
    return r


def database_as_indexed(case, dust=None):
    """the database sequences the reference indexes for `case` and whether lower case is left out of the index"""
    c = CASES[case]
    seqs = list(data()["db_seqs"])
    if c["dbmask"] == "dust":
        seqs = [bytearray(s.upper()) for s in seqs]
        for i, a, b in dust:
            seqs[i][a:b] = bytes(seqs[i][a:b]).lower()
        return [bytes(s) for s in seqs], True
    if c["hardmask"]:
        return [re.sub(rb"[a-z]", b"N", s) for s in seqs], True
    return seqs, c["dbmask"] != "none"


def word_counts(seqs, k, skip_lower):
    """(sorted k-mers, the number of sequences holding each)"""
    allk = np.concatenate([kmers(s, k, skip_lower) for s in seqs] + [np.zeros(0, dtype=np.int64)])
    return np.unique(allk, return_counts=True)


def orient_rows(queries, k, qmask_lower, words, counts):
    """[[strand, count_fwd, count_rev], ...] of every query against the word counts"""
    def lookup(v):
        i = np.searchsorted(words, v)
        i = np.minimum(i, max(words.shape[0] - 1, 0))
        return np.where((words.shape[0] > 0) & (words[i] == v), counts[i], 0).astype(np.int64)
    rows = []
    for s in queries:
        w = kmers(s, k, qmask_lower)
        f, r = lookup(w), lookup(rc_kmers(w, k))
        cf = int((f > 8 * r).sum())
        cr = int(((f <= 8 * r) & (r > 8 * f)).sum())
        strand = 0 if cf >= 1 and cf >= 4 * cr else 1 if cr >= 1 and cr >= 4 * cf else 2
        rows.append([strand, cf, cr])
    return rows
