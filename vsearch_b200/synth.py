"""Deterministic synthetic FASTA-shaped workloads (SURVEY.md §8(d)).

Alphabet uniform over ACGT; mutation operator ``mut(s, r)``: per base with probability
``r``: 80 % substitution (uniform base), 10 % deletion, 10 % insertion after the base.
Everything is generated with numpy's PCG64 from a fixed seed so that the CPU baseline,
the oracle and the GPU path all see byte-identical inputs.
"""
from __future__ import annotations

import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def random_seqs(rng: np.random.Generator, n: int, length: int) -> np.ndarray:
    """n iid sequences of a fixed length as an (n, length) uint8 ASCII matrix."""
    return ACGT[rng.integers(0, 4, size=(n, length), dtype=np.uint8)]


def mutate(rng: np.random.Generator, s: np.ndarray, r: float) -> np.ndarray:
    """mut(s, r) of SURVEY §8(d) on one ASCII uint8 sequence."""
    n = s.shape[0]
    hit = rng.random(n) < r
    kind = rng.random(n)
    sub = hit & (kind < 0.8)
    dele = hit & (kind >= 0.8) & (kind < 0.9)
    ins = hit & (kind >= 0.9)
    out = s.copy()
    out[sub] = ACGT[rng.integers(0, 4, size=int(sub.sum()), dtype=np.uint8)]
    # build with insertions after the base, deletions dropped
    reps = np.ones(n, dtype=np.int64)
    reps[dele] = 0
    reps[ins] = 2
    idx = np.repeat(np.arange(n), reps)
    res = out[idx]
    # second copy of an inserted position becomes a random base
    second = np.zeros(idx.shape[0], dtype=bool)
    if idx.shape[0] > 1:
        second[1:] = idx[1:] == idx[:-1]
    res[second] = ACGT[rng.integers(0, 4, size=int(second.sum()), dtype=np.uint8)]
    return res


class SeqSet:
    """Concatenated ASCII sequences + offsets/lengths (the layout Database::add builds,
    reference src/core/db.cpp:170-226, minus headers)."""

    def __init__(self, seqs):
        self.lens = np.array([len(s) for s in seqs], dtype=np.int32)
        self.offs = np.zeros(len(seqs), dtype=np.int64)
        if len(seqs):
            np.cumsum(self.lens[:-1], out=self.offs[1:])
        total = int(self.lens.sum())
        self.cat = np.empty(total + 1, dtype=np.uint8)
        self.cat[total] = 0
        pos = 0
        for s in seqs:
            a = np.frombuffer(s, dtype=np.uint8) if isinstance(s, (bytes, bytearray)) else np.asarray(s, dtype=np.uint8)
            self.cat[pos:pos + a.shape[0]] = a
            pos += a.shape[0]

    def __len__(self):
        return int(self.lens.shape[0])

    def seq(self, i: int) -> bytes:
        o = int(self.offs[i])
        return self.cat[o:o + int(self.lens[i])].tobytes()

    @classmethod
    def from_matrix(cls, m: np.ndarray) -> "SeqSet":
        self = cls.__new__(cls)
        n, L = m.shape
        self.lens = np.full(n, L, dtype=np.int32)
        self.offs = np.arange(n, dtype=np.int64) * L
        self.cat = np.empty(n * L + 1, dtype=np.uint8)
        self.cat[:-1] = m.reshape(-1)
        self.cat[-1] = 0
        return self


def config1_allpairs(n_reads: int = 1000, n_roots: int = 20, length: int = 200,
                     div: float = 0.10, seed: int = 12345) -> SeqSet:
    """C1: reads i = mut(root[i mod n_roots], div)."""
    rng = np.random.default_rng(seed)
    roots = random_seqs(rng, n_roots, length)
    return SeqSet([mutate(rng, roots[i % n_roots], div) for i in range(n_reads)])


def config2_search(n_db: int = 100_000, db_len: int = 1500, n_q: int = 1_000_000,
                   q_len: int = 250, div: float = 0.05, seed: int = 2024):
    """C2: DB iid; query = mut(window of a uniformly chosen DB sequence, div).
    Returns (db SeqSet, queries SeqSet, source target of every query)."""
    rng = np.random.default_rng(seed)
    dbm = random_seqs(rng, n_db, db_len)
    src = rng.integers(0, n_db, size=n_q)
    start = rng.integers(0, db_len - q_len + 1, size=n_q)
    qs = [mutate(rng, dbm[src[i], start[i]:start[i] + q_len], div) for i in range(n_q)]
    return SeqSet.from_matrix(dbm), SeqSet(qs), src


def config5_allpairs(n_reads: int = 200_000, n_roots: int = 2000, length: int = 400,
                     div: float = 0.15, seed: int = 5) -> SeqSet:
    rng = np.random.default_rng(seed)
    roots = random_seqs(rng, n_roots, length)
    pick = rng.integers(0, n_roots, size=n_reads)
    return SeqSet([mutate(rng, roots[pick[i]], div) for i in range(n_reads)])


def write_fasta(path: str, ss: SeqSet, prefix: str) -> None:
    with open(path, "wb") as f:
        for i in range(len(ss)):
            f.write(b">" + prefix.encode() + str(i).encode() + b"\n" + ss.seq(i) + b"\n")


def mutate_batch(rng: np.random.Generator, m: np.ndarray, r: float) -> SeqSet:
    """mut(., r) applied to every row of an (n, L) ASCII matrix at once (vectorised; the draw
    order differs from `mutate`, so the two generators give different — equally distributed —
    sequences for the same seed)."""
    n, L = m.shape
    hit = rng.random((n, L)) < r
    kind = rng.random((n, L))
    sub = hit & (kind < 0.8)
    dele = hit & (kind >= 0.8) & (kind < 0.9)
    ins = hit & (kind >= 0.9)
    out = m.copy()
    out[sub] = ACGT[rng.integers(0, 4, size=int(sub.sum()), dtype=np.uint8)]
    reps = np.ones((n, L), dtype=np.int64)
    reps[dele] = 0
    reps[ins] = 2
    flat_reps = reps.reshape(-1)
    idx = np.repeat(np.arange(n * L), flat_reps)
    res = out.reshape(-1)[idx]
    second = np.zeros(idx.shape[0], dtype=bool)
    if idx.shape[0] > 1:
        second[1:] = idx[1:] == idx[:-1]
    res[second] = ACGT[rng.integers(0, 4, size=int(second.sum()), dtype=np.uint8)]
    ss = SeqSet.__new__(SeqSet)
    ss.lens = reps.sum(axis=1).astype(np.int32)
    ss.offs = np.zeros(n, dtype=np.int64)
    np.cumsum(ss.lens[:-1], out=ss.offs[1:])
    ss.cat = np.empty(res.shape[0] + 1, dtype=np.uint8)
    ss.cat[:-1] = res
    ss.cat[-1] = 0
    return ss


def config2_db(n_db: int = 100_000, db_len: int = 1500, seed: int = 2024) -> np.ndarray:
    """C2 database as an (n_db, db_len) ASCII matrix."""
    return random_seqs(np.random.default_rng(seed), n_db, db_len)


def config2_query_batch(dbm: np.ndarray, n_q: int, q_len: int = 250, div: float = 0.05,
                        seed: int = 2024, batch: int = 0):
    """Batch `batch` of the C2 query stream: windows of uniformly chosen DB sequences, mut(., div).
    Returns (SeqSet, source target per query)."""
    rng = np.random.default_rng([seed, 7919, batch])
    n_db, db_len = dbm.shape
    src = rng.integers(0, n_db, size=n_q)
    start = rng.integers(0, db_len - q_len + 1, size=n_q)
    cols = start[:, None] + np.arange(q_len)[None, :]
    win = dbm[src[:, None], cols]
    return mutate_batch(rng, win, div), src


# ---- SINTAX: a taxonomy database and amplicon-shaped queries ------------------------------------------------------------
SINTAX_LEVELS = "dpcofgs"
_RC = bytes.maketrans(b"ACGTacgtNn", b"TGCAtgcaNn")


def revcomp(s: bytes) -> bytes:
    return s.translate(_RC)[::-1]


def sintax_data(seed: int = 77, length: int = 1450, fanout=(2, 2, 2, 2, 2, 2, 3), n_q: int = 300, q_len: int = 250):
    """A reference tree of ranks d, p, c, o, f, g, s: every node is a mutation of its parent (rates falling from 10 % at
    the domain to 2 % at the species), the species are ~`length`-nt leaves, and one species per genus is held out of
    the database.  The database (headers ``r{i};tax=d:...,s:...;``) also holds the header variants of tax_parse /
    tax_split (tax= not preceded by ';', no trailing ';', upper-case level letters, missing levels, a ',' after the tax
    field), an exact duplicate with another taxonomy (ties broken by sequence number), a copy one base longer placed
    first (ties broken by length), species with lower-case low-complexity stretches (so that --dbmask changes the
    index) and one record under 32 nt (which --sintax drops).  Queries: mutated `q_len`-nt windows, 30 % of them
    reverse-complemented, some from held-out species, some random, the low-complexity regions in upper case, a few with
    fewer than 32 distinct k-mers (one of 10 nt), IUPAC and lower-case symbols, and two longer than 2 100 nt.
    Returns dict(db_heads, db_seqs, q_heads, q_seqs, meta)."""
    rng = np.random.default_rng(seed)
    rates = (0.10, 0.08, 0.06, 0.05, 0.04, 0.03, 0.02)
    leaves, held = [], []   # (names per level, sequence)

    def grow(seq, names, level):
        if level == len(SINTAX_LEVELS):
            leaves.append((names, seq))
            return
        n = fanout[level] + (1 if level == len(SINTAX_LEVELS) - 1 else 0)
        for j in range(n):
            child = mutate(rng, seq, rates[level])
            nm = names + [f"{SINTAX_LEVELS[level].upper()}{len(leaves) if level == 6 else ''}{'_'.join(names[-1:])}x{j}"]
            if level == len(SINTAX_LEVELS) - 1 and j == n - 1:
                held.append((nm, child))
            else:
                grow(child, nm, level + 1)

    grow(random_seqs(rng, 1, length)[0], [], 0)
    lc = set(range(3, len(leaves), 17))   # species with low-complexity stretches
    db_heads, db_seqs = [], []
    for i, (names, s) in enumerate(leaves):
        seq = s.tobytes()
        if i in lc:
            unit = bytes(ACGT[rng.integers(0, 4, size=int(rng.integers(2, 4)))])
            stretch = (unit * 200)[:180].lower()
            p = int(rng.integers(100, len(seq) - 400))
            seq = seq[:p] + stretch + seq[p + 180:]
        db_seqs.append(seq)
        tax = ",".join(f"{SINTAX_LEVELS[l]}:{names[l]}" for l in range(len(SINTAX_LEVELS)))
        db_heads.append(f"r{i};tax={tax};")
    # header variants
    n = len(db_heads)
    db_heads[1] = db_heads[1].replace(";tax=", ";size=3;tax=").rstrip(";")                       # no trailing ';'
    db_heads[2] = "r2 xtax=d:Fake;" + db_heads[2][3:]                                            # tax= after 'x' skipped
    db_heads[4] = db_heads[4].replace("d:", "D:").replace("g:", "G:")                          # upper-case levels
    db_heads[5] = ",".join(p for p in db_heads[5].split(",") if not p.startswith(("c:", "o:")))  # missing levels
    db_heads[6] = db_heads[6] + "note=a,b"                                                       # ',' after the field
    # an exact duplicate with another species name (ties by number), and a copy one base longer placed before the
    # original (ties by length): both of species 8 / 9, whose windows become queries below
    dup_of, long_of = 8, 9
    db_heads.append(db_heads[dup_of].split(";")[0] + "dup;tax=" + db_heads[dup_of].split("tax=")[1].replace("s:", "s:Dup"))
    db_seqs.append(db_seqs[dup_of])
    long_head = db_heads[long_of].split(";")[0] + "long;tax=" + db_heads[long_of].split("tax=")[1].replace("s:", "s:Long")
    db_heads.insert(0, long_head)
    db_seqs.insert(0, db_seqs[long_of] + b"A")
    # shifted by the insertion: original long_of is now long_of + 1, dup_of + 1 and the duplicate is the last one
    meta = {"tie_seqno": (dup_of + 1, len(db_seqs) - 1), "tie_length": (0, long_of + 1),
            "lc_species": sorted(i + 1 for i in lc)}
    db_heads.append("short;tax=d:Short;")
    db_seqs.append(b"ACGTACGTACGTACGTACGT")   # 20 nt: dropped by --sintax (minseqlength 32)

    q_heads, q_seqs = [], []

    def window(s: bytes, up=True):
        p = int(rng.integers(0, max(1, len(s) - q_len)))
        w = s[p:p + q_len].upper() if up else s[p:p + q_len]
        return mutate(rng, np.frombuffer(w, dtype=np.uint8), 0.03).tobytes()

    sources = list(range(len(leaves))) + [dup_of] * 6 + [long_of] * 6
    for i in range(n_q):
        kind = i % 10
        if kind == 9:
            seq = random_seqs(rng, 1, q_len)[0].tobytes()
        elif kind == 8:
            seq = window(held[int(rng.integers(0, len(held)))][1].tobytes())
        else:
            src = sources[int(rng.integers(0, len(sources)))] if kind < 6 else sorted(lc)[i % len(lc)]
            s = db_seqs[src + 1] if src != dup_of else db_seqs[dup_of + 1]
            if kind >= 6:   # low-complexity region of an lc species, in upper case
                lo = s.find(s[[c.islower() for c in s.decode()].index(True):][:20]) if any(chr(c).islower() for c in s) else 0
                seq = s[max(0, lo - 40):max(0, lo - 40) + q_len].upper()
            else:
                seq = window(s)
        if rng.random() < 0.3:
            seq = revcomp(seq)
        q_seqs.append(seq)
        q_heads.append(f"q{i}" if i % 7 else f"q{i} sample=s{i % 5};")
    # specials: fewer than 32 distinct k-mers, IUPAC / lower case, longer than 2 100 nt
    specials = [("q_short10", b"ACGTTGCAAC"), ("q_short30", db_seqs[12][100:130]), ("q_polyA", b"A" * 120),
                ("q_iupac", window(db_seqs[20])[:100] + b"NNRYKM" + window(db_seqs[20])[:120]),
                ("q_lower", window(db_seqs[30]).lower()),
                ("q_long1", db_seqs[40].upper() + db_seqs[41].upper()), ("q_long2", revcomp(db_seqs[50].upper() * 2))]
    for j, (h, s) in enumerate(specials):
        q_heads.insert(5 + 11 * j, h)
        q_seqs.insert(5 + 11 * j, s)
    meta["short_queries"] = [q_heads.index("q_short10"), q_heads.index("q_short30"), q_heads.index("q_polyA")]
    meta["long_queries"] = [q_heads.index("q_long1"), q_heads.index("q_long2")]
    return {"db_heads": db_heads, "db_seqs": db_seqs, "q_heads": q_heads, "q_seqs": q_seqs, "meta": meta}


def orient_data(seed: int = 91, n_roots: int = 40, per_root: int = 50, length: int = 1400, n_q: int = 360,
                q_len: int = 250, long_len: int = 105_000):
    """Reads of mixed orientation against a 16S-shaped database, for --orient.  The database: `n_roots` random roots of
    ~`length` nt with `per_root` mutants each (4 %), so that a read's k-mers are held by many sequences; in one family
    every other member is reverse-complemented (its k-mers are as common on both strands, so they vote for neither);
    every 7th sequence has a random lower-case stretch of 120 nt and every 11th an upper-case low-complexity one of
    100 nt (masking matters).  Reads (headers ``o{i}``, some with a blank and more text): mutated `q_len`-nt forward
    windows, reverse-complemented windows, random reads, joins of a forward and a reverse-complemented window whose
    shares fall on both sides of the 4x rule (either way round), reads shorter than 13 nt, reads with IUPAC codes and U,
    reads with lower-case stretches, and one read of `long_len` nt made of database stretches.  FASTQ qualities are
    random.  Returns dict(db_heads, db_seqs, q_heads, q_seqs, q_quals, meta)."""
    rng = np.random.default_rng(seed)
    db_heads, db_seqs = [], []
    for r in range(n_roots):
        root = random_seqs(rng, 1, length)[0]
        for j in range(per_root):
            s = mutate(rng, root, 0.04).tobytes()
            i = len(db_seqs)
            if i % 7 == 3:
                p = int(rng.integers(50, len(s) - 200))
                s = s[:p] + s[p:p + 120].lower() + s[p + 120:]
            if i % 11 == 5:
                unit = bytes(ACGT[rng.integers(0, 4, size=int(rng.integers(1, 4)))])
                p = int(rng.integers(50, len(s) - 200))
                s = s[:p] + (unit * 100)[:100] + s[p + 100:]
            if r == 1 and j % 2 == 1:
                s = revcomp(s)
            db_seqs.append(s)
            db_heads.append(f"db{i};root={r}")

    def window(n, mut=0.03):
        src = db_seqs[int(rng.integers(0, len(db_seqs)))].upper()
        p = int(rng.integers(0, max(1, len(src) - n)))
        return mutate(rng, np.frombuffer(src[p:p + n], dtype=np.uint8), mut).tobytes()

    q_heads, q_seqs = [], []
    kinds = []
    for i in range(n_q):
        kind = i % 9
        if kind in (0, 1):
            s = window(q_len)
        elif kind in (2, 3):
            s = revcomp(window(q_len))
        elif kind == 4:
            s = random_seqs(rng, 1, q_len)[0].tobytes()
        elif kind in (5, 6):   # a forward and a reverse-complemented window, forward share around 4/5 (or 1/5)
            share = float(rng.choice([0.5, 0.7, 0.76, 0.78, 0.8, 0.82, 0.84, 0.9, 0.95]))
            a = int(round(2 * q_len * share))
            s = window(a) + revcomp(window(2 * q_len - a))
            if kind == 6:
                s = revcomp(s)
        elif kind == 7:        # IUPAC codes and U
            s = bytearray(window(q_len))
            for p in rng.integers(0, len(s), size=int(rng.integers(1, 12))):
                s[int(p)] = b"NRYKMSWBDHVU"[int(rng.integers(0, 12))]
            s = bytes(s)
        else:                  # lower-case stretches
            s = window(q_len)
            if rng.random() < 0.5:
                s = revcomp(s)
            p = int(rng.integers(0, q_len - 60))
            n = int(rng.integers(20, 200))
            s = s[:p] + s[p:p + n].lower() + s[p + n:]
        kinds.append(kind)
        q_seqs.append(s)
        q_heads.append(f"o{i}" if i % 5 else f"o{i} extra=text {kind}")
    # reads shorter than the word length, and one of more than 100 000 nt from database stretches (a fifth of them
    # reverse-complemented)
    specials = [("o_short5", window(5)), ("o_short11", window(11)), ("o_short12", window(12)), ("o_short13", window(13))]
    parts, n = [], 0
    while n < long_len:
        w = window(int(rng.integers(500, 1300)), 0.02)
        parts.append(revcomp(w) if rng.random() < 0.2 else w)
        n += len(parts[-1])
    specials.append(("o_long", b"".join(parts)))
    for j, (h, s) in enumerate(specials):
        q_heads.insert(7 + 53 * j, h)
        q_seqs.insert(7 + 53 * j, s)
    q_quals = [bytes(rng.integers(33, 74, size=len(s), dtype=np.uint8)) for s in q_seqs]
    meta = {"long_query": q_heads.index("o_long"),
            "short_queries": [q_heads.index(h) for h in ("o_short5", "o_short11")]}
    return {"db_heads": db_heads, "db_seqs": db_seqs, "q_heads": q_heads, "q_seqs": q_seqs, "q_quals": q_quals, "meta": meta}


def write_fastq(path: str, heads, seqs, quals) -> None:
    """FASTQ, one line per sequence and quality"""
    with open(path, "wb") as f:
        for h, s, q in zip(heads, seqs, quals):
            f.write(b"@" + (h if isinstance(h, bytes) else h.encode()) + b"\n" + s + b"\n+\n" + q + b"\n")


def write_records(path: str, heads, seqs, width: int = 80) -> None:
    """FASTA with the given headers, sequence lines wrapped at `width`"""
    with open(path, "wb") as f:
        for h, s in zip(heads, seqs):
            f.write(b">" + (h if isinstance(h, bytes) else h.encode()) + b"\n")
            for i in range(0, max(len(s), 1), width):
                f.write(s[i:i + width] + b"\n")
