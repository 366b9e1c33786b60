"""--search_exact's semantics pinned without a GPU: a plain Python restatement of the command (normalise, dictionary lookup
on both strands, the size and label filters, search_joinhits order, the writers, the OTU tables) writes the output files
of every case of search_exact_cases.py from the case's inputs, and each must equal the reference CLI's file
(sha256, tests/golden/search_exact_reference.json).  DUST is not restated: a file that prints sequences DUST-masked
(--matched / --notmatched with --qmask dust, --dbmatched / --dbnotmatched with --dbmask dust) is left to the GPU test."""
import re

import pytest

import search_exact_cases as cases

def read_fastx(path, notrunclabels=False):
    labels, seqs = [], []
    text = open(path).read()
    if text.startswith("@"):
        lines = text.splitlines()
        for i in range(0, len(lines), 4):
            labels.append(lines[i][1:])
            seqs.append(lines[i + 1])
    else:
        for rec in text.split(">")[1:]:
            h, _, body = rec.partition("\n")
            labels.append(h)
            seqs.append(body.replace("\n", ""))
    if not notrunclabels:
        labels = [re.split(r"[ \t]", h)[0] for h in labels]
    return labels, seqs


def key(seq):
    """what seqcmp compares: the 4-bit code of every symbol (case and U / T do not matter)"""
    return seq.upper().replace("U", "T")


def size_of(h):
    """header_get_size: (^|;)size=[0-9]+(;|$), else 1"""
    m = re.search(r"(?:^|;)size=([0-9]+)(?=;|$)", h)
    return int(m.group(1)) if m else 1


def strip_size(h, strip):
    """header_fprint_strip with --xsize: (label, whether it ends with ';')"""
    m = re.search(r"(?:^|;)(size=[0-9]+)(?=;|$)", h) if strip else None
    if m is None:
        return h, h.endswith(";")
    s, e = m.span(1)
    out = (h[:s - 1] if s > 1 else "") + (h[e:] if len(h) > e + 1 else "")
    last = (len(h) - 1) if len(h) > e + 1 else (s - 2 if s > 1 else -1)
    return out, last >= 0 and h[last] == ";"


def fasta(head, seq, abundance, o):
    sizeout = o.get("sizeout", 0) and abundance > 0
    lab, trailing = strip_size(head, o.get("xsize", 0) or sizeout)
    out = ">" + lab
    if sizeout:
        out += ("" if trailing else ";") + f"size={abundance}"
    out += "\n"
    w = o.get("fasta_width", 80)
    if w < 1:
        return out + seq + "\n"
    return out + "".join(seq[i:i + w] + "\n" for i in range(0, len(seq), w))


def attribute(h, name):
    m = re.search(r"(?:^|;)" + name + r"=([^;]*)", h)
    return m


class OtuTable:
    def __init__(self):
        self.otus, self.samples, self.count, self.tax = set(), set(), {}, {}

    def add(self, query, target, abundance):
        sample = otu = None
        if query is not None:
            m = re.search(r"(?:^|;)(?:sample|barcodelabel)=([^;]*)", query)
            sample = m.group(1) if m else re.match(r"[A-Za-z0-9_]*", query).group(0)
            self.samples.add(sample)
        if target is not None:
            m = attribute(target, "otu")
            otu = m.group(1) if m else target.split(";")[0]
            t = attribute(target, "tax")
            if t:
                self.tax[otu] = t.group(1)
            self.otus.add(otu)
        if sample is not None and otu is not None and abundance:
            self.count[(otu, sample)] = self.count.get((otu, sample), 0) + abundance

    def otutabout(self):
        bo = lambda s: s.encode()
        samples, otus = sorted(self.samples, key=bo), sorted(self.otus, key=bo)
        out = "#OTU ID" + "".join("\t" + s for s in samples) + ("\ttaxonomy" if self.tax else "") + "\n"
        for o in otus:
            out += o + "".join(f"\t{self.count.get((o, s), 0)}" for s in samples)
            if self.tax:
                out += "\t" + self.tax.get(o, "")
            out += "\n"
        return out

    def mothur(self):
        bo = lambda s: s.encode()
        samples, otus = sorted(self.samples, key=bo), sorted(self.otus, key=bo)
        out = "label\tGroup\tnumOtus" + "".join("\t" + o for o in otus) + "\n"
        for s in samples:
            out += f"vsearch\t{s}\t{len(otus)}" + "".join(f"\t{self.count.get((o, s), 0)}" for o in otus) + "\n"
        return out


def ratio_ok(q, ratio, t, sign):
    """abundance_ratio_cmp(q, ratio, t) compared with 0 (the double product: every size here is small)"""
    prod = ratio * t
    c = (q > prod) - (q < prod)
    return c >= 0 if sign > 0 else c <= 0


def search_exact(qpath, dbpath, o):
    """{output: text} of `vsearch --search_exact qpath --db dbpath --threads 1` with the options o (search_exact_command
    keywords)"""
    notrunc = o.get("notrunclabels", 0)
    dl, ds = read_fastx(dbpath, notrunc)
    keep = [i for i in range(len(ds)) if o.get("minseqlength", 1) <= len(ds[i]) <= o.get("maxseqlength", 50000)]
    dl, ds = [dl[i] for i in keep], [ds[i] for i in keep]
    hard = o.get("hardmask", 0)
    hm = lambda s: re.sub("[a-z]", "N", s)
    if hard and o.get("dbmask") == "soft":
        ds = [hm(s) for s in ds]
    dprint = ds   # as read unless DUST-masked (not restated here)
    tsize = [size_of(h) for h in dl]
    index = {}
    for i, s in enumerate(ds):
        index.setdefault((len(s), key(s)), []).append(i)
    ql, qs = read_fastx(qpath, notrunc)
    strands = 2 if o.get("strand_both") else 1
    maxhits = o.get("maxhits", 0) or len(ds) + 1
    out = {k: "" for k in cases.OUTPUTS}
    dbmatched = [0] * len(ds)
    otu = OtuTable()
    matched = 0
    for qh, q in zip(ql, qs):
        if hard and o.get("qmask") == "soft":
            q = hm(q)
        qsize = size_of(qh)
        hits = []
        for strand in range(strands):
            s = q if strand == 0 else cases.revcomp(q.encode()).decode()
            for t in index.get((len(s), key(s)), []):
                if not (qsize <= o.get("maxqsize", 2 ** 63) and tsize[t] >= o.get("mintsize", 0)
                        and ratio_ok(qsize, o.get("minsizeratio", 0.0), tsize[t], 1)
                        and (o.get("maxsizeratio") is None or ratio_ok(qsize, o["maxsizeratio"], tsize[t], -1))
                        and not (o.get("self") and qh == dl[t])):
                    continue
                hits.append((t, strand))
        hits.sort(key=lambda h: h[0])   # hit_compare_byid: all at 100 %, target ascending; stable, so plus before minus
        rep = hits[:maxhits]
        for t, strand in rep:
            qs_, qe = (len(q), 1) if strand else (1, len(q))
            out["blast6out"] += f"{qh}\t{dl[t]}\t100.0\t{len(q)}\t0\t0\t{qs_}\t{qe}\t1\t{len(q)}\t-1\t0\n"
        if not rep and o.get("output_no_hits"):
            out["blast6out"] += f"{qh}\t*\t0.0\t0\t0\t0\t0\t0\t0\t0\t-1\t0\n"
        for j, (t, strand) in enumerate(rep):
            if j == 0 or o.get("uc_allhits"):
                out["uc"] += (f"H\t{t}\t{len(q)}\t100.0\t{'-' if strand else '+'}\t0\t0\t=\t{strip_size(qh, o.get('xsize'))[0]}\t"
                              f"{strip_size(dl[t], o.get('xsize'))[0]}\n")
        if not rep:
            out["uc"] += f"N\t*\t*\t*\t.\t*\t*\t*\t{qh}\t*\n"
        otu.add(qh, dl[rep[0][0]] if rep else None, qsize)
        qprint = q
        if hits:
            matched += 1
            out["matched"] += fasta(qh, qprint, qsize, o)
        else:
            out["notmatched"] += fasta(qh, qprint, qsize, o)
        for t, _ in hits:
            dbmatched[t] += qsize if o.get("sizein") else 1
    for t in range(len(ds)):
        if dbmatched[t]:
            out["dbmatched"] += fasta(dl[t], dprint[t], dbmatched[t], o)
        else:
            otu.add(None, dl[t], 0)
            out["dbnotmatched"] += fasta(dl[t], dprint[t], 0, o)
    out["otutabout"] = otu.otutabout()
    out["mothur_shared_out"] = otu.mothur()
    return out, {"matched": matched, "queries": len(qs)}


@pytest.mark.parametrize("name", sorted(set(cases.CASES) - set(cases.DUST_CASES)))
def test_search_exact_oracle_equals_reference(tmp_path, name):
    inp, cli, kw, outputs = cases.CASES[name]
    q, db = cases.input_files(inp, str(tmp_path))
    want = cases.golden()[name]
    assert cases.sha256(q) == want["query_sha256"] and cases.sha256(db) == want["db_sha256"]
    files, counts = search_exact(q, db, kw)
    dusted = {o for o in outputs if (o in ("matched", "notmatched") and kw.get("qmask", "dust") == "dust")
              or (o in ("dbmatched", "dbnotmatched") and kw.get("dbmask", "dust") == "dust")}
    got = {o: cases.sha256_bytes(files[o].encode()) for o in outputs if o not in dusted}
    assert got == {o: h for o, h in want["files"].items() if o not in dusted}
    assert counts == {k: want[k] for k in counts}
