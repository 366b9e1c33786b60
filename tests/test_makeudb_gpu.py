"""Making UDB files on the GPU (vsg_udb_make, vsg_udb_write, vsg_makeudb_usearch) against the reference's
`vsearch --makeudb_usearch`: byte identity with the stored digests of its files (and with a fresh run of
oracle/_ref/vsearch when it is built), the refusals, the round trip through vsg_udb_open / vsg_udb_load / a search, and the
in-memory database against the file and the oracle's index."""
import ctypes as C
import gzip
import os

import numpy as np
import pytest

import checkers
import makeudb_cases as mc
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return str(tmp_path_factory.mktemp("makeudb_inputs"))


def run_case(c, name, inputs, out):
    inp, cli, opts = mc.CASES[name]
    path = mc.input_file(inp, inputs)
    g = mc.golden()[name]
    assert mc.sha256(path) == g["input_sha256"]
    st = c.makeudb_usearch(path, out, **opts)
    assert os.path.getsize(out) == g["size"]
    assert mc.sha256(out) == g["sha256"]
    if os.path.exists(mc.STOCK):
        ref = out + ".ref"
        mc.reference_makeudb(path, ref, cli)
        assert open(ref, "rb").read() == open(out, "rb").read()
    return st


@pytest.mark.parametrize("name", [n for n in mc.CASES if not n.startswith("many")])
def test_makeudb_file_equals_the_reference(tmp_path, ctx, inputs, name):
    out = str(tmp_path / "db.udb")
    st = run_case(ctx, name, inputs, out)
    if name == "all_discarded":
        assert st["sequences"] == 0 and st["discarded_short"] == 25
        # the reference's own reader refuses such a file, and so does vsg_udb_open
        with pytest.raises(vlib.VsgError, match="Invalid UDB file"):
            vlib.Udb(out)
        return
    u = vlib.Udb(out)
    assert u.n == st["sequences"] and u.info.index_entries == st["index_entries"]
    assert u.info.nucleotides == st["nucleotides"]
    db, ix, ml = ctx.udb_load(u)
    assert ml == 1   # upper-cased input: the file's index agrees with the masked-lower-case convention in every case
    ix.close(); db.close(); u.close()
    if name == "lengths_default":
        assert (st["discarded_short"], st["discarded_long"]) == (3, 3)
    if name == "lengths_wide":
        assert (st["discarded_short"], st["discarded_long"]) == (0, 0)
    if name == "symbols":
        assert st["stripped"] > 0


@pytest.mark.parametrize("budget_mb", [None, 4])
@pytest.mark.parametrize("name", ["many", "many_none_k12"])
def test_makeudb_many_sequences_in_many_ranges(tmp_path, inputs, monkeypatch, name, budget_mb):
    """72 000 records at the default scratch budget and at 4 MiB (a quarter of it holds 65 536 keys: the index is built
    in over a hundred word ranges, and with --dbmask none the homopolymer's word alone has more windows than that)"""
    if budget_mb is not None:
        monkeypatch.setenv("VSG_DIR_BUDGET_MB", str(budget_mb))
    c = vlib.Context(0)
    try:
        st = run_case(c, name, inputs, str(tmp_path / "db.udb"))
    finally:
        c.close()
    assert st["sequences"] == 72000


def test_refusals(tmp_path, ctx):
    out = str(tmp_path / "x.udb")

    def refused(path, pattern, **opts):
        with pytest.raises(vlib.VsgError, match=pattern) as e:
            ctx.makeudb_usearch(path, out, **opts)
        assert "(-3)" in str(e.value)   # VSG_EINVAL
        assert not os.path.exists(out)

    fa = str(tmp_path / "dash.fasta")
    open(fa, "w").write(">a\nACGTACGT\n>b\nAC-GT\n")
    refused(fa, r"Illegal character '-' in sequence on line 4")
    open(fa, "w").write(">a\nACGT.ACGT\n")
    refused(fa, r"Illegal character '\.' in sequence on line 2")
    open(fa, "w").write(">a\nACGT\x01ACGT\n")
    refused(fa, r"unprintable ASCII character no 1 in sequence on line 2")
    gz = str(tmp_path / "in.fasta.gz")
    with gzip.open(gz, "wb") as f:
        f.write(b">a\nACGTACGTACGTACGTACGTACGTACGTACGTACGT\n")
    refused(gz, "gzip")
    ok = str(tmp_path / "ok.fasta")
    open(ok, "w").write(">a\n" + "ACGT" * 20 + "\n")
    refused(ok, "wordlength 2", wordlength=2)
    refused(ok, "wordlength 16", wordlength=16)
    refused(ok, "unknown dbmask", dbmask=7)
    with pytest.raises(vlib.VsgError, match="output file must be specified"):
        ctx.makeudb_usearch(ok, None)
    # the same FASTA is fine
    ctx.makeudb_usearch(ok, out)
    assert vlib.Udb(out).n == 1


@pytest.mark.parametrize("dbmask", mc.SEARCH_MASKS)
def test_search_on_a_made_database_equals_the_reference_cli(tmp_path, dbmask):
    """vsg_usearch_stream on vsg_group_create_udb of a made file writes the --blast6out the reference CLI writes with
    --db on its own UDB file of the same FASTA"""
    d = str(tmp_path)
    fasta, qf = mc.search_inputs(d)
    g = mc.golden()[f"search_{dbmask}"]
    assert mc.sha256(fasta) + mc.sha256(qf) == g["input_sha256"]
    udb = os.path.join(d, "db.udb")
    c = vlib.Context(0)
    try:
        c.makeudb_usearch(fasta, udb, dbmask=dbmask)
    finally:
        c.close()
    u = vlib.Udb(udb)
    grp = vlib.Group.from_udb([0], u)
    labels = [u.header(i) for i in range(u.n)]
    o = vlib.default_search_opts(); o.id = 0.9; o.maxaccepts = 2; o.maxrejects = 16
    out = os.path.join(d, "got.b6")
    st = grp.stream(labels, qf, o, out, batch_queries=512)
    grp.close(); u.close()
    assert st["queries"] == 1500
    assert os.path.getsize(out) == g["size"] and mc.sha256(out) == g["sha256"]


@pytest.mark.parametrize("k,dbmask,hardmask", [(8, "dust", 0), (8, "none", 0), (5, "dust", 1), (12, "dust", 0), (11, "soft", 0)])
def test_in_memory_equals_on_disk_and_the_oracle_index(tmp_path, ctx, k, dbmask, hardmask):
    rng = np.random.default_rng(21 + k)
    seqs, heads = [], []
    for i in range(300):
        s = bytearray(synth.random_seqs(rng, 1, int(rng.integers(0, 700)))[0].tobytes())
        if i % 4 == 0 and len(s) > 80:
            s[10:70] = b"ACGACGACG" * 6 + b"ACGACG"
        if i % 5 == 0 and len(s) > 30:
            s[3:20] = bytes(s[3:20]).lower()
        if i % 6 == 0 and len(s) > 5:
            s[2] = ord("U"); s[4] = ord("y")
        seqs.append(bytes(s)); heads.append(f"h{i} with blanks")
    u = ctx.udb_make(seqs, heads, wordlength=k, dbmask=dbmask, hardmask=hardmask)
    path = str(tmp_path / "m.udb")
    u.write(path)
    f = vlib.Udb(path)
    for field, _ in vlib.UdbInfo._fields_:
        assert getattr(u.info, field) == getattr(f.info, field), field
    a, b = u.sequences(), f.sequences()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert [u.header(i) for i in range(u.n)] == [f.header(i) for i in range(f.n)] == heads
    kc, ki = u.words()
    fkc, fki = f.words()
    assert np.array_equal(kc, fkc) and np.array_equal(ki, fki)
    # the file's sequences: the records upper-cased, with DUST's mask as lower case (or 'N' with hardmask)
    cat, off, ln = a
    got = [cat[off[i]: off[i] + ln[i]].tobytes() for i in range(u.n)]
    assert [g.upper() for g in got] == [s.upper() for s in seqs] or hardmask
    if dbmask != "dust":
        assert got == [s.upper() for s in seqs]
    # the index == the oracle's index of the masked sequences
    od = checkers.OracleDb(synth.SeqSet(got), k=k, mask_lower=0 if dbmask == "none" else 1)
    o = checkers.oracle()
    start = np.zeros((1 << (2 * k)) + 1, dtype=np.uint64)
    o.oracle_index_starts(C.c_void_p(od.h), start.ctypes.data_as(C.POINTER(C.c_uint64)))
    post = np.zeros(int(start[-1]) + 1, dtype=np.uint32)
    o.oracle_index_postings(C.c_void_p(od.h), post.ctypes.data_as(C.POINTER(C.c_uint32)))
    assert np.array_equal(np.diff(start).astype(np.uint32), kc)
    assert np.array_equal(post[: int(start[-1])], ki)
    od.close()
    # the made database loads like the file
    db, ix, ml = ctx.udb_load(u)
    assert ml == 1
    ix.close(); db.close(); u.close(); f.close()
