"""vsg_cluster_command, the --cluster_fast / --cluster_size / --cluster_smallmem / --cluster_unoise command, against the
reference CLI: every --uc, --centroids and --clusters file byte for byte (sha256, tests/golden/cluster_command_reference.json)
and the counts of its summary, for the option sets of cluster_command_cases.py; and each refusal, with no output file
left behind.  With oracle/_ref/vsearch present the reference's files are also made afresh and compared with the goldens."""
import bz2
import gzip
import os

import numpy as np
import pytest

import cluster_command_cases as cases
from vsearch_b200 import lib as vlib

pytestmark = pytest.mark.gpu

COUNTS = ("sequences", "discarded_short", "discarded_long", "discarded_minsize", "clusters", "singletons")


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    return cases.golden()


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_cluster_command_equals_reference_cli(ctx, golden, tmp_path, name):
    inp, command, cli, kw, outputs = cases.CASES[name]
    path = cases.input_file(inp, str(tmp_path))
    want = golden[name]
    assert cases.sha256(path) == want["input_sha256"]
    mine = tmp_path / "mine"
    mine.mkdir()
    paths = cases.output_files(str(mine), name, outputs)
    st = ctx.cluster_command(path, command=command, **paths, **kw)
    assert cases.output_digests(paths) == want["files"]
    assert {k: st[k] for k in COUNTS} == {k: want[k] for k in COUNTS}
    assert st["nucleotides"] > 0 or st["sequences"] == 0
    if os.path.exists(cases.STOCK):
        ref = tmp_path / "ref"
        ref.mkdir()
        rpaths = cases.output_files(str(ref), name, outputs)
        counts = cases.reference_run(path, command, cli, rpaths)
        assert cases.output_digests(rpaths) == want["files"]
        assert {k: counts[k] for k in COUNTS} == {k: want[k] for k in COUNTS}


def _made(directory):
    return sorted(os.listdir(directory))


def _refused(ctx, tmp_path, inp, match, command="cluster_fast", **kw):
    out = tmp_path / "out"
    out.mkdir(exist_ok=True)
    paths = cases.output_files(str(out), "x", ("uc", "centroids", "clusters"))
    with pytest.raises(vlib.VsgError, match=match) as e:
        ctx.cluster_command(inp, command=command, **paths, **kw)
    assert "(-3)" in str(e.value)          # VSG_EINVAL
    assert _made(out) == []


def test_cluster_command_refusals(ctx, tmp_path):
    plain = cases.input_file("small", str(tmp_path))
    raw = open(plain, "rb").read()
    gz = tmp_path / "small.fasta.gz"
    gz.write_bytes(gzip.compress(raw))
    _refused(ctx, tmp_path, str(gz), "gzip", id=0.97)
    bz = tmp_path / "small.fasta.bz2"
    bz.write_bytes(bz2.compress(raw))
    _refused(ctx, tmp_path, str(bz), "bzip2", id=0.97)
    _refused(ctx, tmp_path, plain, "hardmask", id=0.97, qmask="dust", hardmask=1)
    for k in (11, 13, 15):
        _refused(ctx, tmp_path, plain, "wordlength 3..10", id=0.97, wordlength=k)
    zero = tmp_path / "zero.fasta"
    zero.write_bytes(raw.replace(b">h0003\n", b">h0003;size=0\n", 1))
    _refused(ctx, tmp_path, str(zero), "zero", id=0.97)
    _refused(ctx, tmp_path, str(tmp_path / "missing.fasta"), "cannot open", id=0.97)


def test_cluster_smallmem_needs_sorted_input_or_usersort(ctx, tmp_path):
    unsorted = cases.input_file("unsorted_lower", str(tmp_path))
    _refused(ctx, tmp_path, unsorted, "Sequences not sorted by length and --usersort not specified", command="cluster_smallmem",
             id=0.95)
    out = tmp_path / "ok"
    out.mkdir()
    st = ctx.cluster_command(unsorted, command="cluster_smallmem", uc=str(out / "x.uc"), id=0.95, usersort=1)
    assert st["sequences"] == 400 and os.path.getsize(out / "x.uc") > 0
    sorted_in = cases.input_file("length_sorted", str(tmp_path))
    st = ctx.cluster_command(sorted_in, command="cluster_smallmem", uc=str(out / "y.uc"), id=0.97)
    assert st["sequences"] == 300


def test_cluster_command_refuses_a_deferred_pair(tmp_path):
    """every pair deferred (a gap penalty outside 16 bits): with a fallback callback the clustering itself goes through,
    but the CIGAR of an H record cannot come from it, so the command names the read and writes nothing"""
    rng = np.random.default_rng(5)
    s = bytes(rng.choice(list(b"ACGT"), size=200).astype(np.uint8))
    inp = tmp_path / "same.fasta"
    inp.write_text("".join(f">s{i}\n{s.decode()}\n" for i in range(5)))
    pen = np.array(vlib.DEFAULT_PEN, dtype=np.int64)
    pen[4] = 2 ** 31 - 1
    c = vlib.Context(0, pen=pen)
    try:
        c.set_fallback(lambda q, strand, t: (400, 200, 200, 0, 0, 0, 0, 0, 0))
        _refused(c, tmp_path, str(inp), "defers the alignment of s1", id=0.97, threads=2)
    finally:
        c.close()
