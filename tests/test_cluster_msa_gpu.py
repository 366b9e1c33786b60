"""--msaout, --consout and --profile of vsg_cluster_command_outputs against the reference CLI: every file byte for byte
(sha256, tests/golden/cluster_msa_reference.json) for the cases of cluster_msa_cases.py, and with oracle/_ref/vsearch
present also a fresh reference run; vsg_cluster_msa's arrays element by element against the numpy restatement of msa();
the device work cut into several chunks; and a failed write that leaves no file."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import cluster_msa_cases as cases
from vsearch_b200 import lib as vlib, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = vlib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    return cases.golden()


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_cluster_msa_equals_reference_cli(ctx, golden, tmp_path, name):
    inp, command, cli, kw = cases.CASES[name]
    path = cases.input_file(inp, str(tmp_path))
    want = golden[name]
    assert cases.sha256(path) == want["input_sha256"]
    mine = tmp_path / "mine"
    mine.mkdir()
    paths = cases.output_files(str(mine), name)
    ctx.cluster_command(path, command=command, **paths, **kw)
    assert cases.output_digests(paths) == want["files"]
    if os.path.exists(cases.STOCK):
        ref = tmp_path / "ref"
        ref.mkdir()
        rpaths = cases.output_files(str(ref), name)
        cases.reference_run(path, command, cli, rpaths)
        assert cases.output_digests(rpaths) == want["files"]


@pytest.mark.parametrize("name", cases.ARRAY_CASES)
def test_cluster_msa_arrays_equal_restatement(ctx, tmp_path, name):
    """the records of the command's own --uc, the CIGARs from vsg_align_pairs, then vsg_cluster_msa against restate()"""
    inp, command, cli, kw = cases.CASES[name]
    assert not kw.get("strand_both")
    path = cases.input_file(inp, str(tmp_path))
    uc = str(tmp_path / "x.uc")
    ctx.cluster_command(path, command=command, uc=uc, **kw)
    labels, seqs = cases.cc.read_input(path)
    order = cases.processing_order(command, labels, seqs)
    records = cases.cc.uc_records(open(uc).read(), labels)
    assert [r[0] for r in records] == order
    pos = {rec: k for k, rec in enumerate(order)}
    res = np.zeros(len(order), dtype=vlib.CLUSTER_DT)
    res["cluster"] = [r[1] for r in records]
    res["centroid"] = [pos[r[2]] if r[2] >= 0 else -1 for r in records]
    oseqs = [seqs[i] for i in order]
    ss = ctx.seqset(_seqset(oseqs))
    h = np.nonzero(res["centroid"] >= 0)[0]
    al = ctx.align_pairs(ss, ss, h.astype(np.uint32), res["centroid"][h].astype(np.uint32), cigar=True)
    cigars = [None] * len(order)
    for j, k in enumerate(h):
        cigars[int(k)] = al.cigars[j]
    weights = np.array([cases.abundance(labels[i]) if kw.get("sizein") else 1 for i in order], dtype=np.uint64)
    got = ctx.cluster_msa(ss, res, weights, cigars)
    ins, first, prof, cons = cases.restate(oseqs, res, weights, cigars)
    np.testing.assert_array_equal(got["insertions"], ins)
    np.testing.assert_array_equal(got["col_first"], first)
    np.testing.assert_array_equal(got["profile"], prof)
    assert got["consensus"].tobytes() == cons


def _seqset(seqs):
    class S:
        pass
    s = S()
    s.cat = np.frombuffer(b"".join(seqs), dtype=np.uint8)
    s.lens = np.array([len(x) for x in seqs], dtype=np.int32)
    s.offs = np.concatenate(([0], np.cumsum(s.lens[:-1], dtype=np.int64))).astype(np.int64)
    return s


_CHUNKED = r"""
import json, os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "tests")]
import cluster_msa_cases as cases
from vsearch_b200 import lib as vlib
out = {}
ctx = vlib.Context(0)
for name in ("p_singletons", "c_size_sizes", "o_long"):
    inp, command, cli, kw = cases.CASES[name]
    paths = cases.output_files(sys.argv[2], name)
    ctx.cluster_command(cases.input_file(inp, sys.argv[2]), command=command, **paths, **kw)
    out[name] = cases.output_digests(paths)
ctx.close()
print(json.dumps(out))
"""


def test_cluster_msa_in_several_chunks(golden, tmp_path):
    """a 1 MiB direction budget (256 KiB of MSA scratch) cuts the clusters into several chunks; the files stay the same"""
    env = dict(os.environ, VSG_DIR_BUDGET_MB="1", VSG_TRACE="1")
    r = subprocess.run([sys.executable, "-c", _CHUNKED, cases.checkers.ROOT, str(tmp_path)], capture_output=True, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for name, digests in got.items():
        assert digests == golden[name]["files"], name
    chunks = [int(line.split(" chunks")[0].split(", ")[-1].split(" + ")[0]) for line in r.stderr.splitlines()
              if line.startswith("[vsg] cluster_msa:") and " chunks" in line]
    assert max(chunks) > 1, r.stderr[-3000:]


def test_cluster_msa_failed_write_leaves_no_file(ctx, tmp_path):
    """a --profile path in a missing directory: VSG_EINVAL, and neither the cluster files nor the other two remain"""
    path = cases.input_file("small", str(tmp_path))
    out = tmp_path / "out"
    out.mkdir()
    with pytest.raises(vlib.VsgError, match=r"cannot write") as e:
        ctx.cluster_command(path, uc=str(out / "x.uc"), centroids=str(out / "x.fa"), clusters=str(out / "c_"),
                            msaout=str(out / "x.msa"), consout=str(out / "x.cons"), profile=str(out / "no" / "x.prof"), id=0.97)
    assert "(-3)" in str(e.value)
    assert os.listdir(out) == []


def test_cluster_msa_cap(ctx):
    """the binding's first call has cap 0 (VSG_ECAP with the column count), the second the room it asked for; a D run
    of two against a gap in one row of two ties, and the symbol wins"""
    rng = np.random.default_rng(3)
    root = synth.random_seqs(rng, 1, 60)[0].tobytes()
    seqs = [root, root[:30] + b"GG" + root[30:]]
    ss = ctx.seqset(_seqset(seqs))
    res = np.zeros(2, dtype=vlib.CLUSTER_DT)
    res["centroid"] = [-1, 0]
    got = ctx.cluster_msa(ss, res, [1, 1], [None, "30M2D30M"])
    assert got["col_first"].tolist() == [0, 62]
    assert got["insertions"][30] == 2 and got["insertions"].sum() == 2
    assert got["consensus"].tobytes() == root[:30] + b"GG" + root[30:]
    assert got["profile"][30].tolist() == [0, 0, 1, 0, 0, 1]
