"""vsg_cluster_msa_write and the numpy restatement of msa() (cluster_msa_cases.restate) against the reference CLI without
a GPU: the records come from the reference's own --uc (stored with the goldens), the CIGARs from the oracle aligner, the
column layout, profile and consensus from the restatement.  Every --msaout, --consout and --profile file must equal the
reference's byte for byte (sha256).  Only cases without DUST: DUST needs the device."""
import os

import numpy as np
import pytest

import checkers
import cluster_msa_cases as cases
from vsearch_b200 import lib as vlib


def rebuild(name, directory):
    """(printed sequences, headers, abundances, results, cigars, weights) of case `name` in processing order"""
    inp, command, cli, kw = cases.CASES[name]
    want = cases.golden()[name]
    path = cases.input_file(inp, directory)
    assert cases.sha256(path) == want["input_sha256"]
    labels, seqs = cases.cc.read_input(path, kw.get("notrunclabels", 0))
    minsize = kw.get("minsize", 8) if command == "cluster_unoise" else 1
    keep = [i for i in range(len(labels)) if kw.get("minseqlength", 32) <= len(seqs[i]) <= kw.get("maxseqlength", 50000)
            and cases.abundance(labels[i]) >= minsize]
    order = [keep[k] for k in cases.processing_order(command, [labels[i] for i in keep], [seqs[i] for i in keep])]
    records = want["records"]
    assert [r[0] for r in records] == order
    if kw.get("hardmask"):
        seqs = [bytes(78 if 97 <= ch <= 122 else ch for ch in s) for s in seqs]   # lower case to "N"
    pos = {rec: k for k, rec in enumerate(order)}
    res = np.zeros(len(order), dtype=vlib.CLUSTER_DT)
    cigars = []
    for k, (rec, cluster, centroid, strand, ident) in enumerate(records):
        res["cluster"][k] = cluster
        if centroid < 0:
            res["centroid"][k] = -1
            cigars.append(None)
            continue
        q = cases.revcomp(seqs[rec]) if strand else seqs[rec]
        score, aligned, matches, mismatches, gaps, cigar = checkers.oracle_nw16(q, seqs[centroid])
        res[k] = (cluster, pos[centroid], matches, mismatches, gaps, aligned, score, strand, ident)
        cigars.append(cigar)
    ab = [cases.abundance(labels[i]) for i in order]
    weights = ab if kw.get("sizein") else [1] * len(order)
    return [seqs[i] for i in order], [labels[i] for i in order], ab, res, cigars, weights


@pytest.mark.parametrize("name", cases.CPU_CASES)
def test_cluster_msa_write_equals_reference_files(tmp_path, name):
    inp, command, cli, kw = cases.CASES[name]
    seqs, heads, ab, res, cigars, weights = rebuild(name, str(tmp_path))
    ins, first, prof, cons = cases.restate(seqs, res, weights, cigars)
    msa = {"insertions": ins, "col_first": first, "profile": prof, "consensus": np.frombuffer(cons, dtype=np.uint8)}
    paths = cases.output_files(str(tmp_path), name)
    del paths["uc"]
    opts = {k: v for k, v in kw.items() if k in {f for f, _ in vlib.ClusterCmdOpts._fields_}}
    vlib.cluster_msa_write(heads, seqs, ab, res, cigars, msa, command=command, **paths, **opts)
    want = cases.golden()[name]["files"]
    assert cases.output_digests(paths) == {o: want[o] for o in paths}


def test_cluster_msa_write_removes_its_files_on_failure(tmp_path):
    """a --profile path in a directory that does not exist: the call fails and leaves no --msaout or --consout file"""
    res = np.zeros(2, dtype=vlib.CLUSTER_DT)
    res["centroid"] = [-1, 0]
    res[1] = (0, 0, 4, 0, 0, 4, 8, 0, 100.0)
    ins, first, prof, cons = cases.restate([b"ACGT", b"ACGT"], res, [1, 1], [None, "4M"])
    msa = {"insertions": ins, "col_first": first, "profile": prof, "consensus": np.frombuffer(cons, dtype=np.uint8)}
    with pytest.raises(vlib.VsgError, match=r"cannot write.*\(-3\)|\(-3\).*cannot write"):
        vlib.cluster_msa_write(["a", "b"], [b"ACGT", b"ACGT"], [1, 1], res, [None, "4M"], msa, msaout=str(tmp_path / "x.msa"),
                               consout=str(tmp_path / "x.cons"), profile=str(tmp_path / "no" / "x.prof"))
    assert os.listdir(tmp_path) == []
    vlib.cluster_msa_write(["a", "b"], [b"ACGT", b"ACGT"], [1, 1], res, [None, "4M"], msa, consout=str(tmp_path / "x.cons"),
                           profile=str(tmp_path / "x.prof"))
    assert open(tmp_path / "x.cons").read() == ">centroid=a;seqs=2\nACGT\n"
    assert open(tmp_path / "x.prof").read() == (">centroid=a;seqs=2\n0\tA\t2\t0\t0\t0\t0\t0\n1\tC\t0\t2\t0\t0\t0\t0\n"
                                                "2\tG\t0\t0\t2\t0\t0\t0\n3\tT\t0\t0\t0\t2\t0\t0\n\n")


def test_cluster_msa_write_refuses_arrays_that_do_not_match(tmp_path):
    res = np.zeros(2, dtype=vlib.CLUSTER_DT)
    res["centroid"] = [-1, 0]
    res[1] = (0, 0, 4, 0, 0, 4, 8, 0, 100.0)
    ins, first, prof, cons = cases.restate([b"ACGT", b"ACGT"], res, [1, 1], [None, "4M"])
    msa = {"insertions": ins, "col_first": first + np.array([0, 1]), "profile": prof,
           "consensus": np.frombuffer(cons, dtype=np.uint8)}
    with pytest.raises(vlib.VsgError, match="do not match"):
        vlib.cluster_msa_write(["a", "b"], [b"ACGT", b"ACGT"], [1, 1], res, [None, "4M"], msa, msaout=str(tmp_path / "x.msa"))
    assert os.listdir(tmp_path) == []
