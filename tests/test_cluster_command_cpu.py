"""vsg_cluster_write, the host-only writer of the clustering commands, against the reference CLI without a GPU: the
records come from the reference's own --uc (cluster numbers, centroids and strands by label, stored with the goldens),
the alignments from the oracle aligner, the processing order from the command's sort rule restated here.  Every --uc,
--centroids and --clusters file must equal the reference's byte for byte (sha256).  Only cases without DUST: DUST needs
the device."""
import os
import re

import numpy as np
import pytest

import checkers
import cluster_command_cases as cases
from vsearch_b200 import lib as vlib


def _abundance(label):
    m = re.search(r"(?:^|;)size=(\d+)(?:;|$)", label)
    return int(m.group(1)) if m else 1


def _processing_order(command, labels, seqs):
    """Database::sortbylength / sortbyabundance (core/db.cpp:433-485), or the input order for --cluster_smallmem"""
    n = len(labels)
    key = {"cluster_fast": lambda i: (-len(seqs[i]), -_abundance(labels[i]), labels[i].encode(), i),
           "cluster_size": lambda i: (-_abundance(labels[i]), labels[i].encode(), i),
           "cluster_unoise": lambda i: (-_abundance(labels[i]), labels[i].encode(), i),
           "cluster_smallmem": lambda i: i}[command]
    return sorted(range(n), key=key)


@pytest.mark.parametrize("name", cases.CPU_CASES)
def test_cluster_write_equals_reference_files(tmp_path, name):
    inp, command, cli, kw, outputs = cases.CASES[name]
    assert kw.get("qmask") in ("none", "soft") and not kw.get("hardmask")
    want = cases.golden()[name]
    path = cases.input_file(inp, str(tmp_path))
    assert cases.sha256(path) == want["input_sha256"]
    labels, seqs = cases.read_input(path, kw.get("notrunclabels", 0))
    assert len(labels) == want["sequences"]       # no record of these inputs is discarded
    order = _processing_order(command, labels, seqs)
    records = want["records"]
    assert [r[0] for r in records] == order       # the reference processed the records in the restated order
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
    assert any(c is not None for c in cigars)
    out = tmp_path / "out"
    out.mkdir()
    paths = cases.output_files(str(out), name, outputs)
    opts = {k: v for k, v in kw.items() if k in {f for f, _ in vlib.ClusterCmdOpts._fields_}}
    singletons = vlib.cluster_write([labels[i] for i in order], [seqs[i] for i in order],
                                    [_abundance(labels[i]) for i in order], res, cigars, command=command, **paths, **opts)
    assert cases.output_digests(paths) == want["files"]
    assert singletons == want["singletons"]


def test_cluster_write_removes_its_files_on_failure(tmp_path):
    """a --clusters prefix in a directory that does not exist: the call fails and leaves no --uc or --centroids file"""
    res = np.zeros(2, dtype=vlib.CLUSTER_DT)
    res["centroid"] = [-1, 0]
    res[1] = (0, 0, 4, 0, 0, 4, 8, 0, 100.0)
    with pytest.raises(vlib.VsgError, match="clusters file"):
        vlib.cluster_write(["a", "b"], [b"ACGT", b"ACGT"], [1, 1], res, [None, "4M"], uc=str(tmp_path / "x.uc"),
                           centroids=str(tmp_path / "x.fa"), clusters=str(tmp_path / "no" / "c"))
    assert os.listdir(tmp_path) == []
    vlib.cluster_write(["a", "b"], [b"ACGT", b"ACGT"], [1, 1], res, [None, "4M"], uc=str(tmp_path / "x.uc"))
    assert open(tmp_path / "x.uc").read() == ("S\t0\t4\t*\t*\t*\t*\t*\ta\t*\nH\t0\t4\t100.0\t+\t0\t0\t=\tb\ta\n"
                                             "C\t0\t2\t*\t*\t*\t*\t*\ta\t*\n")
