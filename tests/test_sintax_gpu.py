"""SINTAX on the GPU against the reference: vsg_sintax_stream's --tabbedout equals `vsearch --sintax ... --threads 1
--randseed S` byte for byte for the option sets (a)-(e), every bootstrap winner of vsg_sintax equals vsref_sintax's,
query numbering survives slicing, batching and device groups, and the errors come back with their codes."""
import os

import numpy as np
import pytest

import checkers
import sintax_cases as sc
from vsearch_b200 import lib, synth

pytestmark = pytest.mark.gpu


def _seqset(seqs):
    return synth.SeqSet(seqs)


def _group(case, devices=(0,)):
    k, mask, _, _, _, from_udb = sc.CASES[case]
    return lib.Group(list(devices), _seqset(sc.database()[1]), wordlength=k, mask_lower=mask)


def _stream(case, tmp, devices=(0,), batch_queries=65536):
    _, _, both, cutoff, seed, from_udb = sc.CASES[case]
    _, qf = sc.write_inputs(tmp)
    if from_udb:
        udb = lib.Udb(sc.udb_path(tmp))
        g = lib.Group.from_udb(list(devices), udb)
        heads = [udb.header(i) for i in range(udb.n)]
    else:
        g = _group(case, devices)
        heads = sc.database()[0]
    out = os.path.join(tmp, f"{case}.gpu.tsv")
    st = g.sintax_stream(heads, qf, out, seed, strand_both=both, cutoff=cutoff, batch_queries=batch_queries)
    g.close()
    return open(out, "rb").read(), st


@pytest.mark.parametrize("case", list(sc.CASES))
def test_stream_matches_reference_cli(case, tmp_path):
    got, st = _stream(case, str(tmp_path))
    assert checkers.digest(got) == sc.reference("cli", case, lambda: sc.run_cli(case, str(tmp_path)))
    rows = got.decode().splitlines()
    nq = len(sc.data()["q_seqs"])
    assert len(rows) == nq == st["rows"] == st["queries"]
    cls = [r for r in rows if r.split("\t")[1] != ""]
    assert 0 < len(cls) < nq and st["matched"] == len(cls)
    if sc.CASES[case][2]:
        assert any(r.split("\t")[2] == "-" for r in cls)
    # the stream in many small batches numbers its queries the same way
    if case == "a_defaults":
        small, st2 = _stream(case, str(tmp_path), batch_queries=37)
        assert small == got and st2["batches"] > 5


def test_dbmask_changes_rows(tmp_path):
    """(a) excludes the database's lower-case low-complexity stretches from the index, (b) does not"""
    a, _ = _stream("a_defaults", str(tmp_path))
    b, _ = _stream("b_nomask_both_cutoff", str(tmp_path))
    ra, rb = a.decode().splitlines(), b.decode().splitlines()
    d = sc.data()
    lc_rows = [i for i, s in enumerate(d["q_seqs"]) if i < len(ra) and ra[i].split("\t")[1] != rb[i].split("\t")[1]]
    assert lc_rows


@pytest.mark.parametrize("case", sc.PER_BOOTSTRAP)
def test_bootstraps_match_reference(case):
    k, mask, both, _, seed, _ = sc.CASES[case]
    ctx = lib.Context(0)
    db = ctx.seqset(_seqset(sc.database()[1]))
    ix = ctx.index(db, wordlength=k, mask_lower=mask)
    q = sc.data()["q_seqs"]
    qs = ctx.seqset(_seqset(q))
    res = ctx.sintax(ix, qs, 0, len(q), seed, strand_both=both)
    arr = sc.as_array(res)
    assert checkers.digest(arr) == sc.reference("boots", case, lambda: sc.ref_bootstraps(case))
    meta = sc.data()["meta"]
    assert (arr[meta["short_queries"], 1:3] == 0).all()        # fewer than 32 distinct k-mers: no bootstraps
    assert (arr[meta["long_queries"], 1:3].max(axis=1) > 0).all()   # the HBM first-occurrence path ran
    # the database's tie pairs: a winner that ties with its copy must be the lower number / the shorter one
    lo, hi = meta["tie_seqno"]
    longer, shorter = meta["tie_length"]
    winners = arr[:, 5:]
    assert (winners == lo).any() and not (winners == hi).any()          # exact duplicates: the lower number wins
    assert (winners == shorter).any() and not (winners == longer).any()  # one base longer: the shorter one wins
    # a slice with its own query numbers equals that slice of the whole call
    part = sc.as_array(ctx.sintax(ix, qs, 100, 57, seed, strand_both=both, query_number0=100))
    assert (part == arr[100:157]).all()
    for h in (qs, ix, db):
        h.close()
    ctx.close()


def test_group_of_two_equals_one(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one, _ = _stream("c_k12_both", str(tmp_path))
    two, _ = _stream("c_k12_both", str(tmp_path), devices=(0, 1))
    assert one == two


def test_errors():
    ctx = lib.Context(0)
    db = ctx.seqset(_seqset(sc.database()[1][:20]))
    ix = ctx.index(db, wordlength=8, mask_lower=1)
    qs = ctx.seqset(_seqset([b"ACGT" * 60, b"ACGT" * 17000]))
    with pytest.raises(lib.VsgError, match=r"\(-3\).*sintax_random"):
        ctx.sintax(ix, qs, 0, 1, 1, random_ties=1)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*out of bounds"):
        ctx.sintax(ix, qs, 1, 5, 1)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*out of bounds"):
        ctx.sintax(ix, qs, -1, 1, 1)
    with pytest.raises(lib.VsgError, match=r"\(-3\).*longer than the device ranker supports \(65 534 \+ wordlength nt\)"):
        ctx.sintax(ix, qs, 1, 1, 1)
    o = lib.sintax_opts(1, cutoff=2.0)
    r = np.zeros(1, dtype=lib.SINTAX_DT)
    import ctypes as C
    assert lib.load().vsg_sintax(ctx.h, ix.h, qs.h, C.c_int64(0), C.c_int64(1), C.byref(o), r.ctypes.data_as(C.c_void_p)) == -3
    assert ctx.sintax(ix, qs, 0, 0, 1)["strand"].shape == (0,)   # an empty batch is a no-op
    import torch
    if torch.cuda.device_count() >= 2:
        ctx1 = lib.Context(1)
        with pytest.raises(lib.VsgError, match=r"\(-3\).*another device"):
            lib.Context.sintax(ctx1, ix, qs, 0, 1, 1)
        ctx1.close()
    for h in (qs, ix, db):
        h.close()
    ctx.close()
