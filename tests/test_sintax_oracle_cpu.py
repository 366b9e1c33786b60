"""The SINTAX oracle (oracle/sintax.c) pinned to the reference on the CPU: oracle_sintax's 205-int row equals
vsref_sintax's (the reference's own k-mers, generator, draws and sintax_search_topscores) query by query, on the
SINTAX fixture at every word length from 3 to 15 with and without lower-case masking on one and on both strands, on a
database of three index shards with planted ties across them, and under extreme seeds and query numbers.  The GPU
tests compare vsg_sintax with this oracle at shapes the reference's stored digests cannot reach."""
import ctypes as C

import numpy as np
import pytest

import checkers
import sintax_cases as sc
from vsearch_b200 import synth

needs_ref = pytest.mark.skipif(not sc.reference_available(), reason="oracle/_ref (reference CLI + sintax shim) not built")

pytestmark = needs_ref


class RefSintax:
    def __init__(self, ss, k, mask_lower):
        self.lens = ss.lens.astype(np.int32)
        self.cat = ss.cat.tobytes()
        self.h = sc.shim().vsref_sintax_db_create(len(ss), self.cat, ss.offs.ctypes.data_as(C.POINTER(C.c_int64)),
                                                  self.lens.ctypes.data_as(C.POINTER(C.c_int)), k, mask_lower)

    def row(self, q, query_number, seed, strand_both):
        out = np.zeros(205, dtype=np.int32)
        sc.shim().vsref_sintax(self.h, q, len(q), query_number, seed, strand_both, out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    def close(self):
        sc.shim().vsref_sintax_db_free(self.h)


def compare(ss, queries, k, mask_lower, runs):
    """runs: (query numbers, seed, strand_both) triples; returns the reference's rows of the last run"""
    ref = RefSintax(ss, k, mask_lower)
    od = checkers.OracleDb(ss, k=k, mask_lower=mask_lower)
    try:
        for qnums, seed, both in runs:
            want = np.stack([ref.row(q, n, seed, both) for q, n in zip(queries, qnums)])
            got = np.stack([od.sintax(q, n, seed, both) for q, n in zip(queries, qnums)])
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.shape[0] == 0, (k, mask_lower, seed, both, len(bad), int(bad[0]), got[bad[0], :12].tolist(),
                                       want[bad[0], :12].tolist())
    finally:
        od.close(); ref.close()
    return want


@pytest.mark.parametrize("k", list(range(3, 16)))
def test_oracle_equals_reference_every_wordlength(k):
    _, seqs = sc.database()
    q = sc.data()["q_seqs"]
    ss = synth.SeqSet(seqs)
    nums = list(range(len(q)))
    for mask_lower in (0, 1):
        rows = compare(ss, q, k, mask_lower, [(nums, 42, 0), (nums, 2 ** 33 + 5, 1)])
        # the fixture classifies on both strands at every k: bootstraps succeed on each
        assert (rows[:, 1] > 0).sum() > 100 and (rows[:, 2] > 0).sum() > 50 and (rows[:, 0] == 1).any(), k


@pytest.mark.parametrize("k", [3, 8, 11, 15])
def test_oracle_equals_reference_three_shards(k):
    d = sc.three_shard_data()
    ss = synth.SeqSet(d["db_seqs"])
    assert len(ss) > 2 * sc.SHARD and (len(ss) - 2 * sc.SHARD) % 2 == 1
    q = d["q_seqs"]
    rows = compare(ss, q, k, 0, [(list(range(len(q))), 9, 1)])
    winners = rows[:, 5:]
    assert not np.isin(winners, d["meta"]["never"]).any()
    assert {int(t) // sc.SHARD for t in winners[winners >= 0]} == {0, 1, 2}


def test_oracle_equals_reference_seeds_and_query_numbers():
    _, seqs = sc.database()
    q = sc.data()["q_seqs"][:60]
    runs = [([2 ** 32 - 3 + i for i in range(len(q))], seed, 1) for seed in (0, 1, 2 ** 63, 2 ** 64 - 1)]
    runs.append(([2 ** 40 + 7 + i for i in range(len(q))], 2 ** 64 - 1, 0))
    compare(synth.SeqSet(seqs), q, 8, 1, runs)
