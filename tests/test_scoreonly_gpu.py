"""Score-only checkpoint tasks (align_ckpt.cuh, CK_SCOREONLY / CK_RERUN): in a search call with traceback on demand, a
forward task whose two pairs are both group followers stores no checkpoints, and the tasks phase 2 walks after all are
recomputed with stores once the leaders' verdicts are in.  The hit tables must not depend on it: the shapes of
test_search_gpu.py's traceback-on-demand test, with every leader forced to "rejected" (so every score-only task is
re-run and every follower walked from the re-run's checkpoints), with the score-only tasks switched off, and both."""
import contextlib
import os

import pytest

import checkers
from vsearch_b200 import lib as vlib
from vsearch_b200 import synth

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def rows_of(res, counts, q, max_results):
    out = []
    for j in range(int(counts[q])):
        r = res[q * max_results + j]
        out.append([r.target, r.id, r.matches, r.mismatches, r.gaps, r.alignment_length, r.accepted, r.strand])
    return out


@pytest.mark.parametrize("maxaccepts,ident", [(1, 0.9), (1, 0.97), (3, 0.9)])
def test_scoreonly_tasks_do_not_change_the_hit_tables(maxaccepts, ident):
    dbs, qss, src = synth.config2_search(n_db=600, db_len=1500, n_q=400, q_len=250, div=0.05, seed=91)
    kw = dict(id=ident, maxaccepts=maxaccepts, maxrejects=16)

    def run_reference():
        rows, th = checkers.ref_search(dbs, qss, **kw)
        return checkers.digest(rows), th
    want, th = checkers.reference("traceback_on_demand", (dbs, qss, kw), run_reference, checkers.ref() is not None)
    ctx = vlib.Context(0)
    db = ctx.seqset(dbs); qs = ctx.seqset(qss)
    ix = ctx.index(db, 8, 0)
    o = vlib.default_search_opts()
    o.id = ident; o.maxaccepts = maxaccepts; o.maxrejects = 16; o.strand_both = 0; o.mask_lower = 0; o.wordlength = 8
    try:
        # the checkpoint kernels at this call size too, no tail prefetch (every round goes through the gated calls)
        with env(VSG_CKPT_MIN_PAIRS="0", VSG_TAIL_PAIRS="0"):
            for case in ({"VSG_TB_GATE_FORCE": "2"}, {"VSG_TB_GATE_FORCE": "2", "VSG_CK_SCOREONLY": "0"},
                         {"VSG_CK_SCOREONLY": "0"}, {}):
                with env(**case):
                    res, counts, work = ctx.search(ix, db, qs, 0, len(qss), o, th)
                assert checkers.digest([rows_of(res, counts, i, th) for i in range(len(qss))]) == want, case
                # nwscore included: a follower's score comes from the score-only pass
                assert checkers.check_search_rows(res, counts, th, qss, dbs) > 0, case
    finally:
        ix.close(); db.close(); qs.close()
        ctx.close()
