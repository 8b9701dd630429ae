"""GPU parity of the conjunction kernels on constructed worst cases (and_fixtures.py; test_and_edges_cpu.py checks the
fixtures themselves): term-led conjunctions on lead and probe block edges, galloping, items cut by range_postings,
every freq width, EF / BITSET blocks, MUST_NOT, FILTER and -0.0 (k_eval_and<false, *>); the ReqOpt running mean
(k_eval_and<true, *>); range leads and range probes (k_eval_and_ranges<*, *>).  TopDocs must be the oracle's, bit for
bit, in both collector modes, in the planner default, with eager score columns and without bitmaps."""
import numpy as np
import pytest

import and_fixtures as A
import helpers
import points_oracle as po
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

FLAGS = {"default": 0, "eager": engine.CFG_EAGER_COLUMNS, "no_bitmaps": engine.CFG_NO_BITMAPS}
MODES = (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL)


def _term_batch(segs, specs, k, mode, rp, flags):
    """-> (TopDocs, planner stats)"""
    s = search.GpuIndexSearcher(search.IndexReader(segs), range_postings=rp, flags=flags)
    try:
        qa, ca = s.compile_batch(helpers.to_queries(specs))
        bt = s.engine.prepare(qa, ca, k, k1=s.similarity.k1, mode=mode)
        try:
            bt.run()
            return bt.fetch(), bt.stats()
        finally:
            bt.close()
    finally:
        s.engine.close()


def _oracle(segs, specs, k, mode):
    q, c = A.queries(specs)
    return helpers.oracle_index(segs).search_batch(q, c, k, parallel_mode=mode, n_threads=4)


# ---- A. term-led conjunctions ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(A.A_VARIANTS))
def test_term_led_conjunction_edges(variant):
    f = A.TermLeadFixture(variant)
    if A.A_VARIANTS[variant][1]:
        assert f.block_counts[1] + f.block_counts[2] > 0, f.block_counts   # k_eval_and<false, true> runs
    specs = f.specs()
    for k in (10, 1000):
        for mode in MODES:
            want = _oracle(f.segs, specs, k, mode)
            for name, flags in FLAGS.items():
                for rp in (0, A.A_CUT_RP):
                    if k == 10 and (name != "default" or rp):
                        continue
                    got, _ = _term_batch(f.segs, specs, k, mode, rp, flags)
                    helpers.assert_same_topdocs(got, want, "%s k=%d mode=%d %s rp=%d" % (variant, k, mode, name, rp))


# ---- B. ReqOpt ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ef", [False, True], ids=["plain", "ef"])
def test_reqopt_running_mean(ef):
    f = A.ReqOptFixture(ef=ef)
    if ef:
        assert f.counts[4][1] + f.counts[4][2] > 0, f.counts[4]   # k_eval_and<true, true> runs
    specs = f.specs()
    for k in (A.B_K, 1000):
        for mode in MODES:
            want = _oracle(f.segs, specs, k, mode)
            for name, flags in FLAGS.items():
                for rp in (0, 64):
                    got, st = _term_batch(f.segs, specs, k, mode, rp, flags)
                    helpers.assert_same_topdocs(got, want, "ef=%d k=%d mode=%d %s rp=%d" % (ef, k, mode, name, rp))
    # the ReqOpt leaves stay one item each (their chain is sequential); the plain leaf 4 is cut at rp = 64
    _, st = _term_batch(f.segs, specs, A.B_K, 0, 64, 0)
    assert st["items"] > 4 * len(specs), st


# ---- C. range conjunctions ---------------------------------------------------------------------------------------------
def _engine_queries(oq):
    q = np.zeros(len(oq), engine.QUERY_DTYPE)
    for fld in ("clause_begin", "n_clauses", "min_should_match"):
        q[fld] = oq[fld]
    q["flags"] = np.where(oq["is_boolean"] == 1, engine.Q_BOOLEAN, 0)
    return q


@pytest.mark.parametrize("ef", [False, True], ids=["plain", "ef"])
def test_range_conjunction_edges(ef):
    f = A.RangeFixture(ef=ef)
    if ef:
        assert f.block_counts[1] + f.block_counts[2] > 0, f.block_counts   # k_eval_and_ranges<*, true> runs
    ix = po.PointsIndex(f.segs)
    for si, leaf in enumerate(f.points):
        for fld, (nb, d, p, _) in leaf.items():
            ix.add_points(si, fld, nb, d, p)
    specs = f.specs(len(f.ranges))
    oq, oc = A.queries(specs)
    eq, ec = _engine_queries(oq), ix.engine_clauses(oc)
    seen = {"skipped": 0, "whole": 0, "scanned": 0}
    for k in (10, 1000):
        for mode in MODES:
            want = ix.search_batch(oq, oc, f.ranges, k, parallel_mode=mode)
            for name, flags in FLAGS.items():
                for rp in (0, A.C_SPLIT_RP):
                    s = search.GpuIndexSearcher(search.IndexReader(f.segs), range_postings=rp, flags=flags)
                    try:
                        for si, leaf in enumerate(f.points):
                            for fld, (nb, d, p, _) in leaf.items():
                                s.engine.upload_points(si, fld, nb, d, p)
                        bt = s.engine.prepare(eq, ec, k, k1=s.similarity.k1, mode=mode, ranges=f.ranges)
                        try:
                            bt.run()
                            got = bt.fetch()
                            rs, st = bt.range_stats(), bt.stats()
                        finally:
                            bt.close()
                    finally:
                        s.engine.close()
                    helpers.assert_same_topdocs(got, want, "ef=%d k=%d mode=%d %s rp=%d" % (ef, k, mode, name, rp))
                    for n in seen:
                        seen[n] += rs[n]
                    if rp:   # range-led conjunctions and range-only ReqOpts on range 7 (and others) are cut into 4
                        assert st["items"] >= items_whole + 3 * 4, (st, items_whole)
                    else:
                        items_whole = st["items"]
    assert seen["skipped"] > 0 and seen["whole"] > 0 and seen["scanned"] > 0, seen
