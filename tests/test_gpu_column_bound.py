"""GPU parity of the decode-free k_eval_or's column bound: a whole window in which only score columns have postings is
counted from the columns' presence bitmaps when their block maxima cannot beat theta, and summed as before otherwise.
TopDocs must be the oracle's whatever theta does (large k keeps it low), wherever the columns sit in clause order, next
to very sparse lists, for ranges that are not 32-aligned, with live docs and two leaves."""
import numpy as np
import pytest

import helpers
import oracle_binding as ob
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

# 0-4: score columns at the default threshold (df >= max_doc / 8); 5-9: scored lists; 10-13: very sparse lists
DFS = [40000, 25000, 12000, 9000, 6500, 3000, 1500, 700, 385, 129, 40, 9, 3, 1]


def _segments(rng):
    return [helpers.build_segment(rng, 50000, DFS, doc_version=1, live_fraction=0.9 if i else None)[0] for i in range(2)]


def _specs(rng):
    def sh(ts):
        return ("bool", [(ob.SHOULD, t) for t in ts], 0)
    specs = []
    for _ in range(2):  # every shape twice: a column needs two uses in the batch
        specs += [sh([0, 7]), sh([1, 12]), sh([8, 2, 11]), sh([9, 10, 3]), sh([6, 0, 1, 13]),  # first / middle / last
                  sh([0, 1]), sh([2, 3, 4]), sh([0, 1, 2, 3, 4]),                               # columns only
                  sh([4, 13]), sh([12, 3]), sh([0, 10, 11, 12, 13])]                             # next to sparse lists
    for ts in helpers.distinct_query_terms(rng, len(DFS), 40, 2, 6):
        specs.append(sh(ts))
    return specs


def _run(s, specs, k, mode):
    qa, ca = s.compile_batch(helpers.to_queries(specs))
    b = s.engine.prepare(qa, ca, k, k1=s.similarity.k1, mode=mode)
    try:
        b.run()
        return b.fetch(), b.debug()
    finally:
        b.close()


def test_column_bound_matches_the_oracle(monkeypatch):
    rng = np.random.default_rng(707)
    segs = _segments(rng)
    ix = helpers.oracle_index(segs)
    specs = _specs(rng)
    q, c = ob.make_queries(specs)
    for den in (None, "64"):  # 64: the lists of terms 5 and 6 become columns too
        if den is None:
            monkeypatch.delenv("RG_OR_COL_DEN", raising=False)
        else:
            monkeypatch.setenv("RG_OR_COL_DEN", den)
        for mode in (0, 1):
            for k in (1, 10, 100, 1000):
                want = ix.search_batch(q, c, k, parallel_mode=mode, n_threads=4)
                for flags in (0, engine.CFG_EAGER_COLUMNS):
                    for rp in (0, 700):  # 700: many ranges per leaf, most of them not 32-aligned
                        label = "den=%s mode=%d k=%d flags=%d rp=%d" % (den, mode, k, flags, rp)
                        s = search.GpuIndexSearcher(search.IndexReader(segs), range_postings=rp, flags=flags)
                        try:
                            got, dbg = _run(s, specs, k, mode)
                            helpers.assert_same_topdocs(got, want, label)
                            assert dbg["decode_free_items"] > 0, label
                        finally:
                            s.engine.close()


def test_column_sweep_switch_and_counters(monkeypatch):
    """RG_CFG_STATS counts the columns-only windows of the decode-free kernel; RG_COLUMN_SWEEP=1 reads every column
    cell (nothing counted from bitmaps) and gives the same TopDocs."""
    rng = np.random.default_rng(808)
    segs = _segments(rng)
    ix = helpers.oracle_index(segs)
    specs = _specs(rng)
    q, c = ob.make_queries(specs)
    want = ix.search_batch(q, c, 10, parallel_mode=0, n_threads=4)
    seen = {}
    for sweep in ("0", "1"):
        monkeypatch.setenv("RG_COLUMN_SWEEP", sweep)
        s = search.GpuIndexSearcher(search.IndexReader(segs), range_postings=0, flags=engine.CFG_STATS)
        try:
            got, dbg = _run(s, specs, 10, 0)
            helpers.assert_same_topdocs(got, want, "RG_COLUMN_SWEEP=" + sweep)
            seen[sweep] = dbg
        finally:
            s.engine.close()
    assert seen["0"]["column_windows_from_bitmaps"] > 0, seen["0"]
    assert seen["1"]["column_windows_from_bitmaps"] == 0, seen["1"]
    assert seen["1"]["column_windows_swept"] > 0, seen["1"]
