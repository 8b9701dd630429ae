"""GPU parity of the decode-free k_eval_or: plain-sum disjunctions whose clauses that are not score columns get
batch-local scored lists, so every clause of the item is a column or a list.  Which configurations route items
there, and that the TopDocs are the oracle's for every block layout, vint tails, docid ranges that cut blocks,
live docs and several leaves."""
import numpy as np
import pytest

import helpers
import oracle_binding as ob
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu


def _decode_free_items(s, specs, k, mode, want, label):
    qa, ca = s.compile_batch(helpers.to_queries(specs))
    b = s.engine.prepare(qa, ca, k, k1=s.similarity.k1, mode=mode)
    try:
        b.run()
        helpers.assert_same_topdocs(b.fetch(), want, label)
        return b.debug()["decode_free_items"]
    finally:
        b.close()


def test_decode_free_route_every_block_layout():
    rng = np.random.default_rng(505)
    dfs = [40000, 25000, 12000, 6000, 3000, 1500, 700, 385, 300, 129, 128, 127, 5, 1]
    for version, use_ef in ((1, False), (0, False), (1, True)):
        segs = [helpers.build_segment(rng, 50000, dfs, doc_version=version, use_ef=use_ef,
                                      live_fraction=0.9 if i else None)[0] for i in range(2)]
        ix = helpers.oracle_index(segs)
        specs = [("term", t) for t in range(len(dfs))]
        for ts in helpers.distinct_query_terms(rng, len(dfs), 60, 1, 6):
            specs.append(("bool", [(ob.SHOULD, t) for t in ts], 0))
        # a MUST_NOT clause and a zero boost keep their queries on the stream path
        specs += [("bool", [(ob.SHOULD, 0), (ob.SHOULD, 9), (ob.MUST_NOT, 3)], 0),
                  ("bool", [(ob.SHOULD, 1, 0.0), (ob.SHOULD, 12)], 0)]
        for mode in (0, 1):
            q, c = ob.make_queries(specs)
            want = ix.search_batch(q, c, 20, parallel_mode=mode, n_threads=4)
            for flags, routed in ((0, True), (engine.CFG_EAGER_COLUMNS, True),
                                  (engine.CFG_EAGER_COLUMNS | engine.CFG_NO_LISTS, False),
                                  (engine.CFG_NO_BITMAPS | engine.CFG_NO_LISTS, False)):
                for rp in (0, 3000):
                    label = "decode-free v%d ef%d flags=%d mode=%d rp=%d" % (version, use_ef, flags, mode, rp)
                    s = search.GpuIndexSearcher(search.IndexReader(segs), range_postings=rp, flags=flags)
                    try:
                        n = _decode_free_items(s, specs, 20, mode, want, label)
                        assert (n > 0) == routed, (label, n)
                    finally:
                        s.engine.close()


def test_local_list_budget_keeps_the_rest_on_block_streams(monkeypatch):
    """Batch-local lists are taken smallest first within a byte budget: a tighter budget routes fewer items to the
    decode-free kernel (the items it leaves keep block streams next to the lists they did get, in the stream variant),
    and every budget gives the oracle's TopDocs."""
    rng = np.random.default_rng(606)
    dfs = [40000, 25000, 12000, 6000, 3000, 1500, 700, 385, 300, 129, 128, 127, 5, 1]
    segs = [helpers.build_segment(rng, 50000, dfs, doc_version=1, live_fraction=0.9 if i else None)[0] for i in range(2)]
    ix = helpers.oracle_index(segs)
    specs = [("term", t) for t in range(len(dfs))]
    for ts in helpers.distinct_query_terms(rng, len(dfs), 60, 1, 6):
        specs.append(("bool", [(ob.SHOULD, t) for t in ts], 0))
    q, c = ob.make_queries(specs)
    want = ix.search_batch(q, c, 20, parallel_mode=0, n_threads=4)
    routed = []
    for kb in (None, "64", "0"):
        if kb is None:
            monkeypatch.delenv("RG_LOCAL_LISTS_KB", raising=False)
        else:
            monkeypatch.setenv("RG_LOCAL_LISTS_KB", kb)
        s = search.GpuIndexSearcher(search.IndexReader(segs), range_postings=3000, flags=0)
        try:
            routed.append(_decode_free_items(s, specs, 20, 0, want, "local list budget %s KB" % kb))
        finally:
            s.engine.close()
    full, mid, none = routed
    assert full > mid >= none, routed
