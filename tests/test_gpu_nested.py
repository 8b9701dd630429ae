"""Nested BooleanQuerys on the device (rg_search_batch_nested, k_eval_and_nested): pure-SHOULD groups of terms as
MUST / FILTER / SHOULD / MUST_NOT clauses beside terms and point ranges, against the oracle's recursive
BooleanWeight::create_scorer (tests/cpp/orc_nested.cpp), bit for bit: docids, f32 score bits, tie order, counts and
total_hits, in both collector modes."""
import numpy as np
import pytest

import nested_fixtures as nf
import nested_oracle as no
import oracle_binding as ob
import points_oracle as po
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

_CACHE = {}
_EDGE = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    """each cached searcher holds an engine's arenas in HBM: give them back before later modules start processes"""
    yield
    for cache in (_CACHE, _EDGE):
        for entry in cache.values():
            entry[-2].engine.close()
        cache.clear()


def fixture(doc_version=1, flags=0, range_postings=0):
    key = (doc_version, flags, range_postings)
    if key not in _CACHE:
        segs, points, _ = nf.build(31 + doc_version, doc_version=doc_version)
        s = search.GpuIndexSearcher(search.IndexReader(segs), device=0, range_postings=range_postings, flags=flags)
        ix = no.NestedIndex(segs)
        for si, leaf in enumerate(points):
            for f, (nb, d, p, _) in leaf.items():
                ix.add_points(si, f, nb, d, p)
                s.engine.upload_points(si, f, nb, d, p)
        _CACHE[key] = (segs, points, s, ix)
    return _CACHE[key]


def ranges():
    return np.array([po.make_range(0, 8, po.long_pack(1275), po.long_pack(200000)),
                     po.make_range(1, 4, po.int_pack(-(1 << 29)), po.int_pack(1 << 28)),
                     po.make_range(0, 8, po.long_pack(-(1 << 40)), po.long_pack(1 << 40))], po.RANGE_DTYPE)


def same(got, want, label):
    gh, gc, gt = got
    wh, wc, wt = want
    assert np.array_equal(gt, wt), (label, "total_hits", np.nonzero(gt != wt)[0][:5])
    assert np.array_equal(gc, wc), (label, "counts", np.nonzero(gc != wc)[0][:5])
    for i in range(len(gc)):
        n = int(wc[i])
        assert np.array_equal(gh[i][:n]["doc"], wh[i][:n]["doc"]), (label, "docs of query", i)
        assert np.array_equal(gh[i][:n]["score"].view(np.uint32), wh[i][:n]["score"].view(np.uint32)), (label, "scores", i)


def run(s, ix, sp, k, mode=engine.MODE_SEARCH):
    rg = ranges()
    oq, oc, og = no.to_arrays(sp)
    eq, ec, eg = no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og)
    want = ix.search_batch(oq, oc, og, k, ranges=rg, parallel_mode=mode)
    got = s.engine.search_batch_nested(eq, ec, eg, k, k1=s.similarity.k1, mode=mode, ranges=rg)
    return got, want


@pytest.mark.parametrize("doc_version", [0, 1])
@pytest.mark.parametrize("k", [1, 10, 1000])
def test_every_shape_matches_the_oracle(doc_version, k):
    segs, points, s, ix = fixture(doc_version)
    sp = nf.specs([0, 1, 2])
    for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
        got, want = run(s, ix, sp, k, mode)
        same(got, want, ("v", doc_version, "k", k, "mode", mode))


@pytest.mark.parametrize("flags", [engine.CFG_EAGER_COLUMNS, engine.CFG_NO_BITMAPS, engine.CFG_NO_LISTS])
def test_engine_configurations(flags):
    segs, points, s, ix = fixture(1, flags)
    for k in (10, 1000):
        same(*run(s, ix, nf.specs([0, 1, 2]), k), ("flags", flags, k))


@pytest.mark.parametrize("rp", [0, 300])
def test_docid_ranges(rp):
    """range_postings 0 (one item per leaf) and a small value (group leads cut into many items: docs at lo - 1 and
    lo of each item)."""
    segs, points, s, ix = fixture(1, 0, rp)
    for k in (10, 1000):
        same(*run(s, ix, nf.specs([0, 1, 2]), k), ("range_postings", rp, k))


def test_group_leads_run():
    """The 8-member group leads and merges postings that several members share."""
    segs, points, s, ix = fixture(1)
    sp = [("bool", [(ob.MUST, [(4,), (5,), (8,), (9,), (3,), (1,), (7,), (2,)], 0), (ob.MUST, 0)], 0),
          ("bool", [(ob.MUST, [(0,), (6,)], 0), (ob.MUST, [(1,), (2,)], 0)], 0)]
    oq, oc, og = no.to_arrays(sp)
    b = s.engine.prepare(no.engine_queries(oq), ix.engine_clauses(oc), 100, k1=s.similarity.k1,
                         groups=no.engine_queries(og))
    try:
        b.run()
        st = b.group_stats()
        got = b.fetch()
    finally:
        b.close()
    same(got, ix.search_batch(oq, oc, og, 100), "stats batch")
    assert st["items"] >= 2 * len(segs) - 2 and st["merged"] > 0 and st["holes"] > 0, st


def test_refused_shapes():
    segs, points, s, ix = fixture(1)
    for sp in nf.refused_specs():
        oq, oc, og = no.to_arrays([sp])
        with pytest.raises(engine.Unsupported):
            s.engine.search_batch_nested(no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og), 10)


def test_old_entry_points_reject_the_group_bit():
    segs, points, s, ix = fixture(1)
    oq, oc, og = no.to_arrays([("bool", [(ob.MUST, [(0,), (1,)], 0), (ob.MUST, 2)], 0)])
    eq, ec = no.engine_queries(oq), ix.engine_clauses(oc)
    with pytest.raises(engine.EngineError) as e:
        s.engine.search_batch(eq, ec, 10)
    assert e.value.code == engine.RG_EINVAL
    with pytest.raises(engine.EngineError) as e:
        s.engine.search_batch_ranges(eq, ec, ranges(), 10)
    assert e.value.code == engine.RG_EINVAL


def test_invalid_groups():
    segs, points, s, ix = fixture(1)
    oq, oc, og = no.to_arrays([("bool", [(ob.MUST, [(0,), (1,)], 0), (ob.MUST, 2)], 0)])
    eq, ec, eg = no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og)
    bad = ec.copy()
    bad[0]["term_id"] = 5  # group index outside the array
    overlap = eg.copy()
    overlap[0]["clause_begin"] = 1  # members overlap the query's own clauses
    oob = eg.copy()
    oob[0]["n_clauses"] = 50
    member = ec.copy()
    member[2]["occur"] = 7  # unknown occur
    for c, gr in ((bad, eg), (ec, overlap), (ec, oob), (member, eg)):
        with pytest.raises(engine.EngineError) as e:
            s.engine.search_batch_nested(eq, c, gr, 10)
        assert e.value.code == engine.RG_EINVAL


# ---- constructed edges of a group that leads -----------------------------------------------------------------------


def edge_fixture(doc_version, use_ef, rp):
    key = (doc_version, use_ef, rp)
    if key not in _EDGE:
        seg, post = nf.edge_leaf(doc_version=doc_version, use_ef=use_ef)
        s = search.GpuIndexSearcher(search.IndexReader([seg]), device=0, range_postings=rp)
        _EDGE[key] = (seg, s, no.NestedIndex([seg]))
    return _EDGE[key]


@pytest.mark.parametrize("doc_version,use_ef", [(0, False), (1, False), (1, True)])
@pytest.mark.parametrize("rp", [0, nf.SPLIT_RP])
def test_group_lead_edges(doc_version, use_ef, rp):
    """interleaved member blocks, one docid in all 8 members, a step of exactly 1024 entries, members that run out
    mid-item, singletons and tails, and (at range_postings SPLIT_RP) docs at lo - 1 and lo of every item"""
    seg, s, ix = edge_fixture(doc_version, use_ef, rp)
    sp = nf.edge_specs()
    oq, oc, og = no.to_arrays(sp)
    eq, ec, eg = no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og)
    for k in (10, 1000):
        for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
            want = ix.search_batch(oq, oc, og, k, parallel_mode=mode)
            b = s.engine.prepare(eq, ec, k, k1=s.similarity.k1, mode=mode, groups=eg)
            try:
                b.run()
                st = b.group_stats()
                got = b.fetch()
            finally:
                b.close()
            same(got, want, ("edges", doc_version, use_ef, rp, k, mode))
            # every query but the FILTER one is led by its group; with SPLIT_RP the split query has SPLIT_R items
            assert st["items"] >= len(sp) - 1 + (nf.SPLIT_R - 1 if rp else 0), st
            assert st["holes"] >= 7 + 7, st   # docs 6200 and 15000 in all eight members


# ---- through the public search API ---------------------------------------------------------------------------------
def test_gpu_index_searcher_routes_nested_queries():
    segs, points, s, ix = fixture(1)
    T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
    B = search.BooleanQuery.build
    G = lambda *ts: B([], [T(t) for t in ts], [], [])
    queries = [B([G(0, 1), G(2, 3)], [], [], []), B([T(4), G(5, 6)], [], [], [T(7)]), B([G(0, 6)], [T(2)], [], []),
               B([], [], [G(1, 3)], [T(6)]), B([T(0)], [], [], [G(2, 3)]), B([G(4, 9), T(1)], [G(5, 7)], [], []),
               B([G(0, 1)], [], [], []), B([G(2, 5)], [], [], [T(0)])]
    q, c, r, g = s.compile_batch_nested(queries)
    assert len(g) > 0
    oq = np.zeros(len(q), ob.QUERY_DTYPE)
    oq["clause_begin"], oq["n_clauses"], oq["min_should_match"] = q["clause_begin"], q["n_clauses"], q["min_should_match"]
    oq["is_boolean"] = q["flags"] & engine.Q_BOOLEAN
    og = np.zeros(len(g), ob.QUERY_DTYPE)
    og["clause_begin"], og["n_clauses"], og["min_should_match"], og["is_boolean"] = \
        g["clause_begin"], g["n_clauses"], g["min_should_match"], 1
    oc = np.zeros(len(c), ob.CLAUSE_DTYPE)
    oc["occur"], oc["term_id"], oc["boost"] = c["occur"], c["term_id"], 1.0
    for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
        same(s.search_batch(queries, 100, mode=mode), ix.search_batch(oq, oc, og, 100, parallel_mode=mode),
             ("searcher", mode))
    with pytest.raises(engine.Unsupported):
        s.search_batch([B([], [G(0, 1), G(2, 3)], [], [])], 10)   # (a|b) (c|d)
    with pytest.raises(engine.Unsupported):
        s.search_batch([B([B([T(0)], [T(1)], [], []), T(2)], [], [], [])], 10)   # a group with a MUST member
