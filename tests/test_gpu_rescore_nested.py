"""Rescoring with nested groups and point ranges on the device (rg_batch_rescore_nested / rg_rescore_hits_nested,
k_rescore<true>), against QueryRescorer over the oracle's recursive scorer trees (tests/cpp/orc_rescore_nested.cpp), bit
for bit: docids, f32 score bits, order, counts and total_hits."""
import numpy as np
import pytest

import nested_fixtures as nf
import nested_oracle as no
import oracle_binding as ob
import points_oracle as po
import rescore_nested_oracle as rno
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER
R = po.RANGE
MODES = (engine.RESCORE_TOTAL, engine.RESCORE_MULTIPLY, engine.RESCORE_AVG)
_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for entry in _CACHE.values():
        entry[0].engine.close()
    _CACHE.clear()


def ranges():
    return np.array([po.make_range(0, 8, po.long_pack(1275), po.long_pack(200000)),
                     po.make_range(1, 4, po.int_pack(-(1 << 29)), po.int_pack(1 << 28)),
                     po.make_range(0, 8, po.long_pack(-(1 << 40)), po.long_pack(1 << 40))], po.RANGE_DTYPE)


def fixture(kind="nested"):
    """(searcher, first-pass oracle, rescoring oracle, segs, points)"""
    if kind not in _CACHE:
        if kind == "nested":
            segs, points, _ = nf.build(32, doc_version=1)
        else:
            seg, _ = nf.edge_leaf(doc_version=1, use_ef=True)
            segs, points = [seg], [{}]
        s = search.GpuIndexSearcher(search.IndexReader(segs), device=0)
        ix, rx = no.NestedIndex(segs), rno.RescoreNestedIndex(segs)
        for si, leaf in enumerate(points):
            for f, (nb, d, p, _) in leaf.items():
                ix.add_points(si, f, nb, d, p)
                rx.add_points(si, f, nb, d, p)
                s.engine.upload_points(si, f, nb, d, p)
        _CACHE[kind] = (s, ix, rx, segs, points)
    return _CACHE[kind]


def first_specs(n, terms):
    """flat disjunctions, so that a window holds hits the rescoring query matches and hits it does not"""
    return [("bool", [(S, terms[(i + j) % len(terms)]) for j in range(3 + i % 3)], 0) for i in range(n)]


def arrays(ix, specs):
    oq, oc, og = no.to_arrays(specs)
    return (oq, oc, og), (no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og))


def same(got, want, label):
    gh, gc, gt = got
    wh, wc, wt = want
    assert np.array_equal(gt, wt), (label, "total_hits")
    assert np.array_equal(gc, wc), (label, "counts")
    for i in range(len(gc)):
        n = int(wc[i])
        assert np.array_equal(gh[i][:n]["doc"], wh[i][:n]["doc"]), (label, "docs of query", i)
        assert np.array_equal(gh[i][:n]["score"].view(np.uint32), wh[i][:n]["score"].view(np.uint32)), (label, "scores", i)


def device_rescore(s, first, k, cmode, req, window, rmode, nested=True, qw=1.0, rw=1.0):
    """first pass on the device, rescored on the device before the fetch"""
    eq, ec, _ = first
    rq, rc, rg, rr = req
    b = s.engine.prepare(eq, ec, k, k1=s.similarity.k1, mode=cmode)
    try:
        b.run()
        if nested:
            s.engine.rescore_batch(b, rq, rc, window, qw, rw, rmode, k1=s.similarity.k1, groups=rg, ranges=rr)
        else:
            s.engine.rescore_batch(b, rq, rc, window, qw, rw, rmode, k1=s.similarity.k1)
        return b.fetch()
    finally:
        b.close()


def check_specs(kind, specs, terms, k, cmode, windows, rng=None):
    s, ix, rx, segs, _ = fixture(kind)
    (fq, fc, fg), first = arrays(ix, first_specs(len(specs), terms))
    hits, counts, total = ix.search_batch(fq, fc, fg, k, parallel_mode=cmode)
    (oq, oc, og), (eq, ec, eg) = arrays(rx, specs)
    for rmode in MODES:
        for window in windows:
            qw, rw = (0.5, 1.5) if rmode == engine.RESCORE_MULTIPLY else (1.0, 2.0)
            want = rx.rescore(oq, oc, og, hits, counts, total, window, qw, rw, rmode, ranges=rng)
            got = device_rescore(s, first, k, cmode, (eq, ec, eg, rng), window, rmode, qw=qw, rw=rw)
            same(got, (want, counts, total), (kind, k, cmode, rmode, window))


@pytest.mark.parametrize("cmode", [engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL])
@pytest.mark.parametrize("k", [100, 1000])
def test_every_nested_shape_rescores_like_the_oracle(k, cmode):
    """every shape of nested_fixtures.specs as the rescoring query over the EF / BITSET leaf, the leaf with deleted
    docs and the point fields; windows of 1, 50 and the whole row; at k = 1000 the ReqOpt running mean passes 100"""
    check_specs("nested", nf.specs([0, 1, 2]), [0, 6, 3, 4, 7, 1, 9, 2], k, cmode, (1, 50, k), rng=ranges())


@pytest.mark.parametrize("cmode", [engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL])
def test_member_block_edges(cmode):
    """nested_fixtures.edge_leaf: interleaved member blocks, one docid in all 8 members, tails and singletons"""
    check_specs("edge", nf.edge_specs(), [1, 4, 12, 20, 21, 22, 23, 24, 25, 26], 1000, cmode, (50, 1000))


def test_rescore_hits_nested_with_deleted_docs():
    """host rows whose docids include deleted docs of leaf 1 (advance() does not consult live docs)"""
    s, ix, rx, segs, _ = fixture()
    specs = nf.specs([0, 1, 2])
    (oq, oc, og), (eq, ec, eg) = arrays(rx, specs)
    rng = np.random.default_rng(7)
    base1 = segs[0].max_doc
    words = np.asarray(segs[1].live_docs, np.uint64)
    dead = [d for d in range(segs[1].max_doc) if not (int(words[d >> 6]) >> (d & 63)) & 1]
    assert dead
    k = 300
    n_docs = sum(sg.max_doc for sg in segs)
    hits = np.zeros((len(specs), k), engine.HIT_DTYPE)
    for i in range(len(specs)):
        docs = np.concatenate([rng.choice(n_docs, k - 40, replace=False), base1 + rng.choice(dead, 40, replace=False)])
        hits[i]["doc"] = rng.permutation(docs)
        hits[i]["score"] = rng.random(k).astype(np.float32) * 10
    counts = np.full(len(specs), k, np.uint32)
    counts[::7] = 17
    total = np.full(len(specs), 5000, np.uint64)
    rr = ranges()
    for rmode in MODES:
        for window in (1, 50, k):
            want = rx.rescore(oq, oc, og, hits, counts, total, window, 1.0, 2.0, rmode, ranges=rr)
            got = s.engine.rescore_hits(eq, ec, hits, counts, total, window, 1.0, 2.0, rmode, k1=s.similarity.k1,
                                        groups=eg, ranges=rr)
            same((got, counts, total), (want, counts, total), ("hits", rmode, window))


def refused_specs():
    T = lambda *ts: [(t,) for t in ts]
    return nf.refused_specs() + [
        ("bool", [(M, 0), (S | R, 0)], 0),                         # a SHOULD range beside a required clause
        ("bool", [(M, T(0, 1, 2, 3, 4, 5, 6, 7, 8, 9))], 0),       # the query is a group of 10 members
    ]


def test_refused_shapes_leave_the_rows_untouched():
    s, ix, rx, segs, _ = fixture()
    (fq, fc, fg), first = arrays(ix, first_specs(1, [0, 6, 3]))
    for sp in refused_specs():
        _, (eq, ec, eg) = arrays(rx, [sp])
        b = s.engine.prepare(first[0], first[1], 100, k1=s.similarity.k1)
        try:
            b.run()
            with pytest.raises(engine.Unsupported):
                s.engine.rescore_batch(b, eq, ec, 50, groups=eg, ranges=ranges())
            got = b.fetch()
        finally:
            b.close()
        same(got, ix.search_batch(fq, fc, fg, 100), ("refused", sp))
        hits = np.array(got[0])
        with pytest.raises(engine.Unsupported):
            s.engine.rescore_hits(eq, ec, hits, got[1], got[2], 50, groups=eg, ranges=ranges())


def test_invalid_groups():
    s, ix, rx, segs, _ = fixture()
    _, first = arrays(ix, first_specs(1, [0, 6, 3]))
    _, (eq, ec, eg) = arrays(rx, [("bool", [(M, [(0,), (1,)], 0), (M, 2)], 0)])
    bad = ec.copy()
    bad[0]["term_id"] = 5      # group index outside the array
    overlap = eg.copy()
    overlap[0]["clause_begin"] = 1
    oob = eg.copy()
    oob[0]["n_clauses"] = 50
    for c, gr in ((bad, eg), (ec, overlap), (ec, oob)):
        b = s.engine.prepare(first[0], first[1], 10, k1=s.similarity.k1)
        try:
            b.run()
            with pytest.raises(engine.EngineError) as e:
                s.engine.rescore_batch(b, eq, c, 10, groups=gr)
            assert e.value.code == engine.RG_EINVAL
        finally:
            b.close()


@pytest.mark.parametrize("cmode", [engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL])
def test_flat_queries_through_the_nested_entry_point(cmode):
    """flat rescoring queries give the rows rg_batch_rescore gives, bit for bit"""
    s, ix, rx, segs, _ = fixture()
    flat = [("bool", [(M, a), (S, b), (N, c)], 0) for a, b, c in [(0, 3, 4), (6, 1, 2), (2, 9, 8), (7, 0, 5)]]
    flat += [("bool", [(S, a), (S, b)], 0) for a, b in [(0, 1), (3, 9), (4, 6)]]
    flat += [("bool", [(M, a), (F, b)], 0) for a, b in [(0, 6), (1, 3)]]
    _, first = arrays(ix, first_specs(len(flat), [0, 6, 3, 4, 7]))
    _, (eq, ec, eg) = arrays(rx, flat)
    for rmode in MODES:
        old = device_rescore(s, first, 1000, cmode, (eq, ec, None, None), 500, rmode, nested=False)
        new = device_rescore(s, first, 1000, cmode, (eq, ec, eg, ranges()), 500, rmode)
        same(new, old, ("flat", rmode))


def test_old_entry_points_reject_the_group_and_range_bits():
    s, ix, rx, segs, _ = fixture()
    _, first = arrays(ix, first_specs(1, [0, 6, 3]))
    for sp in (("bool", [(M, [(0,), (1,)], 0), (M, 2)], 0), ("bool", [(M, 0), (F | R, 0)], 0)):
        _, (eq, ec, eg) = arrays(rx, [sp])
        b = s.engine.prepare(first[0], first[1], 10, k1=s.similarity.k1)
        try:
            b.run()
            with pytest.raises(engine.EngineError) as e:
                s.engine.rescore_batch(b, eq, ec, 10)
            assert e.value.code == engine.RG_EINVAL
            got = b.fetch()
        finally:
            b.close()
        with pytest.raises(engine.EngineError) as e:
            s.engine.rescore_hits(eq, ec, np.array(got[0]), got[1], got[2], 10)
        assert e.value.code == engine.RG_EINVAL


# ---- through the public search API ---------------------------------------------------------------------------------
def test_gpu_index_searcher_rescores_with_groups_and_ranges():
    _, ix, rx, segs, points = fixture()
    fields = {}
    for name, fid in (("f0", 0), ("f1", 1)):
        fields[name] = [(leaf[fid][1], leaf[fid][2]) if fid in leaf else None for leaf in points]
    s = search.GpuIndexSearcher(search.IndexReader(segs, points=fields), device=0)
    try:
        T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
        B = search.BooleanQuery.build
        G = lambda *ts: B([], [T(t) for t in ts], [], [])
        rng0 = search.PointRangeQuery.new("f0", po.long_pack(1275), po.long_pack(200000))
        firsts = [B([], [T(0), T(6), T(3)], [], []), B([], [T(4), T(7), T(1)], [], []),
                  B([], [T(2), T(0), T(9)], [], []), B([], [T(6), T(3)], [], [])]
        rescoring = [B([G(0, 1), G(2, 3)], [], [], []), B([T(4)], [G(5, 7)], [rng0], []),
                     B([T(0)], [], [], [G(2, 3)]), B([G(0, 6)], [], [], [rng0])]
        req = search.RescoreRequest(None, 0.5, 2.0, search.RescoreMode.Total, 60)
        got = s.search_batch(firsts, 200, rescore=(rescoring, req))
        # the same through the oracle: first pass, then the rescoring queries with their own arrays
        (fq, fc, fg), _ = arrays(ix, [("bool", [(S, 0), (S, 6), (S, 3)], 0), ("bool", [(S, 4), (S, 7), (S, 1)], 0),
                                      ("bool", [(S, 2), (S, 0), (S, 9)], 0), ("bool", [(S, 6), (S, 3)], 0)])
        hits, counts, total = ix.search_batch(fq, fc, fg, 200)
        (oq, oc, og), _ = arrays(rx, [("bool", [(M, [(0,), (1,)], 0), (M, [(2,), (3,)], 0)], 0),
                                      ("bool", [(M, 4), (S, [(5,), (7,)], 0), (F | R, 0)], 0),
                                      ("bool", [(M, 0), (N, [(2,), (3,)], 0)], 0),
                                      ("bool", [(M, [(0,), (6,)], 0), (N | R, 0)], 0)])
        want = rx.rescore(oq, oc, og, hits, counts, total, 60, 0.5, 2.0, engine.RESCORE_TOTAL, ranges=ranges()[:1])
        same(got, (want, counts, total), "searcher")
    finally:
        s.engine.close()
