"""PointRangeQuery clauses on the device (rg_points_upload, rg_search_batch_ranges, k_eval_and_ranges) against the
oracle's BooleanQuery with PointRangeWeight (tests/cpp/orc_points.cpp), bit for bit: docids, f32 score bits, tie
order, counts and total_hits, in both collector modes."""
import numpy as np
import pytest

import oracle_binding as ob
import points_fixtures as pf
import points_oracle as po
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

R = po.RANGE
_CACHE = {}


def fixture(doc_version=1, flags=0):
    key = (doc_version, flags)
    if key not in _CACHE:
        segs, points = pf.build(11 + doc_version, sizes=(70001, 40007, 31001), doc_version=doc_version)
        s = search.GpuIndexSearcher(search.IndexReader(segs), device=0)
        s.engine.set_flags(flags)
        ix = po.PointsIndex(segs)
        for si, leaf in enumerate(points):
            for f, (nb, d, p, _) in leaf.items():
                ix.add_points(si, f, nb, d, p)
                s.engine.upload_points(si, f, nb, d, p)
        _CACHE[key] = (segs, points, s, ix)
    return _CACHE[key]


def ranges_of(points):
    ts = np.sort(points[0][pf.TS][3])
    pct = lambda a: int(ts[min(len(ts) - 1, int(len(ts) * a))])
    out = [po.make_range(pf.TS, 8, po.long_pack(pct(a)), po.long_pack(pct(b))) for a, b in
           [(0.5, 0.51), (0.1, 0.2), (0.2, 0.7), (0.0, 1.0)]]
    # bounds on both sides of 128-doc block edges (timestamps are ~10 * docid)
    out += [po.make_range(pf.TS, 8, po.long_pack(1275), po.long_pack(2565)),
            po.make_range(pf.TS, 8, po.long_pack(1285), po.long_pack(2555)),
            po.make_range(pf.TS, 8, po.long_pack(2560), po.long_pack(5120))]  # blocks 2..3: one doc without a value
    out += [po.make_range(pf.UNI, 4, po.int_pack(-(1 << 31)), po.int_pack((1 << 31) - 1)),
            po.make_range(pf.UNI, 4, po.int_pack(-(1 << 29)), po.int_pack(1 << 28)),
            po.make_range(pf.UNI, 4, po.int_pack(5), po.int_pack(4)),
            po.make_range(pf.PART, 8, po.long_pack(-(1 << 62)), po.long_pack(1 << 39))]
    return np.array(out, po.RANGE_DTYPE)


def specs(n_ranges):
    """Every accepted shape; ("bare", range) is a bare PointRangeQuery."""
    sp = [("bare", ri) for ri in range(n_ranges)]
    sp += [("bool", [(ob.FILTER | R, ri)], 0) for ri in range(n_ranges)]                    # collapses to the range
    sp += [("bool", [(ob.SHOULD | R, ri)], 0) for ri in (0, 7)]
    sp += [("bool", [(ob.MUST, t), (ob.FILTER | R, ri)], 0) for t in (0, 2, 4, 8) for ri in range(n_ranges)]
    sp += [("bool", [(ob.MUST, 1), (ob.MUST, 3), (ob.MUST | R, ri), (ob.FILTER | R, 8)], 0) for ri in (1, 2, 4)]
    sp += [("bool", [(ob.MUST | R, ri), (ob.MUST_NOT, 0)], 0) for ri in (0, 2, 7)]
    sp += [("bool", [(ob.FILTER | R, 2), (ob.MUST_NOT | R, ri)], 0) for ri in (1, 8, 10)]
    sp += [("bool", [(ob.MUST, 1), (ob.MUST_NOT | R, 2), (ob.MUST_NOT, 6)], 0)]
    sp += [("bool", [(ob.FILTER | R, ri), (ob.SHOULD, 1), (ob.SHOULD, 2)], 0) for ri in (0, 2, 3, 7)]   # ReqOpt, split
    sp += [("bool", [(ob.MUST, 0), (ob.FILTER | R, ri), (ob.SHOULD, 2), (ob.SHOULD, 5)], 0) for ri in (2, 3)]
    sp += [("bool", [(ob.MUST, 0, -0.0), (ob.FILTER | R, ri)], 0) for ri in (2, 3)]            # -0.0 term scores
    sp += [("bool", [(ob.MUST, 1, -0.0), (ob.MUST | R, 3), (ob.MUST_NOT | R, 9)], 0)]
    return sp


def to_arrays(sp):
    qs, cs = [], []
    for s in sp:
        if s[0] == "bare":
            qs.append((len(cs), 1, 0, 0))
            cs.append((ob.MUST | R, s[1], 0.0))
        else:
            qs.append((len(cs), len(s[1]), s[2], 1))
            for cl in s[1]:
                cs.append((cl[0], cl[1], cl[2] if len(cl) > 2 else (0.0 if cl[0] & R else 1.0)))
    return np.array(qs, ob.QUERY_DTYPE), np.array(cs, ob.CLAUSE_DTYPE)


def engine_queries(oq):
    q = np.zeros(len(oq), engine.QUERY_DTYPE)
    for f in ("clause_begin", "n_clauses", "min_should_match"):
        q[f] = oq[f]
    q["flags"] = np.where(oq["is_boolean"] == 1, engine.Q_BOOLEAN, 0)
    return q


def same(got, want, label):
    gh, gc, gt = got
    wh, wc, wt = want
    assert np.array_equal(gt, wt), (label, "total_hits", np.nonzero(gt != wt)[0][:5])
    assert np.array_equal(gc, wc), (label, "counts")
    for i in range(len(gc)):
        n = int(wc[i])
        assert np.array_equal(gh[i][:n]["doc"], wh[i][:n]["doc"]), (label, "docs of query", i)
        assert np.array_equal(gh[i][:n]["score"].view(np.uint32), wh[i][:n]["score"].view(np.uint32)), (label, "scores", i)


@pytest.mark.parametrize("doc_version", [0, 1])
@pytest.mark.parametrize("k", [1, 10, 100, 1000])
def test_every_shape_matches_the_oracle(doc_version, k):
    segs, points, s, ix = fixture(doc_version)
    ranges = ranges_of(points)
    oq, oc = to_arrays(specs(len(ranges)))
    eq, ec = engine_queries(oq), ix.engine_clauses(oc)
    for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
        want = ix.search_batch(oq, oc, ranges, k, parallel_mode=mode)
        got = s.engine.search_batch_ranges(eq, ec, ranges, k, k1=s.similarity.k1, mode=mode)
        same(got, want, ("v", doc_version, "k", k, "mode", mode))


@pytest.mark.parametrize("flags", [engine.CFG_EAGER_COLUMNS, engine.CFG_NO_BITMAPS])
def test_engine_configurations(flags):
    segs, points, s, ix = fixture(1, flags)
    ranges = ranges_of(points)
    oq, oc = to_arrays(specs(len(ranges)))
    eq, ec = engine_queries(oq), ix.engine_clauses(oc)
    for k in (10, 1000):
        same(s.engine.search_batch_ranges(eq, ec, ranges, k, k1=s.similarity.k1),
             ix.search_batch(oq, oc, ranges, k), ("flags", flags, k))


def test_range_led_and_term_led_and_counters():
    segs, points, s, ix = fixture(1)
    ranges = ranges_of(points)
    # term 8 has df 1 (term leads), term 0 has df 30000 vs a 1 % range (range leads), same shape
    oq, oc = to_arrays([("bool", [(ob.MUST, 8), (ob.FILTER | R, 0)], 0), ("bool", [(ob.MUST, 0), (ob.FILTER | R, 0)], 0),
                        ("bare", 2)])
    eq, ec = engine_queries(oq), ix.engine_clauses(oc)
    b = s.engine.prepare(eq, ec, 10, k1=s.similarity.k1, ranges=ranges)
    try:
        b.run()
        got = b.fetch()
        st = b.range_stats()
    finally:
        b.close()
    same(got, ix.search_batch(oq, oc, ranges, 10), "lead choice")
    # the timestamp rises with docid: most blocks lie wholly outside a narrow range, many wholly inside a wide one
    assert st["skipped"] > 0 and st["whole"] > 0 and st["scanned"] > 0, st


def test_bare_ranges_tie_order():
    """every score is +0.0: the heap layout alone decides which docs stay and in what order"""
    segs, points, s, ix = fixture(0)
    ranges = ranges_of(points)
    oq, oc = to_arrays([("bare", ri) for ri in range(len(ranges))])
    eq, ec = engine_queries(oq), ix.engine_clauses(oc)
    for k in (1, 7, 100, 1000):
        for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
            got = s.engine.search_batch_ranges(eq, ec, ranges, k, k1=s.similarity.k1, mode=mode)
            same(got, ix.search_batch(oq, oc, ranges, k, parallel_mode=mode), ("bare", k, mode))
            assert np.all(got[0][:, :1]["score"].view(np.uint32) == 0)


def test_refused_and_invalid():
    segs, points, s, ix = fixture(1)
    ranges = ranges_of(points)

    def run(sp, rr=ranges, dismax=False):
        oq, oc = to_arrays(sp)
        eq, ec = engine_queries(oq), ix.engine_clauses(oc)
        if dismax:
            eq["flags"] = engine.Q_DISMAX
        return s.engine.search_batch_ranges(eq, ec, rr, 10, k1=s.similarity.k1)

    for sp in ([("bool", [(ob.SHOULD | R, 0), (ob.SHOULD, 1)], 0)],          # range on a disjunction
               [("bool", [(ob.MUST, 1), (ob.SHOULD | R, 0)], 0)],            # SHOULD range beside a MUST
               [("bool", [(ob.SHOULD, 1), (ob.SHOULD, 2), (ob.MUST_NOT | R, 0)], 0)],  # MUST_NOT range on a disjunction
               [("bool", [(ob.MUST_NOT | R, 0)], 0)],                        # match-all route
               [("bool", [(ob.MUST, 1, 1.0), (ob.FILTER | R, 0, 2.0)], 0)]):  # a boosted range
        with pytest.raises(engine.Unsupported):
            run(sp)
    with pytest.raises(engine.Unsupported):
        run([("bool", [(ob.MUST, 1), (ob.FILTER | R, 0)], 0)], dismax=True)
    with pytest.raises(engine.Unsupported):  # ranges count toward the 9-clause limit
        run([("bool", [(ob.MUST, t) for t in range(5)] + [(ob.FILTER | R, i) for i in range(5)], 0)])
    bad = ranges.copy()
    bad[0]["bytes_per_dim"] = 4  # the timestamp field was uploaded with 8 bytes per dim
    with pytest.raises(engine.EngineError) as ei:
        run([("bool", [(ob.MUST, 1), (ob.FILTER | R, 0)], 0)], rr=bad)
    assert ei.value.code == engine.RG_EINVAL
    with pytest.raises(engine.EngineError) as ei:
        run([("bool", [(ob.FILTER | R, 99)], 0)])
    assert ei.value.code == engine.RG_EINVAL
    # the old entry points never read the flag as a range: an unknown occur
    oq, oc = to_arrays([("bool", [(ob.MUST, 1), (ob.FILTER | R, 0)], 0)])
    with pytest.raises(engine.EngineError) as ei:
        s.engine.search_batch(engine_queries(oq), ix.engine_clauses(oc), 10)
    assert ei.value.code == engine.RG_EINVAL
    # rg_points_upload arguments
    e = s.engine
    for args in ((7, 0, 8, [0], np.zeros((1, 8), np.uint8)),        # leaf not uploaded
                 (0, 9, 3, [0], np.zeros((1, 3), np.uint8)),        # bytes_per_dim
                 (0, 9, 4, [segs[0].max_doc], np.zeros((1, 4), np.uint8)),  # docid outside the leaf
                 (0, pf.TS, 8, [0], np.zeros((1, 8), np.uint8))):  # second upload of (leaf, field)
        with pytest.raises(engine.EngineError) as ei:
            e.upload_points(*args)
        assert ei.value.code == engine.RG_EINVAL


def test_reqopt_split_only_without_required_terms():
    """With 1024 postings per item a term-required ReqOpt would be cut into ~30 items; its running mean is sequential
    state, so only the items whose required side is ranges alone may be cut."""
    segs, points, _, ix = fixture(1)
    s = search.GpuIndexSearcher(search.IndexReader(segs), device=0, range_postings=1024)
    for si, leaf in enumerate(points):
        for f, (nb, d, p, _) in leaf.items():
            s.engine.upload_points(si, f, nb, d, p)
    ranges = ranges_of(points)
    sp = [("bool", [(ob.MUST, 0), (ob.FILTER | R, ri), (ob.SHOULD, 1), (ob.SHOULD, 2)], 0) for ri in (3, 7)]
    sp += [("bool", [(ob.FILTER | R, ri), (ob.SHOULD, 1), (ob.SHOULD, 2)], 0) for ri in (3, 7)]
    oq, oc = to_arrays(sp)
    eq, ec = engine_queries(oq), ix.engine_clauses(oc)
    for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
        for k in (10, 1000):
            same(s.engine.search_batch_ranges(eq, ec, ranges, k, k1=s.similarity.k1, mode=mode),
                 ix.search_batch(oq, oc, ranges, k, parallel_mode=mode), ("split", mode, k))
    b = s.engine.prepare(eq[2:], ec, 10, k1=s.similarity.k1, ranges=ranges)
    try:
        assert b.stats()["items"] > 2 * len(segs), b.stats()  # the range-only ReqOpt items were cut
    finally:
        b.close()


def test_public_surface_float_double_points():
    """search.py: FloatPoint / DoublePoint fields with -0.0, +0.0, the infinities and NaNs, queried through
    PointRangeQuery in BooleanQuerys and compared with the oracle"""
    rng = np.random.default_rng(5)
    segs, _ = pf.build(21, sizes=(40001, 31007))
    special32 = np.array([0x80000000, 0x00000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001], np.uint32)
    special64 = np.array([1 << 63, 0, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000,
                          0xFFF8000000000001], np.uint64)
    fields = {}
    for name, nb, special, ftype, pt in (("f", 4, special32, np.float32, search.FloatPoint),
                                         ("d", 8, special64, np.float64, search.DoublePoint)):
        per_leaf = []
        for seg in segs:
            docs = rng.permutation(seg.max_doc)[: seg.max_doc - 100].astype(np.int32)
            bits = rng.normal(0, 100, docs.size).astype(ftype).view(special.dtype)
            bits[: 600] = special[np.arange(600) % len(special)]
            per_leaf.append((docs, np.frombuffer(b"".join(pt.pack_bits(int(b)) for b in bits), np.uint8).reshape(-1, nb)))
        fields[name] = per_leaf
    reader = search.IndexReader(segs, points=fields)
    s = search.GpuIndexSearcher(reader, device=0)
    ix = po.PointsIndex(segs)
    for fid, name in enumerate(sorted(fields)):
        for si, (d, p) in enumerate(fields[name]):
            ix.add_points(si, fid, p.shape[1], d, p)
    T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
    F, D, B = search.FloatPoint, search.DoublePoint, search.BooleanQuery.build
    qs = [F.new_exact_query("f", -0.0), F.new_exact_query("f", 0.0), F.new_range_query("f", -0.0, 0.0),
          F.new_range_query("f", float("-inf"), float("inf")), D.new_range_query("d", 0.0, float("inf")),
          search.PointRangeQuery.new("d", D.pack_bits(0xFFF8000000000001), D.pack(-1e300)),
          search.PointRangeQuery.new("f", F.pack(float("inf")), F.pack_bits(0x7FC00000)),
          B([T(0)], [], [F.new_range_query("f", -5.0, 5.0)], [D.new_exact_query("d", float("inf"))]),
          B([], [T(1), T(2)], [D.new_range_query("d", -50.0, 80.0)], []),
          B([T(2), D.new_range_query("d", float("-inf"), -0.0)], [], [], [])]
    q, c, r = s.compile_batch_ranges(qs)
    oq = np.zeros(len(q), ob.QUERY_DTYPE)
    oq["clause_begin"], oq["n_clauses"], oq["min_should_match"] = q["clause_begin"], q["n_clauses"], q["min_should_match"]
    oq["is_boolean"] = q["flags"] & engine.Q_BOOLEAN
    oc = np.zeros(len(c), ob.CLAUSE_DTYPE)
    oc["occur"], oc["term_id"] = c["occur"], c["term_id"]
    oc["boost"] = np.where(c["occur"] & R, 0.0, 1.0)
    for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
        for k in (1, 10, 1000):
            same(s.search_batch(qs, k, mode=mode), ix.search_batch(oq, oc, r, k, parallel_mode=mode),
                 ("public", mode, k))
    col = search.TopDocsCollector.new(5)
    s.search(qs[0], col)
    assert col.top_docs().total_hits() > 0
