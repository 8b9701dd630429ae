"""QueryRescorer on the device (rg_batch_rescore / rg_rescore_hits) against the oracle's rescorer (orc_rescore,
tests/cpp/orc_rescore.cpp), bit for bit: docids, f32 score bits, order, counts and total_hits.  Every reference row is
also checked against the independent Python model of tests/rescore_model.py."""
import numpy as np
import pytest

import helpers
import oracle_binding as ob
import rescore_model as rm
import rescore_oracle as ro
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

# term ids of the fixture: dense, mid, tail-only, singleton, absent in leaf 1, absent everywhere
DFS0 = [60000, 20000, 9000, 3000, 700, 300, 129, 100, 1, 0, 5000, 4000, 2000, 1500, 1200, 900, 800, 650, 500, 450,
        400, 350, 250, 200, 150, 140, 130, 120, 110, 90, 80, 70]
DFS1 = [40000, 15000, 6000, 2000, 500, 0, 128, 77, 1, 0, 3000, 2500, 1800, 1400, 1000, 800, 600, 500, 400, 350,
        300, 250, 200, 180, 160, 150, 140, 130, 120, 100, 90, 60]
N_TERMS = len(DFS0)


def _fixture(doc_version, use_ef):
    rng = np.random.default_rng(7 + doc_version + 2 * use_ef)
    s0, _ = helpers.build_segment(rng, 200001, DFS0, doc_version=doc_version, use_ef=use_ef)
    s1, _ = helpers.build_segment(rng, 120007, DFS1, doc_version=doc_version, live_fraction=0.9, use_ef=use_ef)
    return [s0, s1]


_CACHE = {}


def fixture(doc_version=1, use_ef=False):
    key = (doc_version, use_ef)
    if key not in _CACHE:
        segs = _fixture(doc_version, use_ef)
        s = search.GpuIndexSearcher(search.IndexReader(segs), device=0)
        ix = helpers.oracle_index(segs)
        _CACHE[key] = (segs, s, rm.Model(ix, segs, s._cache, s.similarity.k1), ro.RescoreIndex(segs))
    return _CACHE[key][:3]


def want_rows(spec, n, hits, counts, total, window, qw=1.0, rw=1.0, mode=rm.TOTAL, doc_version=1, use_ef=False):
    """orc_rescore's rows for `spec` rescoring each of the n rows; the Python model must give the same bits."""
    segs, s, model, oracle = _CACHE[(doc_version, use_ef)]
    oq, oc = ob.make_queries([spec] * n)
    want = oracle.rescore(oq, oc, hits, counts, total, window, qw, rw, mode)
    rq, rc = s.compile_batch(helpers.to_queries([spec] * n))
    other = rm.rescore(model, rq, rc, hits, counts, total, window, qw, rw, mode)
    assert np.array_equal(want.view(np.uint64), other.view(np.uint64)), "orc_rescore and the model disagree"
    return want


def first_pass_specs(n):
    rng = np.random.default_rng(11)
    return [("bool", [(ob.SHOULD, t) for t in rng.choice(N_TERMS, 4, replace=False)], 0) for _ in range(n)]


def T(t, boost=1.0):
    return ("term", t, boost)


def B(clauses, msm=0):
    return ("bool", clauses, msm)


S, M, N, Fi = ob.SHOULD, ob.MUST, ob.MUST_NOT, ob.FILTER
SHAPES = {
    "term": T(2),
    "term_singleton": T(8),
    "term_absent_everywhere": T(9),
    "term_absent_in_leaf1": T(5),
    "should1_with_not": B([(S, 1), (N, 3)]),
    "should2": B([(S, 0), (S, 6)]),
    "should5": B([(S, t) for t in (1, 3, 6, 7, 8)]),
    "should9": B([(S, t) for t in range(9)]),
    "conj_unequal_df": B([(M, 0), (M, 1), (M, 2)]),
    "conj_equal_df": B([(M, 4), (M, 17), (M, 0)]),
    "conj_missing_in_leaf1": B([(M, 0), (M, 5)]),
    "filter": B([(M, 0), (Fi, 1)]),
    "lone_filter": B([(Fi, 2)]),
    "must_not": B([(M, 0), (N, 1), (N, 2)]),
    "should_not": B([(S, 0), (S, 3), (N, 1)]),
    "only_must_not": B([(N, 1), (N, 4)]),
    "msm3": B([(S, t) for t in (0, 1, 2, 3, 4)], 3),
    "msm3_few_in_leaf": B([(S, t) for t in (5, 9, 2, 8)], 3),
    "msm2_wide32": B([(S, t) for t in range(32)], 2),
    "dismax": ("dismax", [(0,), (1,), (3, 2.0)], 0.3),
    "dismax_one_present": ("dismax", [(9,), (2,)], 0.5),
    "reqopt": B([(M, 1), (S, 0), (S, 2), (S, 8)]),
    "reqopt_not": B([(M, 0), (S, 1), (N, 3)]),
    "boosted": B([(S, 0, 2.5), (S, 1, 0.5)]),
}


def run_both(name, spec, k=100, window=50, qw=1.0, rw=1.0, mode=rm.TOTAL, doc_version=1, use_ef=False,
             coll=engine.MODE_SEARCH, n=24):
    segs, s, model = fixture(doc_version, use_ef)
    fq = helpers.to_queries(first_pass_specs(n))
    q, c = s.compile_batch(fq)
    rq, rc = s.compile_batch(helpers.to_queries([spec] * n))
    b = s.engine.prepare(q, c, k, k1=s.similarity.k1, mode=coll)
    try:
        b.run()
        first = b.fetch()
        b.run()
        s.engine.rescore_batch(b, rq, rc, window, qw, rw, mode, k1=s.similarity.k1)
        got = b.fetch()
    finally:
        b.close()
    want = want_rows(spec, n, first[0], first[1], first[2], window, qw, rw, mode, doc_version, use_ef)
    helpers.assert_same_topdocs(got, (want, first[1], first[2]), name)
    return first, got


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shapes(name):
    run_both(name, SHAPES[name])


@pytest.mark.parametrize("mode", [rm.AVG, rm.MAX, rm.MIN, rm.TOTAL, rm.MULTIPLY])
@pytest.mark.parametrize("qw,rw", [(1.0, 1.0), (0.0, 1.0), (-1.0, 0.5), (0.5, -1.0), (1.0, 0.0)])
def test_modes_and_weights(mode, qw, rw):
    run_both("mode", SHAPES["reqopt"], qw=qw, rw=rw, mode=mode)


@pytest.mark.parametrize("window", [0, 1, 37, 100, 5000])
def test_windows(window):
    run_both("window", SHAPES["should5"], window=window)


@pytest.mark.parametrize("coll", [engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL])
@pytest.mark.parametrize("doc_version,use_ef", [(0, False), (1, False), (1, True)])
def test_index_shapes(coll, doc_version, use_ef):
    for name in ("conj_unequal_df", "should5", "must_not", "term_singleton"):
        run_both(name, SHAPES[name], doc_version=doc_version, use_ef=use_ef, coll=coll)


def test_reqopt_running_mean_at_k1000():
    # a window of 1000 passes ReqOptScorer's 100-score threshold in a leaf, and the skip branch is taken there
    _, s, model = fixture()
    model.reqopt_skips = 0
    run_both("reqopt1000", B([(M, 0), (S, 1), (S, 2)]), k=1000, window=1000, n=8)
    assert model.reqopt_skips > 0


@pytest.mark.parametrize("doc_version,use_ef", [(0, False), (1, False), (1, True)])
def test_block_edge_targets(doc_version, use_ef):
    """Targets built on purpose: the first and last docid of full blocks, the docs around a block boundary, vint tail
    docs, a singleton, docids between postings, in both leaves (leaf 1 with deleted docs)."""
    segs, s, model = fixture(doc_version, use_ef)
    ix = model.ix
    docs = set()
    for si, seg in enumerate(segs):
        base = int(model.bases[si])
        for t in (1, 3, 6, 7, 8):
            if t >= len(seg.terms) or int(seg.terms["doc_freq"][t]) == 0:
                continue
            p = ix.postings(si, t, int(seg.terms["doc_freq"][t]))[0].astype(np.int64)
            full = (len(p) // 128) * 128
            for i in [0, 127, 128, 255, 256, full - 1, full, len(p) - 1]:
                if 0 <= i < len(p):
                    docs.add(base + int(p[i]))
                    if int(p[i]) + 1 < seg.max_doc:
                        docs.add(base + int(p[i]) + 1)  # a docid right after a posting, usually not one
    docs = sorted(docs)[:1024]
    rng = np.random.default_rng(doc_version + 2 * use_ef)
    rng.shuffle(docs)
    spec = B([(S, 1), (S, 3), (S, 6), (S, 7), (S, 8)])
    hits = np.zeros((1, 1024), engine.HIT_DTYPE)
    hits[0]["doc"][:len(docs)] = docs
    hits[0]["score"][:len(docs)] = rng.random(len(docs)).astype(np.float32)
    counts, total = np.array([len(docs)], np.uint32), np.array([len(docs)], np.uint64)
    rq, rc = s.compile_batch(helpers.to_queries([spec]))
    got = s.engine.rescore_hits(rq, rc, hits, counts, total, 1024, 1.0, 1.0, rm.TOTAL, k1=s.similarity.k1)
    want = want_rows(spec, 1, hits, counts, total, 1024, 1.0, 1.0, rm.TOTAL, doc_version, use_ef)
    helpers.assert_same_topdocs((got, counts, total), (want, counts, total), "block edges")


def test_rows_with_fewer_hits_and_no_hits():
    # first-pass terms that are rare: rows with count < k, and a query with no hits (total_hits 0, untouched)
    segs, s, model = fixture()
    specs = [T(8), T(9), B([(S, 7), (S, 8)]), T(9)]
    q, c = s.compile_batch(helpers.to_queries(specs))
    rq, rc = s.compile_batch(helpers.to_queries([SHAPES["should5"]] * len(specs)))
    b = s.engine.prepare(q, c, 200, k1=s.similarity.k1)
    try:
        b.run()
        first = b.fetch()
        b.run()
        s.engine.rescore_batch(b, rq, rc, 150, 0.5, 2.0, rm.AVG, k1=s.similarity.k1)
        got = b.fetch()
    finally:
        b.close()
    assert first[2][1] == 0 and first[1][2] < 200
    want = want_rows(SHAPES["should5"], len(specs), first[0], first[1], first[2], 150, 0.5, 2.0, rm.AVG)
    helpers.assert_same_topdocs(got, (want, first[1], first[2]), "short rows")
    assert np.array_equal(got[0][1].view(np.uint64), first[0][1].view(np.uint64))


def test_zero_ties():
    # query_weight -0.0, rescore_weight 0: unmatched hits score -0.0, matched ones -0.0 + 0.0 = +0.0; they all
    # tie, and the docid decides
    _, got = run_both("zeros", SHAPES["should2"], qw=-0.0, rw=0.0, mode=rm.TOTAL, window=100)
    row = got[0][0]
    assert np.all(row["score"] == 0.0)
    signs = row["score"].view(np.uint32) >> 31
    assert 0 < signs.sum() < len(signs)
    assert np.all(np.diff(row["doc"]) > 0)


def test_rescore_hits_on_host_rows_with_deleted_docs():
    segs, s, model = fixture()
    live1 = segs[1].live_docs
    deleted = [d for d in range(2000) if not (int(live1[d >> 6]) >> (d & 63)) & 1][:5]
    base1 = segs[0].max_doc
    # a row from anywhere: deleted docs of leaf 1, docs of leaf 0, unsorted, duplicates of nothing
    docs = np.array([base1 + d for d in deleted] + [5, 17, 99999, 3, base1 + 7], np.int32)
    hits = np.zeros((1, 16), engine.HIT_DTYPE)
    hits[0]["doc"][:len(docs)] = docs
    hits[0]["score"][:len(docs)] = np.linspace(3, 1, len(docs)).astype(np.float32)
    counts, total = np.array([len(docs)], np.uint32), np.array([1000], np.uint64)
    rq, rc = s.compile_batch(helpers.to_queries([SHAPES["should5"]]))
    got = s.engine.rescore_hits(rq, rc, hits, counts, total, 8, 1.0, 1.0, rm.TOTAL, k1=s.similarity.k1)
    want = want_rows(SHAPES["should5"], 1, hits, counts, total, 8, 1.0, 1.0, rm.TOTAL)
    helpers.assert_same_topdocs((got, counts, total), (want, counts, total), "host rows")


def test_rescore_hits_on_oracle_rows_and_python_mirror():
    segs, s, model = fixture()
    specs = first_pass_specs(6)
    ix = helpers.oracle_index(segs)
    oq, oc = ob.make_queries(specs)
    hits, counts, total = ix.search_batch(oq, oc, 50)
    rspec = SHAPES["reqopt"]
    rq, rc = s.compile_batch(helpers.to_queries([rspec] * 6))
    got = s.engine.rescore_hits(rq, rc, hits.astype(engine.HIT_DTYPE), counts, total, 30, 1.0, 2.0, rm.MAX,
                                k1=s.similarity.k1)
    want = want_rows(rspec, 6, hits, counts, total, 30, 1.0, 2.0, rm.MAX)
    helpers.assert_same_topdocs((got, counts, total), (want, counts, total), "oracle rows")
    # QueryRescorer().rescore(searcher, req, top_docs) == the batch path
    req = search.RescoreRequest(helpers.to_queries([rspec])[0], 1.0, 2.0, search.RescoreMode.Max, 30)
    bh, bc, bt = s.search_batch(helpers.to_queries(specs), 50, rescore=(helpers.to_queries([rspec] * 6), req))
    for i, fq in enumerate(helpers.to_queries(specs)):
        coll = search.TopDocsCollector.new(50)
        s.search(fq, coll)
        td = coll.top_docs()
        search.QueryRescorer().rescore(s, req, td)
        assert [d.doc for d in td.score_docs()] == list(bh[i][:bc[i]]["doc"])
        assert np.array_equal(np.array([d.score for d in td.score_docs()], np.float32).view(np.uint32),
                              bh[i][:bc[i]]["score"].view(np.uint32))


def test_call_sequences():
    segs, s, model = fixture()
    k1 = s.similarity.k1
    qa, ca = s.compile_batch(helpers.to_queries(first_pass_specs(8)))
    qb, cb = s.compile_batch(helpers.to_queries(first_pass_specs(8)[::-1]))
    rq, rc = s.compile_batch(helpers.to_queries([SHAPES["conj_unequal_df"]] * 8))
    ref_b = s.engine.search_batch(qb, cb, 40, k1=k1)
    ref_a = s.engine.search_batch(qa, ca, 40, k1=k1)
    # run(i); rescore(i); prepare(i+1); run(i+1); fetch(i): batch i+1 unaffected
    bi = s.engine.prepare(qa, ca, 40, k1=k1)
    bi.run()
    s.engine.rescore_batch(bi, rq, rc, 30, 1.0, 1.0, rm.TOTAL, k1=k1)
    bj = s.engine.prepare(qb, cb, 40, k1=k1)
    bj.run()
    got_i = bi.fetch()
    got_j = bj.fetch()
    want = want_rows(SHAPES["conj_unequal_df"], 8, ref_a[0], ref_a[1], ref_a[2], 30, 1.0, 1.0, rm.TOTAL)
    helpers.assert_same_topdocs(got_i, (want, ref_a[1], ref_a[2]), "rescored batch")
    helpers.assert_same_topdocs(got_j, ref_b, "next batch")
    # rescoring twice composes
    bi.run()
    s.engine.rescore_batch(bi, rq, rc, 30, 1.0, 1.0, rm.TOTAL, k1=k1)
    s.engine.rescore_batch(bi, rq, rc, 20, 0.5, 1.0, rm.AVG, k1=k1)
    twice = bi.fetch()
    want2 = want_rows(SHAPES["conj_unequal_df"], 8, want, ref_a[1], ref_a[2], 20, 0.5, 1.0, rm.AVG)
    helpers.assert_same_topdocs(twice, (want2, ref_a[1], ref_a[2]), "twice")
    assert s.engine.last_kernel_ms("rescore") > 0
    # argument errors
    with pytest.raises(engine.EngineError) as ei:
        s.engine.rescore_batch(bj, rq, rc, 30, 1.0, 1.0, 7, k1=k1)
    assert ei.value.code == engine.RG_EINVAL
    bn = s.engine.prepare(qa, ca, 40, k1=k1)
    with pytest.raises(engine.EngineError) as ei:
        s.engine.rescore_batch(bn, rq, rc, 30, 1.0, 1.0, rm.TOTAL, k1=k1)
    assert ei.value.code == engine.RG_EINVAL
    with pytest.raises(engine.EngineError) as ei:
        s.engine.rescore_batch(bj, rq[:3], rc, 30, 1.0, 1.0, rm.TOTAL, k1=k1)
    assert ei.value.code == engine.RG_EINVAL
    with pytest.raises(engine.EngineError) as ei:
        s.engine.rescore_hits(rq[:1], rc, np.array([[(10 ** 9, 1.0)]], engine.HIT_DTYPE), [1], [1], 5, k1=k1)
    assert ei.value.code == engine.RG_EINVAL
    # DisiPriorityQueue shapes are refused and leave the rows as the first pass made them
    for bad in (B([(S, t) for t in range(10)]), ("dismax", [(t,) for t in range(10)], 0.1),
                B([(S, 0), (S, 1), (S, 2), (N, 3)], 2)):
        wq, wc = s.compile_batch(helpers.to_queries([bad] * 8))
        bj.run()
        with pytest.raises(engine.Unsupported):
            s.engine.rescore_batch(bj, wq, wc, 30, 1.0, 1.0, rm.TOTAL, k1=k1)
        helpers.assert_same_topdocs(bj.fetch(), ref_b, "refused")
    bi.close()
    bj.close()
    bn.close()
    # a stale batch (a norm cache changed after prepare)
    bs = s.engine.prepare(qa, ca, 40, k1=k1)
    bs.run()
    s.engine.set_norm_cache(0, s._cache)
    with pytest.raises(engine.EngineError) as ei:
        s.engine.rescore_batch(bs, rq, rc, 30, 1.0, 1.0, rm.TOTAL, k1=k1)
    assert ei.value.code == engine.RG_EINVAL
    bs.close()
