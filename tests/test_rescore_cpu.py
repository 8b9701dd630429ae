"""The rescoring model of tests/rescore_model.py on the CPU: its scorer trees, iterated with next() like a first
pass, give the oracle's matches and scores for every shape rescoring accepts; its ScoreDocHit sort, its window and
tail handling, and the advance() quirks the device kernel reproduces."""
import numpy as np
import pytest

import helpers
import oracle_binding as ob
import rescore_model as rm
import rescore_oracle as ro
from rucene_b200 import engine

S, M, N, Fi = ob.SHOULD, ob.MUST, ob.MUST_NOT, ob.FILTER
DFS0 = [3000, 1200, 400, 129, 1, 0, 700, 250]
DFS1 = [2000, 800, 0, 128, 1, 77, 500, 300]


@pytest.fixture(scope="module")
def index():
    rng = np.random.default_rng(3)
    s0, _ = helpers.build_segment(rng, 10001, DFS0)
    s1, _ = helpers.build_segment(rng, 6007, DFS1, live_fraction=0.8)
    ix = helpers.oracle_index([s0, s1])
    cache = ix.term_weight(0)[3]
    return [s0, s1], ix, rm.Model(ix, [s0, s1], cache, 1.2)


def engine_format(ix, specs):
    """ob.make_queries specs -> engine query / clause arrays with the oracle's weights (idf * boost)."""
    q, c = ob.make_queries(specs)
    eq = np.zeros(len(q), engine.QUERY_DTYPE)
    eq["clause_begin"], eq["n_clauses"], eq["min_should_match"] = q["clause_begin"], q["n_clauses"], q["min_should_match"]
    eq["flags"] = q["is_boolean"]
    ec = np.zeros(len(c), engine.CLAUSE_DTYPE)
    ec["occur"], ec["term_id"] = c["occur"], c["term_id"]
    ec["weight"] = [ix.term_weight(int(t), float(b))[0] for t, b in zip(c["term_id"], c["boost"])]
    return eq, ec


SHAPES = [
    ("term", 1), ("term", 4), ("term", 5),
    ("bool", [(S, 0), (S, 2)], 0), ("bool", [(S, t) for t in range(8)], 0), ("bool", [(S, 0), (N, 1)], 0),
    ("bool", [(M, 0), (M, 1), (M, 6)], 0), ("bool", [(M, 3), (M, 2)], 0), ("bool", [(M, 0), (Fi, 1)], 0),
    ("bool", [(Fi, 2)], 0), ("bool", [(M, 0), (N, 1), (N, 7)], 0), ("bool", [(N, 1), (N, 3)], 0),
    ("bool", [(S, 0), (S, 1), (S, 6), (S, 7)], 3), ("dismax", [(0,), (1,), (6, 2.0)], 0.25),
    ("bool", [(M, 1), (S, 0), (S, 7)], 0), ("bool", [(M, 0), (S, 1), (N, 6)], 0),
]


def model_first_pass(model, q, clauses):
    """doc -> score of every live match, iterating the model's scorer tree with next()."""
    out = {}
    for si, seg in enumerate(model.segs):
        sc = model.create_scorer(si, q, clauses)
        if sc is None:
            continue
        d = sc.next()
        while d != rm.NO_MORE:
            live = seg.live_docs is None or (int(seg.live_docs[d >> 6]) >> (d & 63)) & 1
            if live:
                out[d + int(model.bases[si])] = sc.score()
            d = sc.next()
    return out


@pytest.mark.parametrize("i", range(len(SHAPES)))
def test_model_scorers_match_the_oracle(index, i):
    segs, ix, model = index
    spec = SHAPES[i]
    q, c = ob.make_queries([spec])
    hits, counts, total = ix.search_batch(q, c, 1024)
    want = {int(h["doc"]): h["score"] for h in hits[0][:counts[0]]}
    eq, ec = engine_format(ix, [spec])
    got = model_first_pass(model, eq[0], ec)
    assert int(total[0]) == len(got)
    assert set(want) <= set(got) and len(want) == min(len(got), 1024)
    for d in want:
        assert np.float32(got[d]).view(np.uint32) == np.float32(want[d]).view(np.uint32), (spec, d)


def test_sort_order_with_signed_zeros():
    hits = [(7, np.float32(-0.0)), (3, np.float32(0.0)), (5, np.float32(1.0)), (1, np.float32(-0.0)),
            (9, np.float32(1.0)), (2, np.float32(-1.0))]
    assert [d for d, _ in rm.sort_hits(hits)] == [5, 9, 1, 3, 7, 2]


def _row(docs, scores, k):
    h = np.zeros((1, k), engine.HIT_DTYPE)
    h[0]["doc"][:len(docs)] = docs
    h[0]["score"][:len(docs)] = scores
    return h


def test_window_tail_and_empty_rows(index):
    segs, ix, model = index
    q, c = engine_format(ix, [("term", 0)])
    docs = np.array([50, 40, 30, 20], np.int32)
    sc = np.array([4, 3, 2, 1], np.float32)
    h = _row(docs, sc, 6)
    # window 0: nothing is rescored, every hit is scaled by query_weight in place
    out = rm.rescore(model, q, c, h, [4], [9], 0, 0.5, 1.0, rm.TOTAL)
    assert list(out[0]["doc"][:4]) == list(docs) and list(out[0]["score"][:4]) == [2, 1.5, 1, 0.5]
    # total_hits 0: untouched, tail included
    out = rm.rescore(model, q, c, h, [4], [0], 2, 0.5, 1.0, rm.TOTAL)
    assert np.array_equal(out, h)
    # window 2: the tail keeps its place and is scaled, even when it then outscores the window
    out = rm.rescore(model, q, c, h, [4], [9], 2, -1.0, 0.0, rm.TOTAL)
    assert list(out[0]["score"][2:4]) == [-2, -1]


def test_min_should_match_is_ignored_by_advance(index):
    segs, ix, model = index
    p1 = ix.postings(0, 1, 10000)[0]
    others = set(ix.postings(0, 0, 10000)[0]) | set(ix.postings(0, 6, 10000)[0]) | set(ix.postings(0, 7, 10000)[0])
    lone = [int(d) for d in p1 if int(d) not in others][:3]
    assert lone
    q, c = engine_format(ix, [("bool", [(S, 0), (S, 1), (S, 6), (S, 7)], 3)])
    h = _row(np.array(lone, np.int32), np.ones(len(lone), np.float32), 4)
    out = rm.rescore(model, q, c, h, [len(lone)], [5], 4, 0.0, 1.0, rm.TOTAL)
    term1 = model.term(0, c[1])
    for d, s in sorted(zip(out[0]["doc"][:len(lone)], out[0]["score"][:len(lone)])):
        term1.advance(int(d))
        assert term1.doc == d and s == term1.score()


def test_must_not_excludes_and_req_opt_mean_skips(index):
    segs, ix, model = index
    # MUST 0, MUST_NOT 1: window docs of term 0 that term 1 also has do not match (score * query_weight only)
    q, c = engine_format(ix, [("bool", [(M, 0), (N, 1)], 0)])
    p0 = ix.postings(0, 0, 10000)[0]
    p1 = set(int(d) for d in ix.postings(0, 1, 10000)[0])
    both = [int(d) for d in p0 if int(d) in p1][:2]
    only = [int(d) for d in p0 if int(d) not in p1][:2]
    h = _row(np.array(both + only, np.int32), np.full(4, 10.0, np.float32), 4)
    out = rm.rescore(model, q, c, h, [4], [4], 4, 1.0, 1.0, rm.TOTAL)
    res = {int(d): float(s) for d, s in zip(out[0]["doc"], out[0]["score"])}
    assert all(res[d] == 10.0 for d in both) and all(res[d] > 10.0 for d in only)
    # ReqOptScorer: past 100 scored docs, a doc whose required score is below half the mean skips the optional side
    q, c = engine_format(ix, [("bool", [(M, 0), (S, 6)], 0)])
    sc = rm.ReqOpt(model.term(0, c[0]), rm.Disj([model.term(0, c[1])]))
    t6 = set(int(d) for d in ix.postings(0, 6, 10000)[0])
    skipped = 0
    for d in p0[:1500]:
        sc.advance(int(d))
        mean = sc.sum / np.float32(sc.num) if sc.num else 0
        req = model.term(0, c[0])
        req.advance(int(d))
        s = sc.score()
        if sc.num > 100 and int(d) in t6 and s == req.score() and 2 * req.score() < mean:
            skipped += 1
    assert skipped > 0


# every shape rescoring accepts, plus the one it refuses for its next() walk (min_should_match > 1 beside MUST_NOT)
RESCORE_SHAPES = SHAPES + [
    ("bool", [(S, 0), (S, 1), (S, 2), (S, 3), (S, 4), (S, 6), (S, 7)], 4), ("dismax", [(5,), (1,)], 0.5),
    ("bool", [(S, 0), (S, 1), (S, 6), (N, 7)], 2), ("bool", [(M, 0), (M, 5)], 0),
]


@pytest.fixture(scope="module")
def first_rows(index):
    segs, ix, model = index
    rng = np.random.default_rng(9)
    specs = [("bool", [(S, int(t)) for t in rng.choice(8, 3, replace=False)], 0) for _ in range(6)]
    specs += [("term", 4), ("term", 5)]  # two hits / no hits at all
    q, c = ob.make_queries(specs)
    return ix.search_batch(q, c, 400)


@pytest.mark.parametrize("i", range(len(RESCORE_SHAPES)))
def test_orc_rescore_matches_the_model(index, first_rows, i):
    """The oracle's rescorer (orc_rescore, C++) and the Python model agree bit for bit, over windows below, at and
    above the row length, every mode and signed weights."""
    segs, ix, model = index
    oracle = ro.RescoreIndex(segs)
    hits, counts, total = first_rows
    spec = RESCORE_SHAPES[i]
    n = len(counts)
    oq, oc = ob.make_queries([spec] * n)
    eq, ec = engine_format(ix, [spec] * n)
    for window, qw, rw, mode in [(400, 1.0, 1.0, rm.TOTAL), (150, 0.5, 2.0, rm.AVG), (1, -1.0, 1.0, rm.MAX),
                                 (0, 2.0, 1.0, rm.MIN), (10 ** 6, -0.0, 0.0, rm.MULTIPLY), (333, 1.0, -1.0, rm.MIN)]:
        got = oracle.rescore(oq, oc, hits, counts, total, window, qw, rw, mode)
        want = rm.rescore(model, eq, ec, hits, counts, total, window, qw, rw, mode)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (spec, window, mode)


def test_orc_rescore_quirks(index):
    """advance() ignores min_should_match; MUST_NOT excludes; ReqOptScorer's mean skips the optional side; live docs
    are not consulted — on the oracle's rescorer, checked against per-term postings."""
    segs, ix, model = index
    oracle = ro.RescoreIndex(segs)
    p = {t: set(int(d) for d in ix.postings(0, t, 10000)[0]) for t in (0, 1, 6, 7)}
    lone = sorted(p[1] - p[0] - p[6] - p[7])[:3]
    q, c = ob.make_queries([("bool", [(S, 0), (S, 1), (S, 6), (S, 7)], 3)])
    out = oracle.rescore(q, c, _row(np.array(lone, np.int32), np.zeros(3, np.float32), 4), [3], [3], 4, 1.0, 1.0,
                         rm.TOTAL)
    assert np.all(out[0]["score"][:3] > 0)  # each matched through its one SHOULD term
    both = sorted(p[0] & p[1])[:2]
    only = sorted(p[0] - p[1])[:2]
    q, c = ob.make_queries([("bool", [(M, 0), (N, 1)], 0)])
    out = oracle.rescore(q, c, _row(np.array(both + only, np.int32), np.full(4, 10.0, np.float32), 4), [4], [4], 4)
    res = {int(d): float(s) for d, s in zip(out[0]["doc"], out[0]["score"])}
    assert all(res[d] == 10.0 for d in both) and all(res[d] > 10.0 for d in only)
    # a deleted doc of leaf 1 that has term 0 is scored all the same
    live = segs[1].live_docs
    p1 = ix.postings(1, 0, 10000)[0]
    dead = [int(d) for d in p1 if not (int(live[int(d) >> 6]) >> (int(d) & 63)) & 1][:1]
    assert dead
    q, c = ob.make_queries([("term", 0)])
    out = oracle.rescore(q, c, _row(np.array([segs[0].max_doc + dead[0]], np.int32), np.zeros(1, np.float32), 1),
                         [1], [1], 1)
    assert out[0]["score"][0] > 0
    # ReqOptScorer over a long window of term 0's docs: the model sees skips, and the oracle agrees with it
    docs = np.array(sorted(p[0])[:1024], np.int32)
    h = _row(docs, np.zeros(len(docs), np.float32), 1024)
    eq, ec = engine_format(ix, [("bool", [(M, 0), (S, 6)], 0)])
    oq, oc = ob.make_queries([("bool", [(M, 0), (S, 6)], 0)])
    model.reqopt_skips = 0
    want = rm.rescore(model, eq, ec, h, [len(docs)], [len(docs)], 1024, 1.0, 1.0, rm.TOTAL)
    assert model.reqopt_skips > 0
    got = oracle.rescore(oq, oc, h, [len(docs)], [len(docs)], 1024, 1.0, 1.0, rm.TOTAL)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
