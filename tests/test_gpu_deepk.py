"""Deep top-k on the device (1024 < k <= 16384): the histogram theta bound in every evaluation kernel, the one-warp
heap replay and leaf-record merge, against the oracle bit for bit (docids, f32 score bits, tie order, counts,
total_hits), in both collector modes."""
import os
import subprocess
import sys

import numpy as np
import pytest

import deepk_model as dm
import helpers
import nested_fixtures as nf
import nested_oracle as no
import oracle_binding as ob
import points_oracle as po
from rucene_b200 import codec, engine, search

pytestmark = pytest.mark.gpu

KS = [1025, 2048, 4096, 16384]
MODES = [engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL]
CONFIGS = [engine.CFG_EAGER_COLUMNS | engine.CFG_MAXSCORE, engine.CFG_EAGER_COLUMNS,
           engine.CFG_NO_BITMAPS | engine.CFG_NO_LISTS, engine.CFG_MAXSCORE, 0]
_SEGS = {}


def family_leaves():
    """Two leaves (the second with deleted docs) with dense, mid and sparse terms; term 15 is dense with constant
    freqs (all-equal blocks, massive ties)."""
    if "fam" not in _SEGS:
        rng = np.random.default_rng(4242)
        dfs = [90000, 60000, 30000, 20000, 9000, 5000, 4097, 4096, 2049, 2048, 1025, 700, 129, 1, 0, 50000]
        a, _ = helpers.build_segment(rng, 120000, dfs, dense_terms=(15,))
        b, _ = helpers.build_segment(rng, 70001, [min(d, 60000) for d in dfs], doc_version=0, live_fraction=0.9)
        _SEGS["fam"] = [a, b]
    return _SEGS["fam"]


def family_specs():
    M, S, F, N = ob.MUST, ob.SHOULD, ob.FILTER, ob.MUST_NOT
    sp = [("term", t) for t in (0, 4, 6, 7, 9, 10, 13, 15)]
    sp += [("bool", [(M, 0), (M, 1)], 0), ("bool", [(M, 2), (M, 3), (M, 15)], 0),           # AND
           ("bool", [(S, 0), (S, 1), (S, 2)], 0), ("bool", [(S, 4), (S, 11), (S, 12)], 0),   # OR
           ("bool", [(M, 1), (S, 2), (S, 4)], 0), ("bool", [(M, 3), (S, 0)], 0),            # ReqOpt
           ("bool", [(S, 0), (S, 1), (S, 3), (S, 5)], 2),                                    # min_should_match
           ("dismax", [(0,), (2, 2.0), (4,)], 0.3),                                           # dismax
           ("bool", [(S, 0), (S, 2), (N, 1)], 0), ("bool", [(M, 0), (N, 3)], 0),            # MUST_NOT
           ("bool", [(M, 1), (F, 0)], 0), ("bool", [(F, 2), (S, 4)], 0),                     # FILTER
           ("bool", [(N, 5)], 0),                                                             # match-all
           ("bool", [(S, t) for t in (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11)], 0),            # >= 10 clauses (DPQ)
           ("dismax", [(t,) for t in (0, 2, 3, 5, 6, 7, 8, 9, 10, 11)], 0.1),
           ("bool", [(S, 0, -1.5), (S, 4)], 0), ("term", 2, -0.5),                           # absolute map
           ("bool", [(S, 15), (S, 0, 0.0)], 0)]
    return sp


def run_both(segs, specs, k, mode, flags=0, rp=0, ix=None):
    ix = ix or helpers.oracle_index(segs)
    q, c = ob.make_queries(specs)
    want = ix.search_batch(q, c, k, parallel_mode=mode, n_threads=4)
    s = search.GpuIndexSearcher(search.IndexReader(segs), device=0, range_postings=rp, flags=flags)
    try:
        got = s.search_batch(helpers.to_queries(specs), k, mode=mode)
    finally:
        s.engine.close()
    return got, want


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", MODES)
def test_every_family(k, mode):
    segs = family_leaves()
    got, want = run_both(segs, family_specs(), k, mode)
    helpers.assert_same_topdocs(got, want, ("k", k, "mode", mode))


@pytest.mark.parametrize("flags", CONFIGS)
@pytest.mark.parametrize("rp", [0, 2000])
def test_engine_configurations(flags, rp):
    """Every evaluation route; range_postings 2000 cuts the lists into chains of many items that inherit histograms."""
    segs = family_leaves()
    ix = helpers.oracle_index(segs)
    for k, mode in ((2048, engine.MODE_SEARCH), (4096, engine.MODE_SEARCH_PARALLEL)):
        got, want = run_both(segs, family_specs(), k, mode, flags, rp, ix)
        helpers.assert_same_topdocs(got, want, ("flags", flags, "rp", rp, "k", k))


@pytest.mark.parametrize("k", [1025, 4096, 16384])
def test_point_ranges_and_nested_groups(k):
    segs, points, _ = nf.build(31)
    s = search.GpuIndexSearcher(search.IndexReader(segs), device=0, range_postings=300)
    ix = no.NestedIndex(segs)
    try:
        for si, leaf in enumerate(points):
            for f, (nb, d, p, _) in leaf.items():
                ix.add_points(si, f, nb, d, p)
                s.engine.upload_points(si, f, nb, d, p)
        rg = np.array([po.make_range(0, 8, po.long_pack(1275), po.long_pack(200000)),
                       po.make_range(1, 4, po.int_pack(-(1 << 29)), po.int_pack(1 << 28)),
                       po.make_range(0, 8, po.long_pack(-(1 << 40)), po.long_pack(1 << 40))], po.RANGE_DTYPE)
        oq, oc, og = no.to_arrays(nf.specs([0, 1, 2]))
        eq, ec, eg = no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og)
        for mode in MODES:
            want = ix.search_batch(oq, oc, og, k, ranges=rg, parallel_mode=mode)
            got = s.engine.search_batch_nested(eq, ec, eg, k, k1=s.similarity.k1, mode=mode, ranges=rg)
            helpers.assert_same_topdocs(got, want, ("nested/ranges k", k, "mode", mode))
    finally:
        s.engine.close()


def _write(max_doc, postings, norms, live=None):
    w = codec.PostingsWriter(doc_version=1, max_doc=max_doc)
    for docs, freqs in postings:
        w.add_term(np.asarray(docs, np.int32), np.asarray(freqs, np.int32))
    return w.finish(norms=norms, live_docs=live)


def test_seeds_and_spikes():
    """4096 seed docs score H (the first docids, so they are collected first and fill the histogram); up to 4096
    spikes per query score above H, scattered over many items.  The TopDocs are the spikes, then the first seeds: one
    spike that was not emitted leaves an extra seed in them."""
    rng = np.random.default_rng(11)
    M, K, FS = 600000, 4096, 6
    d = np.arange(M)
    posts = []
    for t, n_spikes in enumerate((4096, 1500)):
        f = np.ones(M, np.int32)
        f[:K] = FS
        spikes = np.sort(rng.choice(np.arange(K, M), n_spikes, replace=False))
        f[spikes] = FS + 1 + rng.integers(0, 40, n_spikes)
        mask = (d % (2 + t) != 0) | (d < K)
        mask[spikes] = True
        posts.append((d[mask], f[mask]))
    posts.append((d[d % 11 == 0], np.ones(np.count_nonzero(d % 11 == 0), np.int32)))   # a third, sparse clause
    seg = _write(M, posts, np.full(M, 100, np.uint8))
    specs = [("term", 0), ("term", 1), ("bool", [(ob.SHOULD, 0), (ob.SHOULD, 2, 0.01)], 0)]
    ix = helpers.oracle_index([seg])
    for flags in (0, engine.CFG_NO_BITMAPS | engine.CFG_NO_LISTS, engine.CFG_EAGER_COLUMNS | engine.CFG_MAXSCORE):
        for rp in (0, 5000):
            got, want = run_both([seg], specs, K, engine.MODE_SEARCH, flags, rp, ix)
            helpers.assert_same_topdocs(got, want, ("spikes", flags, rp))


def _edge_boost(idf, cache, k1, freq, nb, rng):
    """A boost whose TermQuery score at (freq, norm byte nb) lies exactly on the lower edge of its bucket: the
    planner's map puts the top bucket at U = nextafter(nextafter(w1)), so the score's ordered value must equal
    ord(U) modulo 2^18 (numpy search over boosts, the score formula of bm25_scores_numpy)."""
    f = np.float32(freq)
    for _ in range(200):
        boost = (1.0 + rng.random(1 << 20)).astype(np.float32)
        w = (np.float32(idf) * boost).astype(np.float32)
        w1 = (w * (np.float32(k1) + np.float32(1))).astype(np.float32)
        s = ((w1 * f).astype(np.float32) / np.float32(f + cache[nb])).astype(np.float32)
        u = w1.view(np.uint32).astype(np.int64) + 2
        ok = np.nonzero((dm.to_ordered(s).astype(np.int64) - ((u | 0x80000000) - (255 << 18))) % (1 << 18) == 0)[0]
        if len(ok):
            return float(boost[ok[0]]), float(s[ok[0]])
    raise AssertionError("no boost found")


def test_theta_on_a_bucket_edge_and_ties():
    """The k-th best score equals its bucket's lower edge exactly, and thousands of docs tie at it (across the theta
    bucket and beyond k): with theta = that edge, `score > theta` must drop exactly the ties the heap drops."""
    rng = np.random.default_rng(5)
    M, k = 300000, 2048
    d = np.arange(M)
    f = np.full(M, 2, np.int32)
    posts = [(d[d % 3 != 1], f[d % 3 != 1]), (d[d % 5 == 0], f[d % 5 == 0])]
    hi = np.sort(rng.choice(M, k - 700, replace=False))

    def leaf(nb_tie, nb_hi):
        norms = np.full(M, nb_tie, np.uint8)
        norms[hi] = nb_hi                   # shorter docs: above the tie score
        return _write(M, posts, norms)
    # the norm cache depends on the average field length only: pick a norm byte near it for the ties, a shorter one
    # for the docs above them, so that the tie score sits in the bound's 8 octaves
    _w, idf, _avg, cache = helpers.oracle_index([leaf(1, 1)]).term_weight(0, 1.0)
    nb_tie = int(np.argmin(np.abs(cache[1:] - np.float32(1.2)))) + 1
    nb_hi = int(np.argmin(np.abs(cache[1:] - cache[nb_tie] / 3))) + 1
    assert cache[nb_hi] < cache[nb_tie]
    seg = leaf(nb_tie, nb_hi)
    ix = helpers.oracle_index([seg])
    boost, s_tie = _edge_boost(idf, cache, 1.2, 2, nb_tie, rng)
    w2, _i, _a, _c = ix.term_weight(0, boost)
    assert helpers.bm25_scores_numpy(w2, 1.2, np.array([2]), np.array([nb_tie]), cache)[0] == np.float32(s_tie)
    m = dm.bucket_map(dm.score_bound([np.float32(w2) * (np.float32(1.2) + np.float32(1.0))]))
    assert dm.edge(m, int(dm.key(m, np.float32(s_tie)))) == np.float32(s_tie), "the tie score is a bucket edge"
    specs = [("term", 0, boost), ("bool", [(ob.SHOULD, 0, boost), (ob.MUST_NOT, 1)], 0), ("term", 1, boost)]
    for mode in MODES:
        for flags, rp in ((0, 0), (engine.CFG_NO_BITMAPS | engine.CFG_NO_LISTS, 3000), (engine.CFG_EAGER_COLUMNS, 3000)):
            got, want = run_both([seg], specs, k, mode, flags, rp, ix)
            helpers.assert_same_topdocs(got, want, ("edge", mode, flags, rp))
            assert np.count_nonzero(want[0][0]["score"] == np.float32(s_tie)) > 600


@pytest.mark.parametrize("k", [2048, 4096])
def test_match_counts_around_k(k):
    rng = np.random.default_rng(k)
    M = 50000
    posts = []
    for df in (k - 1, k, k + 1):
        docs = np.sort(rng.choice(M, df, replace=False))
        posts.append((docs, rng.integers(1, 5, df)))
    seg = _write(M, posts, rng.integers(1, 255, M).astype(np.uint8))
    specs = [("term", 0), ("term", 1), ("term", 2), ("bool", [(ob.SHOULD, 0), (ob.SHOULD, 1)], 0),
             ("bool", [(ob.MUST, 1), (ob.FILTER, 2)], 0)]
    for mode in MODES:
        got, want = run_both([seg], specs, k, mode, rp=500)
        helpers.assert_same_topdocs(got, want, ("counts", k, mode))
        assert list(want[1][:3]) == [k - 1, k, k]


def _big_segment():
    if "big" not in _SEGS:
        _SEGS["big"] = codec.synth_segment(0x5EED00D1, 2000000, 3000, doc_version=1)
    return _SEGS["big"]


def test_pruning_works():
    """A disjunction with millions of matches at k = 2048: the candidates are a small fraction of the matches (a theta
    stuck at -inf would emit every match).  One work item per query and leaf: items of one query that run at the
    same time each emit their first k candidates before they have a theta of their own."""
    seg = _big_segment()
    ix = helpers.oracle_index([seg])
    specs = [("bool", [(ob.SHOULD, 0), (ob.SHOULD, 1), (ob.SHOULD, 2)], 0), ("bool", [(ob.MUST, 0), (ob.SHOULD, 3)], 0)]
    q, c = ob.make_queries(specs)
    for flags in (0, engine.CFG_NO_BITMAPS | engine.CFG_NO_LISTS):
        s = search.GpuIndexSearcher(search.IndexReader([seg]), device=0, flags=flags, range_postings=1 << 30)
        try:
            eq, ec = s.compile_batch(helpers.to_queries(specs))
            b = s.engine.prepare(eq, ec, 2048, k1=s.similarity.k1)
            try:
                b.run()
                got = b.fetch()
                st = b.stats()
            finally:
                b.close()
        finally:
            s.engine.close()
        want = ix.search_batch(q, c, 2048)
        helpers.assert_same_topdocs(got, want, ("pruning", flags))
        matches = int(want[2].sum())
        assert want[2][0] >= 1000000, want[2]
        assert st["candidate_slots"] * 20 < matches, (st, matches)


def test_refusals():
    segs = family_leaves()
    s = search.GpuIndexSearcher(search.IndexReader(segs), device=0)
    try:
        with pytest.raises(engine.Unsupported):
            s.search_batch(helpers.to_queries([("term", 0)]), 16385)
        # rescoring a deep batch is refused and leaves its rows as they were
        eq, ec = s.compile_batch(helpers.to_queries([("term", 0), ("bool", [(ob.SHOULD, 1), (ob.SHOULD, 2)], 0)]))
        b = s.engine.prepare(eq, ec, 2048, k1=s.similarity.k1)
        try:
            b.run()
            before = b.fetch()
            rq, rc = s.compile_batch(helpers.to_queries([("term", 3), ("term", 4)]))
            with pytest.raises(engine.Unsupported):
                s.engine.rescore_batch(b, rq, rc, 100)
            after = b.fetch()
            helpers.assert_same_topdocs(after, before, "rows after the refused rescore")
        finally:
            b.close()
    finally:
        s.engine.close()


def test_leaf_record_merge():
    """MODE_SEARCH_PARALLEL leaf records (16 + 8 k bytes each) merged by rg_merge_leaf_records at k = 4096 / 16384."""
    segs = family_leaves()
    ix = helpers.oracle_index(segs)
    specs = family_specs()
    q, c = ob.make_queries(specs)
    s = search.GpuIndexSearcher(search.IndexReader(segs), device=0, range_postings=3000)
    try:
        eq, ec = s.compile_batch(helpers.to_queries(specs))
        for k in (4096, 16384):
            b = s.engine.prepare(eq, ec, k, k1=s.similarity.k1, mode=engine.MODE_SEARCH_PARALLEL)
            try:
                b.run()
                ptr, rec_bytes = b.leaf_records()
                assert rec_bytes == 16 + 8 * k
                got = s.engine.merge_leaf_records(ptr, len(segs), len(specs), k)
            finally:
                b.close()
            helpers.assert_same_topdocs(got, ix.search_batch(q, c, k, parallel_mode=1), ("merge", k))
    finally:
        s.engine.close()


def test_two_ranks_on_one_gpu():
    """Sharded search at k = 4096: two ranks share cuda:0, leaf records over gloo, the device merge."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, SHARDED_SAME_DEVICE="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29531", os.path.join(here, "sharded_deepk_worker.py")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, env=env)
    assert p.returncode == 0 and "SHARDED_DEEPK_OK" in p.stdout, p.stdout[-3000:]
