"""Deep top-k (k > 1024), CPU side: the score bucket map behind the histogram theta bound (monotone, every score of a
bucket at or above its edge, theta never above the k-th best of anything it counted), over random and extreme
floats and both maps; and the oracle's TopDocsCollector at k = 2048 / 4096 against an independent heap model."""
import numpy as np
import pytest

import deepk_model as dm
import helpers
import oracle_binding as ob
from rucene_b200 import codec

F = np.float32
EXTREME = np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1.17e-38, -1.17e-38, 5e-39, -5e-39, 3.4028235e38,
                    -3.4028235e38, 1.0, -1.0, 2.5, 7.75, 1e30, -1e30], np.float32)


def _floats(rng, n):
    """Random finite and non-finite f32 of every magnitude and sign (bit patterns), plus the extremes."""
    bits = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32)
    x = x[~np.isnan(x)]
    return np.concatenate([x, EXTREME, rng.normal(0, 10, n).astype(np.float32)])


MAPS = [dm.bucket_map(F(u)) for u in (F(1e-42), F(0.3), F(11.5), F(3.0e38))] + [dm.bucket_map(F(0)), dm.bucket_map(F(np.inf))]


def test_bucket_maps():
    assert dm.bucket_map(F(0)) == (0, 24) and dm.bucket_map(F(-1)) == (0, 24) and dm.bucket_map(F(np.inf)) == (0, 24)
    m = dm.bucket_map(F(8.0))
    assert m[1] == 18 and dm.edge(m, 255) == F(8.0)
    assert dm.edge(m, 255 - 32) == F(4.0) and dm.edge(m, 255 - 7 * 32) == F(8.0 / 128)
    assert dm.edge(m, 1 + 32) == F(2.0) * dm.edge(m, 1)  # 1/32 octave buckets
    # the absolute map's bucket 128 starts at +0: an all-zero query gets theta = +0, which no zero score beats
    assert dm.edge((0, 24), 128) == F(0) and not np.signbit(dm.edge((0, 24), 128))
    # the planner's bound: round-up sum of nextafter(w1), zero clauses skipped, a negative one disables it
    u = dm.score_bound([F(2.2), F(0.0), F(1.1)])
    assert u > F(2.2) + F(1.1) and u < F(3.3001)
    assert dm.score_bound([F(1), F(-0.5)]) == np.inf and dm.score_bound([F(0), F(-0.0)]) == 0


@pytest.mark.parametrize("mi", range(len(MAPS)))
def test_map_monotone_and_edges(mi):
    m = MAPS[mi]
    rng = np.random.default_rng(100 + mi)
    x = _floats(rng, 20000)
    # values above the map's range: they clamp into the top bucket and are still >= its edge
    with np.errstate(over="ignore"):
        above = np.array([np.nextafter(dm.edge(m, 255), F(np.inf)) * F(3)], np.float32)
    x = np.concatenate([x, above, np.array([dm.edge(m, b) for b in range(1, 256)], np.float32)])
    x = x[~np.isnan(x)]
    # monotone: x < y implies key(x) <= key(y) (-0 and +0 compare equal and may sit in neighbouring buckets)
    u, inv = np.unique(x, return_inverse=True)
    kx = dm.key(m, x)
    lo = np.full(len(u), 1 << 30)
    hi = np.full(len(u), -1)
    np.minimum.at(lo, inv, kx)
    np.maximum.at(hi, inv, kx)
    assert np.all(hi[:-1] <= lo[1:]), "the map is monotone"
    # ... and over the ordered values (-0 just below +0)
    o = np.argsort(dm.to_ordered(x), kind="stable")
    assert np.all(np.diff(dm.key(m, x[o])) >= 0)
    kk = dm.key(m, x)
    edges = np.array([dm.edge(m, b) for b in range(256)], np.float32)
    assert np.all(x[kk >= 1] >= edges[kk[kk >= 1]]), "every score of bucket b >= 1 is >= its edge"
    # each edge lands in its own bucket
    assert np.all(dm.key(m, edges[1:]) == np.arange(1, 256))


@pytest.mark.parametrize("mi", range(len(MAPS)))
def test_theta_of_any_subset_is_below_kth_best(mi):
    m = MAPS[mi]
    rng = np.random.default_rng(200 + mi)
    base = _floats(rng, 3000)
    if m[1] == 18:  # scores concentrated in the map's range, and heavy ties
        top = dm.edge(m, 255)
        base = np.concatenate([base, (rng.random(6000) * top).astype(np.float32),
                               np.repeat(rng.random(8).astype(np.float32) * top, 400)])
    for trial in range(40):
        n = int(rng.integers(1, len(base)))
        scores = rng.choice(base, size=n, replace=False)
        k = int(rng.choice([1, 2, 7, 1025, 2048, 4096, 16384, n, n + 1]))
        kth = np.sort(scores)[::-1][k - 1] if k <= n else F(-np.inf)
        sub = scores[rng.random(n) < rng.random()]
        th = dm.theta(m, dm.histogram(m, sub), k)
        assert th <= kth, (trial, k, th, kth)
        # NaNs are never counted
        th2 = dm.theta(m, dm.histogram(m, np.concatenate([sub, np.full(k, np.nan, np.float32)])), k)
        assert th2 == th


@pytest.mark.parametrize("k", [2048, 4096])
def test_oracle_collector_matches_heap_model(k):
    """Heavy ties around the heap root: which tied docs survive and their order follow std's heap layout."""
    rng = np.random.default_rng(k)
    n = 3 * k + 17
    sc = rng.integers(0, 9, n).astype(np.float32)
    docs = np.arange(n, dtype=np.int32)
    got, _ = ob.topk_stream(list(docs), list(sc), k)
    want, _ = dm.top_docs(list(zip(docs.tolist(), sc.tolist())), k)
    assert [(int(h["doc"]), float(h["score"])) for h in got] == want


@pytest.mark.parametrize("k", [2048, 4096])
def test_oracle_term_query_matches_model(k):
    """A TermQuery at k = 2048 / 4096 through the oracle's IndexSearcher equals the heap model over numpy BM25 scores
    (few distinct norms and freqs: many ties), for df below, at and above k."""
    rng = np.random.default_rng(7 + k)
    max_doc = 40000
    dfs = [k - 1, k, 3 * k + 5]
    w = codec.PostingsWriter(doc_version=1, max_doc=max_doc)
    postings = []
    for df in dfs:
        docs = np.sort(rng.choice(max_doc, size=df, replace=False)).astype(np.int32)
        freqs = rng.integers(1, 4, df).astype(np.int32)
        w.add_term(docs, freqs)
        postings.append((docs, freqs))
    norms = rng.choice(np.array([40, 60, 90], np.uint8), size=max_doc)
    seg = w.finish(norms=norms)
    ix = helpers.oracle_index([seg])
    q, c = ob.make_queries([("term", t) for t in range(len(dfs))])
    hits, counts, total = ix.search_batch(q, c, k)
    for t, (docs, freqs) in enumerate(postings):
        wgt, _idf, _avg, cache = ix.term_weight(t)
        scores = helpers.bm25_scores_numpy(wgt, 1.2, freqs, norms[docs], cache)
        want, tot = dm.top_docs(list(zip(docs.tolist(), scores.tolist())), k)
        assert int(total[t]) == tot and int(counts[t]) == len(want) == min(k, len(docs))
        assert [(int(h["doc"]), float(h["score"])) for h in hits[t][:counts[t]]] == want
