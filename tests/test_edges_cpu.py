"""The constructed indexes of edge_fixtures.py do what they claim: the oracle's TopDocs are the spike set in the order of
the numpy model, total_hits is the model's union count over live docs, and the ulp-level inequalities hold.  A failure
of test_gpu_edges.py then cannot come from a broken fixture."""
import numpy as np
import pytest

import edge_fixtures as E
import helpers
import oracle_binding as ob

F32 = np.float32
SLACK = F32(0.99999237060546875)   # 1 - 2^-17, the column bound's factor on theta (query_kernels.cu)


@pytest.fixture(scope="module")
def spikes():
    return E.SpikeFixture()


def _round_down(x64):
    r = F32(x64)
    return r if float(r) <= x64 else np.nextafter(r, F32(-np.inf))


@pytest.mark.parametrize("mode", [0, 1])
def test_spike_fixture_topdocs_are_the_spikes(spikes, mode):
    f = spikes
    bases = np.cumsum([0] + [s.max_doc for s in f.segs])
    ix = helpers.oracle_index(f.segs)
    q, c = ob.make_queries(f.specs)
    hits, counts, total = ix.search_batch(q, c, E.K, parallel_mode=mode, n_threads=4)
    for qi in range(len(f.specs)):
        scored = E.or_scores(f.segs, f.postings, f.clauses(qi))
        assert total[qi] == E.total_hits(f.segs, scored), qi
        sp = f.spikes(qi)
        assert 0 < len(sp) <= E.K
        h = F32(scored[0][0][0])                                  # the first seed of the first leaf
        for li, (acc, hit) in enumerate(scored):
            live = E.live_mask(f.segs[li])
            assert np.all(acc[:E.K] == h), (qi, li)               # every seed scores H
            other = hit & live
            other[:E.K] = False
            mine = np.array([d for l2, d in sp if l2 == li], np.int64)
            other[mine] = False
            assert acc[mine].min() > h and acc[other].max() < h, (qi, li)
        if f.kind[qi] == "A":   # the deleted spike is a match of no query
            assert not E.live_mask(f.segs[1])[f.dead_spike]
        sc = np.array([scored[li][0][d] for li, d in sp], F32)
        docs = np.array([bases[li] + d for li, d in sp], np.int64)
        order = np.lexsort((docs, -sc.astype(np.float64)))
        n = len(sp)
        assert counts[qi] == E.K
        assert np.array_equal(hits[qi]["doc"][:n], docs[order]), qi
        assert np.array_equal(hits[qi]["score"][:n].view(np.uint32), sc[order].view(np.uint32)), qi
        rest = hits[qi][n:]
        assert np.all(rest["score"] == h), qi
        assert all((d - bases[np.searchsorted(bases, d, "right") - 1]) < E.K for d in rest["doc"]), qi


def test_spike_fixture_geometry(spikes):
    f = spikes
    for li, seg in enumerate(f.segs):
        M = seg.max_doc
        assert M % 2 == 1
        st = f.stride[li]
        assert np.all(np.diff(st) == E.STRIDE) and E.STRIDE % 32 == 1 and E.STRIDE % 128 == 1 and E.STRIDE % 768 == 1
        if li == 0:
            assert len(set((st % 768).tolist())) == 768             # every offset of a window, hence of a block and a word
            assert {M * r // 256 for r in range(1, 256)} <= set(f.boundary[0].tolist())
            assert {M * r // 256 - 1 for r in range(1, 256)} <= set(f.boundary[0].tolist())
        assert M - 1 in set(f.boundary[li].tolist())
        cols = [len(f.postings[li][t][0]) for t in range(3)]
        assert min(cols) * 8 >= M                                   # columns at the default threshold
        lst = f.postings[li][3][0]
        assert 4096 <= len(lst) and len(lst) * 8 < M and len(lst) % 128 == 0
        starts = lst[::128]
        assert np.all(lst.reshape(-1, 128) - starts[:, None] == np.arange(128))   # runs of 128 consecutive docids
        assert np.all(np.diff(starts) % 768 == 1)
    # A queries read the stride column, B queries the boundary column; the list is used twice with one weight
    # (persistent) and once with another (batch-local), before and after the columns
    assert [c[1] for c in f.specs[2][1]] == [3, 0, 2] and [c[1] for c in f.specs[3][1]] == [0, 2, 3]


def test_ulp_case_a_one_ulp_above_theta():
    seg, post = E.ulp_leaf()
    segs = [seg]
    specs = E.ulp_specs_a()
    clauses = [(c[1], c[2]) for c in specs[0][1]]
    acc, hit = E.or_scores(segs, [post], clauses)[0]
    h = acc[E.ULP_A_SEEDS[0]]
    assert np.all(acc[list(E.ULP_A_SEEDS)] == h) and acc[E.ULP_A_X] == h
    assert acc[E.ULP_A_YDOC] == np.nextafter(h, F32(np.inf))
    others = hit.copy()
    others[list(E.ULP_A_SEEDS) + [E.ULP_A_X, E.ULP_A_YDOC]] = False
    assert acc[others].max() < h
    ix = helpers.oracle_index(segs)
    q, c = ob.make_queries(specs)
    hits, counts, total = ix.search_batch(q, c, len(E.ULP_A_SEEDS))
    assert total[0] == np.count_nonzero(hit)
    assert hits[0]["doc"][0] == E.ULP_A_YDOC and set(hits[0]["doc"][1:].tolist()) < set(E.ULP_A_SEEDS)   # ties: heap order
    assert E.ULP_A_X not in hits[0]["doc"]


def test_ulp_case_b_the_slack_of_the_column_bound():
    seg, post = E.ulp_leaf()
    segs = [seg]
    specs = E.ulp_specs_b()
    clauses = [(c[1], c[2]) for c in specs[0][1]]
    acc, hit = E.or_scores(segs, [post], clauses)[0]
    cache = E.norm_cache(segs, 1.2, 0.75)
    a = E.ULP_B_ADOC
    cells = [E.cells(E.weight(segs, t, bo), 1.2, [post[t][1][np.searchsorted(post[t][0], a)]], [cache[seg.norms[a]]])[0]
             for t, bo in clauses]
    c_ub = E.butterfly_round_up(cells)
    exact = sum(float(x) for x in cells)                         # f64: exact for three such f32 values
    assert exact <= float(c_ub) < float(acc[a])                   # A's f32 sum is above the bound C ...
    assert acc[E.ULP_B_BDOC] == c_ub                              # ... which B scores exactly
    assert _round_down(float(c_ub)) == c_ub                       # without the slack the window would clear: C <= theta
    assert _round_down(float(c_ub) * float(SLACK)) < c_ub         # with it, it does not
    # A is the block maximum of every column in its window (and the 32-aligned window holds only columns)
    w0 = a // 768 * 768
    for t, bo in clauses:
        docs, freqs = post[t]
        sel = (docs >= w0 - 128) & (docs < w0 + 768 + 128) & (docs != a)
        other = E.cells(E.weight(segs, t, bo), 1.2, freqs[sel], cache[seg.norms[docs[sel]]])
        assert other.max() < cells[[x[0] for x in clauses].index(t)]
    before = hit.copy()
    before[E.ULP_B_BDOC:] = False
    assert acc[before].max() < c_ub and np.all(acc[hit & (np.arange(len(acc)) > a)] < c_ub)
    ix = helpers.oracle_index(segs)
    q, c = ob.make_queries(specs)
    hits, counts, total = ix.search_batch(q, c, 1)
    assert hits[0]["doc"][0] == a and total[0] == np.count_nonzero(hit)


def test_weight_edges_land_on_both_sides():
    segs = [E.limits_leaf(5)[0]]
    for t, (lo_b, lo_a, hi_b, hi_a) in E.weight_edge_boosts(segs).items():
        w = [E.weight(segs, t, x) for x in (lo_b, lo_a, hi_b, hi_a)]
        assert w[0] < F32(1e-20) <= w[1] and np.nextafter(lo_b, F32(1)) == lo_a, (t, w)
        assert w[2] <= F32(1e30) < w[3] and np.nextafter(hi_b, F32(np.inf)) == hi_a, (t, w)


def test_infinite_subnormal_and_zero_cells():
    seg, post = E.limits_leaf(6, hot=True)
    segs = [seg]
    hi = E.weight_edge_boosts(segs)[7][2]
    # k1 = 1e6, a weight at 1e30: the hot term's cells overflow to +inf from freq 340 on, and are finite below
    cache = E.norm_cache(segs, 1e6, 0.75)
    w = E.weight(segs, E.HOT, hi / 2)
    docs, freqs = post[E.HOT]
    c = E.cells(w, 1e6, freqs, cache[seg.norms[docs]])
    assert np.isinf(c).any() and np.isfinite(c).any() and np.all(c > 0)
    # weights around 1e-40: subnormal, non-zero cells
    cache = E.norm_cache(segs, 1.2, 0.75)
    tiny = np.finfo(F32).smallest_subnormal
    for t in (4, 5, 7):
        docs, freqs = post[t]
        c = E.cells(E.weight(segs, t, E.tiny_boost(segs, t, 1e-40)), 1.2, freqs, cache[seg.norms[docs]])
        assert np.all((c > 0) & (c < np.finfo(F32).tiny))
        # the smallest subnormal weight: some cells round to +0.0f, some do not
        c = E.cells(E.weight(segs, t, E.tiny_boost(segs, t, tiny)), 1.2, freqs, cache[seg.norms[docs]])
        assert (c == 0).any() and (c > 0).any()
    # term 4 has fewer postings than k: the heap never fills, and the docs that score 0 are collected too
    ix = helpers.oracle_index(segs)
    q, cl = ob.make_queries([("term", 4, float(E.tiny_boost(segs, 4, tiny)))])
    hits, counts, total = ix.search_batch(q, cl, 1000)
    assert total[0] == counts[0] == len(post[4][0]) and (hits[0]["score"][:counts[0]] == 0).any()


def test_norm_byte_one_has_a_cache_entry_above_1e10():
    seg, _ = E.limits_leaf(7, norm_byte_one=17)
    assert E.norm_cache([seg], 1.2, 0.75)[1] > 1e10
    assert seg.norms[17] == 1 and np.count_nonzero(seg.norms == 1) == 1
    assert ob.lib().orc_norm_table(1) > 1e10    # the decoded field length behind it
