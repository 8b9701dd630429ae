"""One batch through every kernel route at once, on the planner's threaded path (512 queries or more: the queries are
planned in chunks, one per thread, and the chunks' work items, launch lists and column / list / bitmap references are
merged).  Nested groups, point ranges and the flat shapes of every route (disjunctions as block streams, scored lists,
score columns and presence bitmaps; min_should_match; the DisiPriorityQueue; MUST_NOT only; conjunctions and ReqOpt
with MUST_NOT, FILTER and ranges) against the nested oracle, bit for bit, in both collector modes."""
import pytest

import nested_fixtures as nf
import nested_oracle as no
from rucene_b200 import engine, search
from test_gpu_nested import ranges, same

pytestmark = pytest.mark.gpu

M, S, N, F = nf.M, nf.S, nf.N, nf.F
R = 0x100  # a point-range clause

_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for _segs, s, _ix in _CACHE.values():
        s.engine.close()
    _CACHE.clear()


def fixture(flags):
    if flags not in _CACHE:
        segs, points, _ = nf.build(41)
        s = search.GpuIndexSearcher(search.IndexReader(segs), device=0, flags=flags)
        ix = no.NestedIndex(segs)
        for si, leaf in enumerate(points):
            for f, (nb, d, p, _) in leaf.items():
                ix.add_points(si, f, nb, d, p)
                s.engine.upload_points(si, f, nb, d, p)
        _CACHE[flags] = (segs, s, ix)
    return _CACHE[flags]


def flat_specs():
    """Shapes without groups, over terms 0..10 of nf.LEAF_DFS"""
    sp = []
    for a, b, c in [(0, 1, 2), (6, 7, 3), (2, 4, 9), (0, 6, 5), (1, 8, 10)]:
        sp.append(("bool", [(S, a), (S, b), (S, c)], 0))                     # plain sums
        sp.append(("bool", [(S, a), (S, b), (S, c), (S, 6)], 2))             # min_should_match > 1
        sp.append(("bool", [(N, a), (N, b)], 0))                             # only MUST_NOT: all docs, score 0
        sp.append(("bool", [(M, a), (N, b)], 0))                             # MUST + MUST_NOT
        sp.append(("bool", [(M, a), (M, c), (N, b)], 0))
        sp.append(("bool", [(M, a), (S, b), (S, c)], 0))                     # MUST + SHOULD (ReqOpt)
        sp.append(("bool", [(F, a), (M, b)], 0))                             # FILTER
        sp.append(("bool", [(F, a), (S, b), (S, c)], 0))
        sp.append(("bool", [(M, a), (F | R, 0), (N, c)], 0))                 # conjunctions with ranges
        sp.append(("bool", [(M, a), (S, b), (F | R, 1)], 0))
        sp.append(("bool", [(F | R, 2), (M, b), (N | R, 0)], 0))
    for n in (10, 11, 12):                                                   # DisiPriorityQueue in the first leaf
        sp.append(("bool", [(S, t % 11, 1.0 + t // 11) for t in range(n)], 0))
    return sp


def batch():
    sp = nf.specs([0, 1, 2]) * 4 + flat_specs()
    assert len(sp) >= 512
    return sp


def run(s, ix, sp, k, mode):
    rg = ranges()
    oq, oc, og = no.to_arrays(sp)
    want = ix.search_batch(oq, oc, og, k, ranges=rg, parallel_mode=mode)
    got = s.engine.search_batch_nested(no.engine_queries(oq), ix.engine_clauses(oc), no.engine_queries(og), k,
                                       k1=s.similarity.k1, mode=mode, ranges=rg)
    return got, want


@pytest.mark.parametrize("k", [10, 1000])
@pytest.mark.parametrize("mode", [engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL])
def test_threaded_plan_matches_the_oracle(k, mode):
    _segs, s, ix = fixture(0)
    same(*run(s, ix, batch(), k, mode), ("k", k, "mode", mode))


@pytest.mark.parametrize("flags", [engine.CFG_EAGER_COLUMNS, engine.CFG_MAXSCORE])
def test_threaded_plan_with_columns_and_bitmaps(flags):
    """CFG_EAGER_COLUMNS: every clause that can have a score column or a scored list gets one; CFG_MAXSCORE: plain sums
    go to k_eval_or_ms with presence-bitmap references.  Every thread's chunk refers to them."""
    _segs, s, ix = fixture(flags)
    for mode in (engine.MODE_SEARCH, engine.MODE_SEARCH_PARALLEL):
        same(*run(s, ix, batch(), 1000, mode), ("flags", flags, "mode", mode))
