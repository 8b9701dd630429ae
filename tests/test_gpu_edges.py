"""GPU parity on constructed worst cases (edge_fixtures.py; test_edges_cpu.py checks the fixtures themselves):
decisive docs on window, block, bitmap-word and range edges with k equal to the docs that must beat theta; one ulp
above theta; the slack of the column bound; k1, b, weights, +inf, subnormal and zero cells at the limits of the
positive-score route; norm caches above 1e10; leaves without norms.  TopDocs must be the oracle's, bit for bit."""
import numpy as np
import pytest

import edge_fixtures as E
import helpers
import oracle_binding as ob
from rucene_b200 import engine, search

pytestmark = pytest.mark.gpu

F32 = np.float32
# the seven engine configurations of test_gpu_search._run_both
CONFIGS = (engine.CFG_EAGER_COLUMNS | engine.CFG_MAXSCORE, engine.CFG_EAGER_COLUMNS | engine.CFG_MAXSCORE | engine.CFG_TFPLANES,
           engine.CFG_EAGER_COLUMNS, engine.CFG_EAGER_COLUMNS | engine.CFG_NO_LISTS,
           engine.CFG_NO_BITMAPS | engine.CFG_NO_LISTS, engine.CFG_MAXSCORE, 0)


def _batch(segs, specs, k, k1=1.2, b=0.75, mode=0, rp=0, flags=0):
    """-> (TopDocs, debug counters, number of score columns)"""
    s = search.GpuIndexSearcher(search.IndexReader(segs), similarity=search.BM25Similarity(k1, b), range_postings=rp,
                                flags=flags)
    try:
        qa, ca = s.compile_batch(helpers.to_queries(specs))
        bt = s.engine.prepare(qa, ca, k, k1=k1, mode=mode)
        try:
            bt.run()
            return bt.fetch(), bt.debug(), bt.columns()[0]
        finally:
            bt.close()
    finally:
        s.engine.close()


def _run_all(segs, specs, k, k1=1.2, b=0.75, mode=0, rp=0, label=""):
    ix = ob.Index(k1, b)
    for s in segs:
        ix.add_segment(s)
    q, c = ob.make_queries(specs)
    want = ix.search_batch(q, c, k, parallel_mode=mode, n_threads=4)
    for flags in CONFIGS:
        got, _, _ = _batch(segs, specs, k, k1, b, mode, rp, flags)
        helpers.assert_same_topdocs(got, want, "%s flags=%d" % (label, flags))
    return want


# ---- 1. spikes --------------------------------------------------------------------------------------------------------
SPIKE_CONFIGS = {"default": (0, {}), "eager": (engine.CFG_EAGER_COLUMNS, {}), "den64": (0, {"RG_OR_COL_DEN": "64"}),
                 "sweep": (0, {"RG_COLUMN_SWEEP": "1"}), "no_lists": (engine.CFG_NO_LISTS, {}),
                 "maxscore": (engine.CFG_MAXSCORE, {})}


@pytest.fixture(scope="module")
def spike_case():
    f = E.SpikeFixture()
    ix = helpers.oracle_index(f.segs)
    q, c = ob.make_queries(f.specs)
    want = {mode: ix.search_batch(q, c, E.K, parallel_mode=mode, n_threads=4) for mode in (0, 1)}
    return f, want


@pytest.mark.parametrize("config", list(SPIKE_CONFIGS))
def test_spikes_on_window_block_and_range_edges(spike_case, config, monkeypatch):
    f, want = spike_case
    flags, env = SPIKE_CONFIGS[config]
    for name in ("RG_OR_COL_DEN", "RG_COLUMN_SWEEP"):
        monkeypatch.delenv(name, raising=False)
    for name, v in env.items():
        monkeypatch.setenv(name, v)
    seen = {"decode_free_items": 0, "column_windows_from_bitmaps": 0, "column_windows_swept": 0}
    for mode in (0, 1):
        for rp in E.RANGE_POSTINGS:
            label = "%s mode=%d rp=%d" % (config, mode, rp)
            got, dbg, _ = _batch(f.segs, f.specs, E.K, mode=mode, rp=rp, flags=flags | engine.CFG_STATS)
            helpers.assert_same_topdocs(got, want[mode], label)
            for n in seen:
                seen[n] += dbg[n]
    if config == "default":   # the test reaches what it targets: the bound cleared windows, and swept others
        assert seen["decode_free_items"] > 0 and seen["column_windows_from_bitmaps"] > 0 and seen["column_windows_swept"] > 0, seen
    if config == "sweep":
        assert seen["column_windows_from_bitmaps"] == 0 and seen["column_windows_swept"] > 0, seen


# ---- 2. ulp-level cases -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["a", "b"])
def test_ulp_cases(case, monkeypatch):
    """(a) with k = 5 the seeds set theta = H: a later doc scoring H must stay out, the next float above H must enter.
    (b) with k = 1 doc B sets theta = C, the bound of A's columns-only window, which A's f32 sum exceeds: only the
    slack of the bound keeps that window from being counted from bitmaps."""
    monkeypatch.delenv("RG_COLUMN_SWEEP", raising=False)
    seg, _ = E.ulp_leaf()
    specs, k = (E.ulp_specs_a(), len(E.ULP_A_SEEDS)) if case == "a" else (E.ulp_specs_b(), 1)
    for rp in (0, 1 << 30):   # the planner's grid, one range
        want = _run_all([seg], specs, k, rp=rp, label="ulp %s rp=%d" % (case, rp))
        top = E.ULP_A_YDOC if case == "a" else E.ULP_B_ADOC
        assert want[0][0]["doc"][0] == top
    got, dbg, _ = _batch([seg], specs, k, flags=engine.CFG_STATS)
    assert dbg["decode_free_items"] > 0, dbg
    if case == "b":
        assert dbg["column_windows_from_bitmaps"] > 0, dbg


# ---- 3. the limits of the positive-score route ------------------------------------------------------------------------
def _limit_specs():
    sh = E.sh
    return [sh(7, 5), sh(5, 7), sh(7, 5, 3), sh(6, 4, 7), sh(2, 6, 5, 7), ("term", 6), ("term", 5),
            ("bool", [(ob.MUST, 7), (ob.MUST, 5)], 0), sh(7, 6, 4, 3)]


@pytest.mark.parametrize("k1", [0.0, 1e6, float(np.nextafter(F32(1e6), F32(np.inf)))])
@pytest.mark.parametrize("b", [0.0, 0.75, 1.0])
def test_k1_and_b_at_the_limits(k1, b):
    """k1 = 0: every posting scores w (all ties); k1 = 1e6 is the last k1 of the positive route, the next float is not"""
    segs = [E.limits_leaf(11)[0], E.limits_leaf(12, max_doc=20011, live_fraction=0.8)[0]]
    for mode in (0, 1):
        _run_all(segs, _limit_specs(), 10, k1=k1, b=b, mode=mode, label="k1=%r b=%r mode=%d" % (k1, b, mode))
    _run_all(segs[:1], _limit_specs(), 100, k1=k1, b=b, rp=3000, label="k1=%r b=%r k=100" % (k1, b))


def test_weights_on_both_sides_of_the_route_limits():
    segs = [E.limits_leaf(5)[0]]
    bo = E.weight_edge_boosts(segs)
    specs = []
    for i in range(4):   # each weight twice, so that its column is built
        specs += [E.sh((7, float(bo[7][i])), (5, float(bo[5][i]))), E.sh((5, float(bo[5][i])), (7, float(bo[7][i])), 4)]
    specs += [E.sh((7, float(bo[7][0])), (5, float(bo[5][1]))), E.sh((7, float(bo[7][2])), (5, float(bo[5][3])), 6)]
    for k in (10, 100):
        _run_all(segs, specs, k, label="weights k=%d" % k)


def test_infinite_cells():
    """k1 = 1e6, a weight near 1e30, freqs 300..599: the cells of term HOT are +inf from freq 340 on (ties at +inf, a
    block maximum and theta of +inf)"""
    segs = [E.limits_leaf(6, hot=True)[0]]
    bo = float(E.weight_edge_boosts(segs)[7][2])
    specs = [E.sh((E.HOT, bo / 2), 7), E.sh(7, (E.HOT, bo / 2)), E.sh((E.HOT, bo / 2), (5, bo)), E.sh((5, bo), (E.HOT, bo / 2)),
             ("term", E.HOT, bo / 2), E.sh((7, bo), (5, bo), 4), E.sh((5, bo), (7, bo))]
    for k in (1, 10, 1000):
        _run_all(segs, specs, k, k1=1e6, label="inf k=%d" % k)


def test_subnormal_and_zero_cells():
    """weights around 1e-40: subnormal cells, none flushed to zero; the smallest subnormal weight: some cells are +0.0f,
    and those docs still match (counted, and collected while the heap is open)"""
    segs = [E.limits_leaf(6)[0]]
    tiny = np.finfo(F32).smallest_subnormal
    sub = {t: float(E.tiny_boost(segs, t, 1e-40)) for t in (4, 5, 7)}
    zero = {t: float(E.tiny_boost(segs, t, tiny)) for t in (4, 5, 7)}
    specs = []
    for bo in (sub, zero):
        specs += [E.sh((7, bo[7]), (5, bo[5])), E.sh((5, bo[5]), (7, bo[7])), E.sh((4, bo[4]), (5, bo[5])),
                  ("term", 4, bo[4]), ("bool", [(ob.MUST, 7, bo[7]), (ob.MUST, 5, bo[5])], 0)]
    for k in (10, 1000):
        _run_all(segs, specs, k, label="subnormal k=%d" % k)


def test_norm_cache_above_1e10_next_to_a_clean_leaf():
    """Norm byte 1 selects a cache entry above 1e10: that leaf leaves the positive route (no score column, no decode-free
    item), the clean leaf next to it keeps it"""
    clean = E.limits_leaf(21)[0]
    dirty = E.limits_leaf(22, norm_byte_one=17)[0]
    specs = [E.sh(7, 5), E.sh(5, 7), E.sh(7, 5, 3), E.sh(4, 7), ("term", 7), ("bool", [(ob.MUST, 7), (ob.MUST, 5)], 0)]
    for mode in (0, 1):
        _run_all([clean, dirty], specs, 10, mode=mode, label="clean+dirty mode=%d" % mode)
    for segs, name in (([clean], "clean"), ([dirty], "dirty")):
        _run_all(segs, specs, 10, label=name)
        _, dbg, n_cols = _batch(segs, specs, 10)
        if name == "clean":
            assert dbg["decode_free_items"] > 0 and n_cols > 0, (dbg, n_cols)
        else:
            assert dbg["decode_free_items"] == 0 and n_cols == 0, (dbg, n_cols)


def _every_shape():
    sh = E.sh
    return [("term", 7), ("term", 3), ("bool", [(ob.MUST, 7), (ob.MUST, 5)], 0), sh(7, 5), sh(5, 7), sh(7, 5, 4, 3),
            ("bool", [(ob.MUST, 6), (ob.SHOULD, 7), (ob.SHOULD, 4)], 0),
            ("bool", [(ob.SHOULD, 7), (ob.SHOULD, 5), (ob.MUST_NOT, 6)], 0),
            ("bool", [(ob.MUST, 7), (ob.MUST_NOT, 4)], 0),
            ("bool", [(ob.SHOULD, 7), (ob.SHOULD, 6), (ob.SHOULD, 5)], 2),
            ("dismax", [(7,), (5,), (4,)], 0.3),
            ("bool", [(ob.FILTER, 7), (ob.MUST, 5)], 0), ("bool", [(ob.FILTER, 6)], 0), ("bool", [(ob.MUST_NOT, 5)], 0)]


@pytest.mark.parametrize("leaves", ["alone", "stats_leaf_without_norms", "stats_leaf_with_norms"])
def test_leaves_without_norms(leaves):
    """PostingsWriter.finish(norms=None): cache[norm] is k1 for every posting (stream_refill, k_eval_and, the column
    and list builders), next to a normed leaf whichever supplies the statistics (the larger max_doc)"""
    bare = E.limits_leaf(31, norms=False)[0]
    if leaves == "alone":
        segs = [bare]
    elif leaves == "stats_leaf_without_norms":
        segs = [E.limits_leaf(32, max_doc=20011, live_fraction=0.85)[0], bare]
    else:
        segs = [bare, E.limits_leaf(33, max_doc=40009)[0]]
    specs = _every_shape()
    for k1, b in ((1.2, 0.75), (0.0, 0.75)):
        for mode in (0, 1):
            _run_all(segs, specs, 10, k1=k1, b=b, mode=mode, label="%s k1=%r mode=%d" % (leaves, k1, mode))
    _run_all(segs, specs, 100, rp=2500, label="%s k=100" % leaves)
