"""The conjunction edge fixtures (and_fixtures.py) against the oracle and the numpy model, and each fixture's claim
about the edge it reaches."""
import numpy as np
import pytest

import and_fixtures as A
import helpers
import oracle_binding as ob
import points_oracle as po

F32 = np.float32


def _oracle(segs, specs, k, mode=0):
    ix = helpers.oracle_index(segs)
    q, c = A.queries(specs)
    return ix.search_batch(q, c, k, parallel_mode=mode, n_threads=4)


def _points_oracle(fx, specs, k, mode=0):
    ix = po.PointsIndex(fx.segs)
    for si, leaf in enumerate(fx.points):
        for f, (nb, d, p, _) in leaf.items():
            ix.add_points(si, f, nb, d, p)
    q, c = A.queries(specs)
    return ix.search_batch(q, c, fx.ranges, k, parallel_mode=mode)


# ---- A --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=list(A.A_VARIANTS))
def term_fixture(request):
    return A.TermLeadFixture(request.param)


def test_term_lead_fixture_matches_oracle_and_model(term_fixture):
    f = term_fixture
    specs = f.specs()
    for k in (10, 1000):
        A.same_as_model(_oracle(f.segs, specs, k), A.model_topdocs(f.segs, f.postings, specs), k, (f.variant, k))


def test_term_lead_fixture_reaches_its_edges(term_fixture):
    f = term_fixture
    post = f.postings[0]
    P, nb = f.P, f.nb
    assert nb >= 2000 and len(P) % 128 != 0
    assert [len(post[t][0]) for t in range(1, 9)] == list(A.A_LEAD_DFS)
    for t in range(2, 9):   # every lead hits P's first docid, the last docid of its last full block and its first
        docs = post[t][0]  # tail doc, and has a doc past P's last posting
        assert {int(P[0]), f.last_full, f.first_tail} <= set(docs.tolist()) and docs[-1] > P[-1]
    # lead docs on each probe block's first and last docid
    firsts, lasts = set(P[0:128 * nb:128].tolist()), set(P[127:128 * nb:128].tolist())
    assert len(firsts & set(post[8][0].tolist())) > 300 and len(lasts & set(post[8][0].tolist())) > 300
    # the gallop lead: jumps of 0, 1, 2, 2^k blocks and to nb, and both sides of every 32-slot boundary in one block
    g = post[A.A_GALLOP][0]
    blk = np.searchsorted(P[127:128 * nb:128], g)   # the probe block each lead doc falls in (nb: tail and past)
    jumps = set(np.diff(blk).tolist())
    assert {0, 1, 2, 4, 8, 64, 512, 1024} <= jumps and blk[-1] == nb, sorted(jumps)
    for p in range(31, len(g) - 1, 32):
        assert blk[p] == blk[p + 1] < nb, p
    # freq widths 1..31 in the probe and the width lead
    for t in (A.A_P, A.A_WIDTH):
        fr = post[t][1].astype(np.int64)
        widths = {int(fr[i:i + 128].max()).bit_length() for i in range(0, 128 * (len(fr) // 128), 128)}
        assert set(range(1, 32)) <= widths, (t, sorted(widths))
    # the cut lead: R = 4 items; docs at each item's lo, hi - 1 and hi; its last full block ends at the last lo - 1
    c = post[A.A_CUT][0]
    bounds = f.item_bounds(len(c), A.A_CUT_RP)
    assert len(bounds) == A.A_CUT_R
    cs = set(c.tolist())
    for lo, hi in bounds[1:]:
        assert {lo - 1, lo} <= cs
    assert c[128 * (len(c) // 128) - 1] == bounds[-1][0] - 1
    assert len(cs & set(P.tolist()) & {b for lo, _ in bounds for b in (lo - 1, lo)}) == 2 * (A.A_CUT_R - 1) + 1
    # MUST_NOT hits lead-block edges, probe-block edges and the probe's tail
    n = set(post[A.A_NOT][0].tolist())
    assert n & firsts and n & lasts and n & set(P[128 * nb:].tolist()) and int(post[8][0][127]) in n
    # EF / BITSET blocks where the variant asks for them
    if A.A_VARIANTS[f.variant][1]:
        assert f.block_counts[1] + f.block_counts[2] > 0, f.block_counts
    else:
        assert f.block_counts[1] == f.block_counts[2] == 0


# ---- B --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[False, True], ids=["plain", "ef"])
def reqopt_fixture(request):
    return A.ReqOptFixture(ef=request.param)


def test_reqopt_fixture_matches_oracle_and_model(reqopt_fixture):
    f = reqopt_fixture
    for k in (A.B_K, 1000):
        A.same_as_model(_oracle(f.segs, f.specs(), k), A.model_topdocs(f.segs, f.postings, f.specs()), k, k)


def test_reqopt_fixture_reaches_its_edges(reqopt_fixture):
    f = reqopt_fixture
    segs, post = f.segs, f.postings
    spec = f.specs()[0]
    # leaf 0: the 101st collected doc sits past the first step (1024 lead slots) and gets its optional score, the 102nd
    # does not; docs without o are collected too
    docs, sc, _ = A.model_leaf(segs, post, 0, spec)
    first, second = f.decisive[0]
    i1, i2 = int(np.nonzero(docs == first)[0][0]), int(np.nonzero(docs == second)[0][0])
    assert (i1, i2) == (100, 101) and first // 2 >= 1024
    _, nosk, _ = A.model_leaf(segs, post, 0, spec, skip="none")
    assert sc[i1] == nosk[i1] and sc[i2] != nosk[i2]
    lead_slots = post[0][A.B_A][0]
    dead = ~A.E.live_mask(segs[0])
    pre = lead_slots[:1030]
    assert dead[pre].sum() > 50 and np.isin(pre, post[0][A.B_N][0]).sum() > 50
    assert (~np.isin(docs[:100], post[0][A.B_O][0])).sum() >= 40
    # leaves 1 and 2: 2 * req equal to the f32 mean (and below the exact mean), and one ulp below it
    for li, kept in ((1, True), (2, False)):
        d, s, _ = A.model_leaf(segs, post, li, spec)
        req = A.model_leaf(segs, post, li, ("bool", spec[1][:2], 0))[1]
        assert len(d) == 103 and d[102] == 102
        s101 = F32(0.0)
        for r in req[:102]:
            s101 = F32(s101 + r)
        mean = F32(s101 / F32(102))
        two = F32(2.0) * req[102]
        if kept:
            assert two == mean and float(s101) / 102 > float(mean)
            assert s[102] != req[102]
        else:
            assert two == np.nextafter(mean, F32(-np.inf))
            assert s[102] == req[102]
    # leaf 3 starts again: its low doc is the 5th collected and gets o; leaf 4 has no o
    d3, s3, _ = A.model_leaf(segs, post, 3, spec)
    assert d3[4] == f.decisive[3][0] and s3[4] != A.model_leaf(segs, post, 3, ("bool", spec[1][:2], 0))[1][4]
    assert len(post[4][A.B_O][0]) == 0 and len(post[4][A.B_A][0]) > 0
    if f.ef:
        assert f.counts[4][1] + f.counts[4][2] > 0, f.counts[4]


@pytest.mark.parametrize("variant", ["ge", "le", "double", "none", "opt_only", "carry"])
def test_reqopt_fixture_tells_the_skip_rules_apart(reqopt_fixture, variant):
    """each wrong running-mean rule changes the TopDocs at k = B_K"""
    f = reqopt_fixture
    k = A.B_K
    want = A.model_topdocs(f.segs, f.postings, f.specs())
    kw = {"carry": True} if variant == "carry" else {"skip": variant}
    got = A.model_topdocs(f.segs, f.postings, f.specs(), **kw)
    assert any(not (np.array_equal(a[0][:k], b[0][:k]) and np.array_equal(a[1][:k].view(np.uint32), b[1][:k].view(np.uint32)))
               for a, b in zip(want, got)), variant


# ---- C --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[False, True], ids=["plain", "ef"])
def range_fixture(request):
    return A.RangeFixture(ef=request.param)


def test_range_fixture_matches_oracle_and_model(range_fixture):
    f = range_fixture
    specs = f.specs(len(f.ranges))
    for k in (10, 1000):
        A.same_as_model(_points_oracle(f, specs, k),
                        A.model_topdocs(f.segs, f.postings, specs, f.points, f.ranges), k, k)


def test_range_fixture_reaches_its_edges(range_fixture):
    f = range_fixture
    nb, docs, packed, _ = f.points[0][A.F_MAIN]
    keys = np.zeros(len(docs), np.uint64)
    for j in range(nb):
        keys = (keys << np.uint64(8)) | packed[:, j].astype(np.uint64)
    M = A.C_MAX_DOC
    blk = docs // 128
    rng0 = f.ranges[0]
    lo = np.uint64(int.from_bytes(bytes(rng0["lower"]), "big"))
    hi = np.uint64(int.from_bytes(bytes(rng0["upper"]), "big"))
    take = [bool(np.any(blk == b)) and keys[blk == b].max() >= lo and keys[blk == b].min() <= hi
            for b in range(A.C_BLOCKS)]
    assert [b for b in range(A.C_BLOCKS) if take[b]] == A.C_S
    steps, eighth = A.lead_schedule(take, 0, A.C_BLOCKS)
    assert 0 in eighth and 31 in eighth and len(steps[-1]) < 8 and A.C_BLOCKS % 32
    gaps = np.diff(A.C_S)
    assert gaps.max() > 64 and any(32 < g for g in gaps)
    # block C_W127: 127 docs, 128 values; the last partial block fully valued in F_MAIN, not in F_MISS
    w = blk == A.C_W127
    assert len(np.unique(docs[w])) == 127 and w.sum() == 128
    assert len(np.unique(docs[blk == A.C_BLOCKS - 1])) == M - 128 * (A.C_BLOCKS - 1)
    assert M - 1 in docs and M - 1 not in f.points[0][A.F_MISS][1]
    # the many-valued doc: 40 values, only the largest in the band; the doc above every band range
    m = docs == f.many_doc
    assert m.sum() == 40 and (keys[m] >= lo).sum() == 1
    assert keys[docs == f.above_doc].min() > hi
    # multi-valued docs uploaded with the band key first
    for x in range(128 * A.C_OOO + 3, 128 * A.C_OOO + 128, 9):
        kx = keys[docs == x]
        assert len(kx) == 2 and kx[0] > kx[1]
    # key extremes
    assert {0, 0xFFFFFFFF} <= set(_keys(f, A.F_INT).tolist())
    assert {0, (1 << 63) - 1, 1 << 63, (1 << 64) - 1} <= set(int(x) for x in _keys(f, A.F_LONG))
    # planner: range 3 has points in the leaf and none inside; range 8 counts t_eq's df, one below t_eq1's
    assert f.range_count(0, 3) == 0 and f.range_count(0, 8) == len(f.postings[0][A.C_T_EQ][0]) == 300
    assert len(f.postings[0][A.C_T_EQ1][0]) == 301
    # split items of the F_SEQ range: the matches include each item's first docid
    bounds = f.split_bounds()
    assert len(bounds) == 4
    seq = set(A.pf.model_docs(f.points[0], f.ranges[7]).tolist())
    assert all(lo_ in seq for lo_, _ in bounds[1:])
    if f.ef:
        assert f.block_counts[1] + f.block_counts[2] > 0, f.block_counts


def _keys(f, field):
    nb, _, packed, _ = f.points[0][field]
    keys = np.zeros(len(packed), np.uint64)
    for j in range(nb):
        keys = (keys << np.uint64(8)) | packed[:, j].astype(np.uint64)
    return keys
