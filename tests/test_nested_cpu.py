"""The nested-group oracle (tests/cpp/orc_nested.cpp) on its own, without a GPU: the collapses and the MUST_NOT
flattening give the same TopDocs as the equivalent flat queries, and a group enters a conjunction's sum as one f32
value (0.0f + its members in member order), which a flattened sum does not reproduce."""
import numpy as np

import nested_fixtures as nf
import nested_oracle as no
import oracle_binding as ob

M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER
_IX = {}


def index():
    if not _IX:
        segs, _, _ = nf.build(32, 1)
        _IX["ix"], _IX["segs"] = no.NestedIndex(segs), segs
    return _IX["ix"], _IX["segs"]


def search(sp, k=1000):
    ix, _ = index()
    oq, oc, og = no.to_arrays(sp)
    if len(og) == 0:
        og = np.zeros(1, ob.QUERY_DTYPE)
    return ix.search_batch(oq, oc, og, k)


def same(a, b, label):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), label


def test_collapses_and_flattening():
    pairs = [(0, 1), (2, 3), (4, 5), (5, 9), (8, 4), (3, 10)]
    for a, b in pairs:
        same(search([("bool", [(M, [(a,)], 0), (M, 6)], 0)]), search([("bool", [(M, a), (M, 6)], 0)]), ("one", a))
        same(search([("bool", [(M, [(a,), (b,)], 0)], 0)]), search([("bool", [(S, a), (S, b)], 0)]), ("lone", a, b))
        same(search([("bool", [(M, [(a,), (b,)], 0), (N, 2)], 0)]),
             search([("bool", [(S, a), (S, b), (N, 2)], 0)]), ("reqnot", a, b))
        same(search([("bool", [(M, 0), (N, [(a,), (b,)], 0)], 0)]),
             search([("bool", [(M, 0), (N, a), (N, b)], 0)]), ("flattened MUST_NOT", a, b))


def test_a_group_is_one_value_of_the_conjunction_sum():
    """+(a|b) +(c|d) scores (0 + a + b) + (0 + c + d) in cost order; summing the four terms as one conjunction
    changes some f32 score."""
    ix, segs = index()
    k = sum(s.max_doc for s in segs)
    term = {}
    for t in range(10):
        h, c, _ = search([("bool", [(S, t), (N, 10)], 0)], k)  # (a -absent): the term's docs and scores
        term[t] = dict(zip(h[0][:c[0]]["doc"].tolist(), h[0][:c[0]]["score"].tolist()))
    leaf_of = np.cumsum([0] + [s.max_doc for s in segs])

    def model(groups, rule):
        """Scores of +g1 +g2 ... as {doc: f32 score}: groups in order of their present members' df sum; rule "flat"
        adds the members straight into the conjunction's sum."""
        out = {}
        docs = set.intersection(*[set().union(*[term[m].keys() for m in g]) for g in groups])
        for d in docs:
            li = int(np.searchsorted(leaf_of, d, side="right") - 1)
            df = lambda m: nf.LEAF_DFS[li][m] if m < len(nf.LEAF_DFS[li]) else 0
            present = [[m for m in g if df(m) > 0] for g in groups]
            order = sorted(range(len(groups)), key=lambda i: sum(df(m) for m in present[i]))
            s = np.float32(0)
            first = True
            for i in order:
                if rule == "flat":
                    vals = [np.float32(term[m][d]) for m in present[i] if d in term[m]]
                    for v in vals:
                        s = v if first else np.float32(s + v)
                        first = False
                    continue
                gs = np.float32(0)
                for m in present[i]:
                    if d in term[m]:
                        gs = np.float32(gs + np.float32(term[m][d]))
                s = gs if first else np.float32(s + gs)
                first = False
            out[d] = s
        return out

    cases = [[(0, 1), (2, 3)], [(6, 7), (0, 3)], [(0, 6), (1, 7), (2, 3)], [(1, 9), (7, 3)]]
    flat = 0
    for groups in cases:
        h, c, _ = search([("bool", [(M, [(m,) for m in g], 0) for g in groups], 0)], k)
        got = dict(zip(h[0][:c[0]]["doc"].tolist(), h[0][:c[0]]["score"].astype(np.float32).tolist()))
        want = model(groups, "right")
        assert got.keys() == want.keys()
        assert all(np.float32(got[d]).view(np.uint32) == want[d].view(np.uint32) for d in got), groups
        alt = model(groups, "flat")
        flat += sum(np.float32(got[d]).view(np.uint32) != alt[d].view(np.uint32) for d in got)
    assert flat > 0


# ---- the independent model (tests/nested_model.py) ----------------------------------------------------------------
import nested_model as nm  # noqa: E402


def matches(docs, scores):
    """{doc: f32 bits} of every match (ties leave the TopDocs order to the collector's heap, so sets are compared)"""
    return {int(d): int(np.float32(s).view(np.uint32)) for d, s in zip(docs, scores)}


def oracle_matches(ix, sp, k):
    oq, oc, og = no.to_arrays([sp])
    if len(og) == 0:
        og = np.zeros(1, ob.QUERY_DTYPE)
    h, c, t = ix.search_batch(oq, oc, og, k)
    assert int(c[0]) == int(t[0]), "k must cover every match"
    return matches(h[0][:c[0]]["doc"], h[0][:c[0]]["score"])


def test_model_equals_the_oracle_on_every_shape_without_ranges():
    segs, _, postings = nf.build(32, 1)
    ix = no.NestedIndex(segs)
    R = 0x100
    specs = [sp for sp in nf.specs([0]) if not any(not isinstance(c[1], list) and c[0] & R for c in sp[1])]
    assert len(specs) > 100
    k = sum(s.max_doc for s in segs)
    for sp in specs:
        d, s, tot = nm.topdocs(segs, postings, sp, k)
        assert oracle_matches(ix, sp, k) == matches(d, s), sp


def test_model_equals_the_oracle_on_the_constructed_leaves():
    for seg, post, specs in [nf.edge_leaf() + (nf.edge_specs(),),
                             nf.discrimination_leaf() + (list(nf.discrimination_specs().values()),)]:
        ix = no.NestedIndex([seg])
        for sp in specs:
            d, s, tot = nm.topdocs([seg], [post], sp, seg.max_doc)
            assert oracle_matches(ix, sp, seg.max_doc) == matches(d, s), sp


def test_the_fixtures_tell_the_wrong_rules_apart():
    """a group's sum flattened into the conjunction, a group's cost as its largest member df, a group sum that does
    not start from 0.0f (seen through a -0.0 member): each changes the matches' scores of its query"""
    seg, post = nf.discrimination_leaf()
    ix = no.NestedIndex([seg])
    for rule, sp in nf.discrimination_specs().items():
        want = oracle_matches(ix, sp, seg.max_doc)
        assert want == matches(*nm.topdocs([seg], [post], sp, seg.max_doc)[:2]), rule
        assert want != matches(*nm.topdocs([seg], [post], sp, seg.max_doc, rule=rule)[:2]), rule


def test_edge_leaf_reaches_its_edges():
    seg, post = nf.edge_leaf()
    last = lambda t, i: int(post[t][0][i])
    # interleaved members: the block ends of t1..t3 alternate
    ends = sorted((last(t, j), t) for t in (1, 2, 3) for j in range(127, len(post[t][0]), 128))
    assert [t for _, t in ends[:3]] == [1, 2, 3]
    # eight one-block members whose blocks all end on the shared doc 6200: 8 * 128 = 1024 entries in one step
    assert all(len(post[t][0]) == 128 and last(t, -1) == 6200 for t in range(4, 12))
    assert all(15000 in set(post[t][0].tolist()) for t in range(12, 20))
    assert len(post[20][0]) == 1 and len(post[21][0]) < 128
    los = [nf.EDGE_MAX_DOC * r // nf.SPLIT_R for r in range(1, nf.SPLIT_R)]
    assert set(los) <= set(post[24][0].tolist()) and {lo - 1 for lo in los} <= set(post[23][0].tolist())
    assert -(-(len(post[23][0]) + len(post[24][0])) // nf.SPLIT_RP) == nf.SPLIT_R
