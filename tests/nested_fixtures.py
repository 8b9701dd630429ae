"""Leaves for the nested-group tests: per-leaf term presence differs, so a group has all, some, one or none of its
members in some leaf; one leaf writes EF / BITSET doc blocks, one has deleted docs; every leaf has the point fields of
points_fixtures.  Query specs for nested_oracle.to_arrays."""
import numpy as np

import helpers
import oracle_binding as ob
import points_fixtures as pf

# df of terms 0..10 per leaf (0: absent from that leaf)
LEAF_DFS = [
    [30000, 9000, 3000, 700, 129, 100, 5000, 1500, 1, 256, 0],
    [12000, 0, 2500, 0, 300, 127, 4000, 0, 0, 1, 0],
    [20000, 6000, 0, 900, 0, 0, 3000, 800, 2, 0, 0],
]
SIZES = (70001, 40007, 31001)


def build(seed, doc_version=1):
    """-> (segs, points per leaf, postings per leaf: per term (docs, freqs))"""
    rng = np.random.default_rng(seed)
    segs, points, postings = [], [], []
    for i, md in enumerate(SIZES):
        seg, post = helpers.build_segment(rng, md, LEAF_DFS[i], doc_version=doc_version, use_ef=(i == 2),
                                       live_fraction=0.9 if i == 1 else None)
        segs.append(seg)
        postings.append(post)
        pts = pf.leaf_points(rng, md, i)
        points.append({f: (nb, d, pf.packed_of(nb, v), v) for f, (nb, d, v) in pts.items()})
    return segs, points, postings


M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER


def g(*terms, msm=0):
    return [(t,) if not isinstance(t, tuple) else t for t in terms], msm


def specs(range_ids):
    """Every accepted shape.  A group clause is (occur, members, msm)."""
    def grp(occ, *terms, msm=0):
        mem, m = g(*terms, msm=msm)
        return (occ, mem, m)
    R = 0x100
    sp = []
    pairs = [(0, 1), (2, 3), (4, 5), (6, 7), (1, 3), (5, 9), (8, 4), (3, 10), (10, 9)]
    for a, b in pairs:
        for c, d in pairs[::2]:
            sp.append(("bool", [grp(M, a, b), grp(M, c, d)], 0))            # +(a|b) +(c|d)
    for a, b in pairs:
        sp.append(("bool", [grp(M, a, b), (M, 6)], 0))                     # +(a|b) +c
        sp.append(("bool", [(M, 4), grp(M, a, b)], 0))                     # +a +(b|c)
        sp.append(("bool", [grp(M, a, b), (S, 2), grp(S, 5, 7)], 0))       # +(a|b) c (d|e)
        sp.append(("bool", [(M, 3), grp(S, a, b)], 0))                     # ReqOpt with an optional group
        sp.append(("bool", [grp(F, a, b), (M, 1)], 0))                     # FILTER group
        sp.append(("bool", [grp(F, a, b), (N, 6)], 0))                     # lone FILTER group beside MUST_NOT
        sp.append(("bool", [(M, 0), grp(N, a, b)], 0))                     # -(a|b)
        sp.append(("bool", [grp(M, a, b), (N, 2)], 0))                     # +(a|b) -c: the disjunction a b -c
        sp.append(("bool", [grp(M, a, b)], 0))                             # the query is the group
        sp.append(("bool", [grp(M, a), (M, b)], 0))                        # a group of one clause is its term
        sp.append(("bool", [grp(F, a), grp(M, b, 6)], 0))
    for ri in range_ids:
        sp.append(("bool", [grp(M, 0, 6), (F | R, ri)], 0))
        sp.append(("bool", [grp(M, 4, 5), (M | R, ri), (N | R, range_ids[0])], 0))
        sp.append(("bool", [(F | R, ri), grp(S, 1, 3), (S, 7)], 0))
        sp.append(("bool", [grp(F, 8, 9, 4), (M | R, ri), grp(N, 6, 7)], 0))
    # 8 members leading, one posting in all of them, -0.0 weights, a member msm of 1
    sp.append(("bool", [grp(M, 4, 5, 8, 9, 3, 1, 7, 2), (M, 0)], 0))
    sp.append(("bool", [grp(M, 0, 1, 2, 3, 4, 5, 6, 7), (F, 8)], 0))
    sp.append(("bool", [grp(M, (4, -0.0), (5, -0.0)), (M, 0)], 0))
    sp.append(("bool", [grp(M, (4, -0.0), 9), (F, 0), grp(M, 5, 3, msm=1)], 0))
    sp.append(("bool", [(M, 1, -0.0), grp(S, (4, -0.0), (9, -0.0))], 0))
    return sp


def refused_specs():
    """Shapes the nested entry points refuse with RG_EUNSUPPORTED."""
    def grp(occ, *terms, msm=0):
        mem, m = g(*terms, msm=msm)
        return (occ, mem, m)
    return [
        ("bool", [grp(S, 0, 1), grp(S, 2, 3)], 0),                           # (a|b) (c|d): a group in a disjunction
        ("bool", [grp(S, 0, 1), (S, 2)], 0),
        ("bool", [grp(S, 0, 1), (N, 2)], 0),
        ("bool", [grp(M, 0, 1, msm=2), (M, 2)], 0),                          # min_should_match > 1 in a group
        ("bool", [grp(M, 0, 1, 2, 3, 4), grp(M, 5, 6, 7, 8, 9)], 0),         # 10 clauses after flattening
        ("bool", [(M, 0), grp(N, 1, 2, 3, 4, 5), grp(N, 6, 7, 8, 9)], 0),
    ]


# ---- constructed leaves ------------------------------------------------------------------------------------------
EDGE_MAX_DOC = 20000
SPLIT_R = 16   # items of the split query at range_postings = SPLIT_RP (its group's cost is 32)
SPLIT_RP = 2


def _postings(rng, docs):
    docs = np.unique(np.asarray(docs, np.int32))
    return docs, rng.integers(1, 6, len(docs)).astype(np.int32)


def edge_leaf(seed=5, doc_version=1, use_ef=False):
    """One leaf for the edges of a group that leads (each query is `+group +t0`, t0 on every doc, so the group leads):
      t1..t3    interleaved (docid mod 3): their blocks end in turn, so each member bounds a step in turn
      t4..t11   127 docs each, disjoint, below 6200, plus doc 6200 in all eight: one step of exactly 1024 entries
      t12..t19  300 docs each plus doc 15000 in all eight
      t20       a singleton (doc 100); t21 a vint tail only (50 docs below 3000); t22 one block and a tail (200 docs):
                members that run out while the others go on
      t23, t24  the docs lo - 1 and lo of every item of `+(t23|t24) +t0` at range_postings SPLIT_RP
      t25, t26  random, for ReqOpt beside a group
    -> (codec.Segment, postings)"""
    import and_fixtures as A
    rng = np.random.default_rng(seed)
    md = EDGE_MAX_DOC
    post = [_postings(rng, np.arange(md))]
    for m in range(3):
        post.append(_postings(rng, np.arange(m, 3 * 700, 3)))
    pool = rng.permutation(6200)
    for m in range(8):
        post.append(_postings(rng, np.concatenate([pool[m * 127:(m + 1) * 127], [6200]])))
    for m in range(8):
        post.append(_postings(rng, np.concatenate([rng.choice(np.arange(7000, md), 300, replace=False), [15000]])))
    post.append(_postings(rng, [100]))
    post.append(_postings(rng, rng.choice(3000, 50, replace=False)))
    post.append(_postings(rng, rng.choice(md, 200, replace=False)))
    los = [md * r // SPLIT_R for r in range(1, SPLIT_R)]
    post.append(_postings(rng, [lo - 1 for lo in los] + [5, md - 1]))
    post.append(_postings(rng, los))
    post.append(_postings(rng, rng.choice(md, 900, replace=False)))
    post.append(_postings(rng, rng.choice(md, 4000, replace=False)))
    norms = rng.integers(1, 120, md).astype(np.uint8)
    seg, _ = A.write_leaf(md, post, norms, doc_version=doc_version, use_ef=use_ef)
    return seg, post


def edge_specs():
    T = lambda *ts: [(t,) for t in ts]
    return [
        ("bool", [(M, T(1, 2, 3)), (M, 0)], 0),
        ("bool", [(M, T(4, 5, 6, 7, 8, 9, 10, 11)), (M, 0)], 0),
        ("bool", [(M, T(12, 13, 14, 15, 16, 17, 18, 19)), (M, 0)], 0),
        ("bool", [(M, T(20, 21, 22, 1)), (M, 0)], 0),
        ("bool", [(M, T(23, 24)), (M, 0)], 0),
        ("bool", [(M, T(1, 2, 3)), (S, 25), (S, T(22, 26))], 0),
        ("bool", [(F, T(20, 21, 22)), (M, 0), (N, T(2, 26))], 0),
    ]


def discrimination_leaf(seed=9):
    """A leaf whose queries tell the wrong rules of nested_model apart (see discrimination_specs):
      t0 (50 docs) within t1 (1000) and within t2 | t3 (600 + 600): by the sum of its present members' df the group
      (1200) is added after t1, by its largest member's df (600) before it;
      t4 carries the same docs as t0 and is scored with a -0.0 boost, t5 absent."""
    import and_fixtures as A
    rng = np.random.default_rng(seed)
    md = 8000
    g2 = rng.choice(md, 600, replace=False)
    g3 = rng.choice(np.setdiff1d(np.arange(md), g2), 600, replace=False)
    lead = np.concatenate([g2[:25], g3[:25]])
    t1 = np.union1d(lead, rng.choice(md, 1000 - 50, replace=False))[:1000]
    t1 = np.union1d(t1, lead)
    post = [_postings(rng, lead), _postings(rng, t1), _postings(rng, g2), _postings(rng, g3), _postings(rng, lead),
            (np.zeros(0, np.int32), np.zeros(0, np.int32))]
    norms = rng.integers(1, 120, md).astype(np.uint8)
    seg, _ = A.write_leaf(md, post, norms)
    return seg, post


def discrimination_specs():
    return {
        "flat": ("bool", [(M, [(1,), (2,)], 0), (M, [(0,), (4,)], 0)], 0),
        "max_cost": ("bool", [(M, 0), (M, 1), (M, [(2,), (3,)], 0)], 0),
        "no_zero": ("bool", [(M, [(4, -0.0), (5,)], 0), (M, 0, -0.0)], 0),
    }
