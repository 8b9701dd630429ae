"""The nested rescoring oracle (tests/cpp/orc_rescore_nested.cpp) against an independent numpy model of
QueryRescorer with groups and point ranges, on the nested fixtures' leaves and points (no GPU).  The model takes the
per-doc group values of nested_model (0.0f plus the members on the doc in member order; cost = the sum of the present
members' df) and the range membership of the points fixtures' raw values, restricted to the window's targets; the
ReqOptScorer chain is replayed over the matched targets in docid order."""
import numpy as np
import pytest

import edge_fixtures as E
import nested_fixtures as nf
import nested_oracle as no
import oracle_binding as ob
import points_oracle as po
import rescore_nested_oracle as rno

F32 = np.float32
M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER
R = po.RANGE
# (field, lower, upper) of the ranges below, in raw values
RANGES = [(0, 1275, 200000), (1, -(1 << 29), 1 << 28), (0, -(1 << 40), 1 << 40)]


def range_array():
    pack = {8: po.long_pack, 4: po.int_pack}
    nb = {0: 8, 1: 4}
    return np.array([po.make_range(f, nb[f], pack[nb[f]](lo), pack[nb[f]](hi)) for f, lo, hi in RANGES],
                    po.RANGE_DTYPE)


def leaf_values(segs, post, points, si, spec, k1=1.2, b=0.75):
    """(matched mask, required score, optional sum or NaN) per doc of leaf si, or None when the leaf has no scorer"""
    seg = segs[si]
    md = seg.max_doc
    cache = E.norm_cache(segs, k1, b)

    def term(t, boost, scoring):
        docs, freqs = post[t] if t < len(post) else (np.zeros(0, np.int32), np.zeros(0, np.int32))
        pres = np.zeros(md, bool)
        pres[docs] = True
        cell = np.zeros(md, F32)
        if scoring and len(docs):
            nv = np.full(len(docs), F32(k1)) if seg.norms is None else cache[seg.norms[docs]]
            cell[docs] = E.cells(E.weight(segs, t, F32(boost)), k1, freqs, nv)
        return pres, cell, len(docs)

    def in_range(ri):
        f, lo, hi = RANGES[ri]
        m = np.zeros(md, bool)
        if f in points[si]:
            _, d, _, vals = points[si][f]
            d, vals = np.asarray(d), np.asarray(vals, np.int64)
            m[d[(vals >= lo) & (vals <= hi)]] = True
        return m, f in points[si]

    def value(present, grp):
        if not grp:
            return present[0][1]
        v = np.zeros(md, F32)
        for p, c, _ in present:
            v = np.where(p, (v + c).astype(F32), v).astype(F32)
        return v

    mask = np.ones(md, bool)
    req, opt, req_rng = [], [], False
    for cl in spec[1]:
        occ = cl[0] & ~R
        if cl[0] & R:
            m, has = in_range(cl[1])
            if occ == N:
                mask &= ~m
            else:
                if not m.any():
                    return None
                mask &= m
                req_rng = True
            continue
        scoring = occ not in (F, N)
        if isinstance(cl[1], list):
            members = [term(x[0], x[1] if len(x) > 1 else 1.0, scoring) for x in cl[1]]
            grp = len(members) > 1
            present = [x for x in members if x[2] > 0]
        else:
            present, grp = [x for x in [term(cl[1], cl[2] if len(cl) > 2 else 1.0, scoring)] if x[2] > 0], False
        if occ == N:
            for p, _, _ in present:
                mask &= ~p
            continue
        if not present:
            if occ in (M, F):
                return None
            continue
        (req if occ in (M, F) else opt).append((sum(x[2] for x in present), present, grp))
    score = None
    for _, present, grp in sorted(req, key=lambda e: e[0]):
        p = np.zeros(md, bool)
        for x in present:
            p |= x[0]
        mask &= p
        v = value(present, grp)
        score = v if score is None else (score + v).astype(F32)
    if score is None:
        score = np.zeros(md, F32)
    elif req_rng:
        score = (score + F32(0.0)).astype(F32)   # a range's +0.0f
    osum = None
    if opt:
        osum = np.full(md, np.nan, F32)
        for _, present, grp in opt:
            hit = np.zeros(md, bool)
            for p, _, _ in present:
                hit |= p
            v = value(present, grp)
            osum = np.where(hit, (np.where(np.isnan(osum), F32(0.0), osum) + v).astype(F32), osum).astype(F32)
    return mask, score, osum


def combine(mode, a, b):
    if mode == rno.AVG:
        return F32(F32(a + b) / F32(2.0))
    if mode == rno.TOTAL:
        return F32(a + b)
    return F32(a * b)


def model_rescore(segs, post, points, spec, row, count, window, qw, rw, mode):
    """rescorer.rs's rescore over one row (doc, score) with the model's scorer"""
    row = list(row[:count])
    win = sorted(row[:min(count, window)], key=lambda h: h[0])   # stable by docid
    out = []
    base = np.cumsum([0] + [sg.max_doc for sg in segs])
    for si in range(len(segs)):
        leaf = [h for h in win if base[si] <= h[0] < base[si + 1]]
        if not leaf:
            continue
        vals = leaf_values(segs, post[si], points, si, spec)
        s_sum, n = F32(0.0), 0
        for d, sc in leaf:
            first = F32(F32(sc) * F32(qw))
            ld = d - base[si]
            if vals is None or not vals[0][ld]:
                out.append((d, first))
                continue
            new = vals[1][ld]
            if vals[2] is not None:   # ReqOptScorer over the matched targets, docid order
                if not (n > 100 and F32(F32(2.0) * new) < F32(s_sum / F32(n))):
                    s_sum, n = F32(s_sum + new), n + 1
                    if not np.isnan(vals[2][ld]):
                        new = F32(new + vals[2][ld])
            out.append((d, combine(mode, first, F32(new * F32(rw)))))
    out.sort(key=lambda h: (-float(h[1]), h[0]))
    return out + [(d, F32(F32(sc) * F32(qw))) for d, sc in row[len(out):]]


@pytest.fixture(scope="module")
def nested():
    segs, points, post = nf.build(32, doc_version=1)
    ix, rx = no.NestedIndex(segs), rno.RescoreNestedIndex(segs)
    for si, leaf in enumerate(points):
        for f, (nb, d, p, _) in leaf.items():
            ix.add_points(si, f, nb, d, p)
            rx.add_points(si, f, nb, d, p)
    return segs, points, post, ix, rx


@pytest.mark.parametrize("mode", [rno.TOTAL, rno.MULTIPLY, rno.AVG])
@pytest.mark.parametrize("k,window", [(100, 50), (1000, 1000)])
def test_oracle_matches_the_model(nested, mode, k, window):
    segs, points, post, ix, rx = nested
    specs = nf.specs([0, 1, 2])
    firsts = [("bool", [(S, t) for t in ts], 0) for ts in ([0, 6, 3], [4, 7, 1, 9], [2, 0, 9, 6, 3])]
    fq, fc, fg = no.to_arrays([firsts[i % 3] for i in range(len(specs))])
    hits, counts, total = ix.search_batch(fq, fc, fg, k)
    oq, oc, og = no.to_arrays(specs)
    qw, rw = (0.5, 1.5) if mode == rno.MULTIPLY else (1.0, 2.0)
    got = rx.rescore(oq, oc, og, hits, counts, total, window, qw, rw, mode, ranges=range_array())
    matched_any = False
    for i, sp in enumerate(specs):
        n = int(counts[i])
        want = model_rescore(segs, post, points, sp, [(int(h["doc"]), F32(h["score"])) for h in hits[i]], n, window,
                             qw, rw, mode)
        assert [int(d) for d, _ in want] == [int(x) for x in got[i][:n]["doc"]], (i, sp)
        assert np.array_equal(np.array([s for _, s in want], F32).view(np.uint32), got[i][:n]["score"].view(np.uint32)), (i, sp)
        matched_any = matched_any or not np.array_equal(got[i][:n]["score"], (hits[i][:n]["score"] * F32(qw)).astype(F32))
    assert matched_any
