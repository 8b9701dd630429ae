"""An independent numpy model of BooleanQuerys with pure-SHOULD groups of terms (no ranges), from the leaves' postings:
BM25 cells in f32 (edge_fixtures), per leaf —
  - a group is 0.0f + its present members' cells in member order on the docs any of them has; none present: a
    required group leaves the leaf without a match, an optional or excluded one is left out;
  - required terms and groups are added in order of their cost (a term's df, a group's sum of its present members'
    df; stable), starting from the cheapest one's value; a FILTER term or group adds 0;
  - MUST_NOT terms and groups exclude their docs;
  - beside a required clause, the optional side (0.0f + each present optional term / group in clause order) follows
    ReqOptScorer's sequential (scores_sum, scores_num) chain over the leaf's collected docs.
`rule` swaps in a wrong rule, to show that a fixture tells it apart: "flat" (a group's members added straight into the
conjunction's sum), "max_cost" (a group's cost = its largest present member df), "no_zero" (a group's sum starts from
its first present member's cell instead of 0.0f).
Specs are nested_oracle.to_arrays specs: ("bool", [(occur, term[, boost]) | (occur, [(term[, boost])...], msm)], 0)."""
import numpy as np

import edge_fixtures as E
import oracle_binding as ob

F32 = np.float32
M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER


def _leaf(segs, post, si, spec, rule, k1, b):
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

    mask = np.ones(md, bool)
    req, opt = [], []   # (cost, [(presence, cell)...] members or one term, is_group)
    for cl in spec[1]:
        occ = cl[0]
        scoring = occ not in (F, N)
        if isinstance(cl[1], list):
            members = [term(m[0], m[1] if len(m) > 1 else 1.0, scoring) for m in cl[1]]
            if len(members) == 1:   # a group of one clause is that clause
                members, grp = [members[0]], False
            else:
                grp = True
            present = [x for x in members if x[2] > 0]
        else:
            present, grp = [x for x in [term(cl[1], cl[2] if len(cl) > 2 else 1.0, scoring)] if x[2] > 0], False
        if occ == N:
            for p, _, _ in present:
                mask &= ~p
            continue
        if not present:
            if occ in (M, F):
                return np.zeros(0, np.int64), np.zeros(0, F32)
            continue
        cost = (max if rule == "max_cost" and grp else sum)(x[2] for x in present)
        (req if occ in (M, F) else opt).append((cost, present, grp))
    pres_req = np.ones(md, bool)
    for _, present, _ in req:
        p = np.zeros(md, bool)
        for x in present:
            p |= x[0]
        pres_req &= p

    def value(present, grp):
        """the clause's f32 value per doc (a group: 0.0f + members present on the doc, member order)"""
        if not grp:
            return present[0][1]
        v = None if rule == "no_zero" else np.zeros(md, F32)
        for p, c, _ in present:
            if v is None:
                v = np.where(p, c, F32(0.0)).astype(F32)
                seen = p.copy()
                continue
            if rule == "no_zero":
                v = np.where(p & seen, (v + c).astype(F32), np.where(p, c, v)).astype(F32)
                seen |= p
            else:
                v = np.where(p, (v + c).astype(F32), v).astype(F32)
        return v

    order = sorted(range(len(req)), key=lambda i: req[i][0])
    score = None
    for i in order:
        _, present, grp = req[i]
        if rule == "flat" and grp:
            for p, c, _ in present:
                vv = np.where(p, c, F32(0.0)).astype(F32)
                score = vv if score is None else np.where(p, (score + c).astype(F32), score).astype(F32)
            continue
        v = value(present, grp)
        score = v if score is None else (score + v).astype(F32)
    docs = np.nonzero(mask & pres_req & E.live_mask(seg))[0]
    sc = score[docs].copy()
    if opt:
        osum = np.full(md, np.nan, F32)
        for _, present, grp in opt:
            v = value(present, grp)
            hit = np.zeros(md, bool)
            for p, _, _ in present:
                hit |= p
            osum = np.where(hit, (np.where(np.isnan(osum), F32(0.0), osum) + v).astype(F32), osum).astype(F32)
        s, n = F32(0.0), 0
        for j, d in enumerate(docs):
            r = sc[j]
            if n > 100 and F32(F32(2.0) * r) < F32(s / F32(n)):
                continue
            s, n = F32(s + r), n + 1
            if not np.isnan(osum[d]):
                sc[j] = F32(r + osum[d])
    return docs, sc


def topdocs(segs, postings, spec, k, rule="right", k1=1.2, b=0.75):
    """TopDocs of one spec over all leaves (sequential collector): (docs, f32 scores, total_hits)"""
    all_d, all_s = [], []
    base = 0
    for si, seg in enumerate(segs):
        d, s = _leaf(segs, postings[si], si, spec, rule, k1, b)
        all_d.append(d + base)
        all_s.append(s)
        base += seg.max_doc
    d, s = np.concatenate(all_d), np.concatenate(all_s).astype(F32)
    o = np.lexsort((d, -s.astype(np.float64)))[:k]   # score descending, then docid ascending
    return d[o], s[o], len(d)
