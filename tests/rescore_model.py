"""An independent Python model of QueryRescorer::rescore (search/scorer/rescorer.rs:130-417) for score TopDocs.

It builds the reference's scorer tree per leaf (BooleanWeight::create_scorer, boolean_query.rs:196-279) from
per-term postings (the oracle's orc_postings) and BM25 scores (helpers.bm25_scores_numpy), walks the window in
docid order with doc_id() / advance() / next() / score() exactly as iterative_rescore does, combines, sorts with
ScoreDocHit's order and scales the tail (combine_docs).  Queries and clauses are in the engine's format
(engine.QUERY_DTYPE / CLAUSE_DTYPE: clause weights as the searcher computed them)."""
import numpy as np

from helpers import bm25_scores_numpy

NO_MORE = 0x7FFFFFFF
F = np.float32
MUST, SHOULD, MUST_NOT, FILTER = 0, 1, 2, 3
AVG, MAX, MIN, TOTAL, MULTIPLY = 0, 1, 2, 3, 4


class Term:
    """TermScorer (FILTER clauses: the same docs, score 0f32)."""

    def __init__(self, docs, scores):
        self.docs, self.scores, self.i, self.doc = docs, scores, -1, -1

    def cost(self):
        return len(self.docs)

    def next(self):
        self.i += 1
        self.doc = int(self.docs[self.i]) if self.i < len(self.docs) else NO_MORE
        return self.doc

    def advance(self, t):
        self.i = max(self.i, int(np.searchsorted(self.docs, t, side="left")))
        self.doc = int(self.docs[self.i]) if self.i < len(self.docs) else NO_MORE
        return self.doc

    def score(self):
        return F(self.scores[self.i])


class AllDocs:
    """MatchAllDocsQuery's scorer: every docid of the leaf, score 0."""

    def __init__(self, max_doc):
        self.max_doc, self.doc = max_doc, -1

    def next(self):
        return self.advance(self.doc + 1)

    def advance(self, t):
        self.doc = t if t < self.max_doc else NO_MORE
        return self.doc

    def score(self):
        return F(0.0)


class Conj:
    """ConjunctionScorer: children stably sorted by cost(); score = lead1 + lead2 + others."""

    def __init__(self, children):
        self.s = sorted(children, key=lambda c: c.cost())
        self.doc = -1

    def _align(self, doc):
        lead = self.s[0]
        while doc != NO_MORE:
            moved = False
            for o in self.s[1:]:
                if o.doc < doc:
                    o.advance(doc)
                if o.doc > doc:
                    doc = lead.advance(o.doc)
                    moved = True
                    break
            if not moved:
                break
        self.doc = doc
        return doc

    def next(self):
        return self._align(self.s[0].next())

    def advance(self, t):
        return self._align(self.s[0].advance(t))

    def score(self):
        acc = F(self.s[0].score() + self.s[1].score())
        for o in self.s[2:]:
            acc = F(acc + o.score())
        return acc


class Disj:
    """DisjunctionSumScorer (SimpleQueue): next() honours min_should_match, advance() does not; score = the
    clauses on the doc, in clause order, from 0.0f.  tie is not None: DisjunctionMaxScorer."""

    def __init__(self, children, msm=1, needs_scores=True, tie=None):
        self.s, self.msm, self.needs, self.tie = children, msm, needs_scores, tie
        self.doc = min(c.doc for c in children)

    def next(self):
        msm = max(self.msm, 1)
        while True:
            if self.doc == NO_MORE:
                return self.doc
            cd = self.doc
            for c in self.s:
                if c.doc == cd:
                    c.next()
            self.doc = min(c.doc for c in self.s)
            if msm > 1 and sum(1 for c in self.s if c.doc == self.doc) < msm:
                continue
            return self.doc

    def advance(self, t):
        for c in self.s:
            if c.doc < t:
                c.advance(t)
        self.doc = min(c.doc for c in self.s)
        return self.doc

    def score(self):
        if not self.needs:
            return F(0.0)
        acc, mx = F(0.0), F(-np.inf)
        for c in self.s:
            if c.doc == self.doc:
                v = c.score()
                acc = F(acc + v)
                mx = np.fmax(mx, v)
        if self.tie is None:
            return acc
        return F(mx + F(F(acc - mx) * F(self.tie)))


class ReqOpt:
    """ReqOptScorer (req_opt_scorer.rs:19-65) with its running mean.  skips: scores that took the required side
    alone because it was below half the mean."""

    def __init__(self, req, opt):
        self.req, self.opt, self.sum, self.num, self.skips = req, opt, F(0.0), 0, 0

    @property
    def doc(self):
        return self.req.doc

    def next(self):
        return self.req.next()

    def advance(self, t):
        return self.req.advance(t)

    def score(self):
        cur = self.req.doc
        s = self.req.score()
        if self.num > 100 and F(F(2.0) * s) < F(self.sum / F(self.num)):
            self.skips += 1
            return s
        self.sum = F(self.sum + s)
        self.num += 1
        od = self.opt.doc
        if od < cur:
            od = self.opt.advance(cur)
        if od == cur:
            s = F(s + self.opt.score())
        return s


class ReqNot:
    """ReqNotScorer (req_not_scorer.rs:21-119)."""

    def __init__(self, req, nots):
        self.req, self.nots = req, nots

    @property
    def doc(self):
        return self.req.doc

    def next(self):
        while True:
            d = self.req.next()
            if d == NO_MORE:
                return d
            if d == self.nots.doc:
                continue
            if d < self.nots.doc or d < self.nots.advance(d):
                return d

    def advance(self, t):
        d = self.req.advance(t)
        while d != NO_MORE:
            if d == self.nots.doc:
                return self.next()
            if d < self.nots.doc:
                return d
            self.nots.advance(d)
        return NO_MORE

    def score(self):
        return self.req.score()


class Model:
    """The index side of the model: per-(leaf, term) postings from the oracle, BM25 with the searcher's cache."""

    def __init__(self, ix, segs, cache, k1):
        self.ix, self.segs, self.cache, self.k1 = ix, segs, np.asarray(cache, np.float32), k1
        self.bases = np.concatenate([[0], np.cumsum([s.max_doc for s in segs])]).astype(np.int64)
        self._post = {}
        self.reqopt_skips = 0  # ReqOptScorer skips over every scorer rescore() has built

    def postings(self, si, t):
        key = (si, t)
        if key not in self._post:
            seg = self.segs[si]
            df = int(seg.terms["doc_freq"][t]) if t < len(seg.terms) else 0
            self._post[key] = self.ix.postings(si, t, df) if df > 0 else None
        return self._post[key]

    def term(self, si, c):
        p = self.postings(si, int(c["term_id"]))
        if p is None:
            return None
        docs, freqs = p
        if int(c["occur"]) == FILTER:
            return Term(docs, np.zeros(len(docs), np.float32))
        return Term(docs, bm25_scores_numpy(c["weight"], self.k1, freqs, self.segs[si].norms[docs], self.cache))

    def create_scorer(self, si, q, clauses):
        cl = clauses[int(q["clause_begin"]):int(q["clause_begin"]) + int(q["n_clauses"])]
        if int(q["flags"]) == 0:
            return self.term(si, cl[0])
        if int(q["flags"]) == 2:  # DisjunctionMaxQuery
            if len(cl) == 1:
                return self.term(si, cl[0])
            v = [s for s in (self.term(si, c) for c in cl) if s is not None]
            if not v:
                return None
            tie = float(np.array([q["min_should_match"]], np.int32).view(np.float32)[0])
            return v[0] if len(v) == 1 else Disj(v, tie=tie)
        musts = [c for c in cl if c["occur"] == MUST]
        shoulds = [c for c in cl if c["occur"] == SHOULD]
        filters = [c for c in cl if c["occur"] == FILTER]
        nots = [c for c in cl if c["occur"] == MUST_NOT]
        msm = int(q["min_should_match"])
        msm = msm if msm > 0 else (1 if not musts else 0)
        if not nots and len(musts) + len(shoulds) + len(filters) == 1:
            return self.term(si, (musts + shoulds + filters)[0])  # BooleanQuery::build's collapse
        must = None
        if not (musts or shoulds or filters):
            must = AllDocs(self.segs[si].max_doc)
        reqs = musts + filters
        if reqs:
            v = [self.term(si, c) for c in reqs]
            if any(s is None for s in v):
                return None
            must = Conj(v) if len(v) > 1 else v[0]
        v = [s for s in (self.term(si, c) for c in shoulds) if s is not None]
        should = Disj(v, msm) if v else None
        v = [s for s in (self.term(si, c) for c in nots) if s is not None]
        excl = None if not v else (v[0] if len(v) == 1 else Disj(v, msm, needs_scores=False))
        if must is not None:
            if should is not None:
                must = ReqOpt(must, should)
            return ReqNot(must, excl) if excl is not None else must
        if should is not None:
            return ReqNot(should, excl) if excl is not None else should
        return None


def combine(mode, a, b):
    if mode == AVG:
        return F(F(a + b) / F(2.0))
    if mode == MAX:
        return np.fmax(a, b)
    if mode == MIN:
        return np.fmin(a, b)
    if mode == TOTAL:
        return F(a + b)
    return F(a * b)


def sort_hits(hits):
    """hits.sort() with ScoreDocHit's Ord: score descending (partial_cmp: -0.0 == +0.0), then docid ascending;
    stable."""
    return sorted(hits, key=lambda h: (-float(h[1]), h[0]))


def rescore(model, queries, clauses, hits, counts, total, window, query_weight, rescore_weight, mode):
    """QueryRescorer::rescore on every row; returns the new hits array (counts and total_hits do not change)."""
    out = np.array(hits, copy=True)
    qw, rw = F(query_weight), F(rescore_weight)
    n_segs = len(model.segs)
    for qi in range(len(queries)):
        cnt = int(counts[qi])
        if int(total[qi]) == 0 or cnt == 0:
            continue
        row = out[qi]
        n = min(cnt, int(window))
        win = sorted([(int(row[i]["doc"]), F(row[i]["score"])) for i in range(n)], key=lambda h: h[0])
        reader, cur, end_doc, scorer = -1, -1, 0, None
        new = []
        for doc, sc in win:
            while doc >= end_doc and reader < n_segs - 1:
                reader += 1
                end_doc = int(model.bases[reader + 1])
            if reader != cur:
                if isinstance(getattr(scorer, "req", None), ReqOpt):
                    model.reqopt_skips += scorer.req.skips
                elif isinstance(scorer, ReqOpt):
                    model.reqopt_skips += scorer.skips
                scorer = model.create_scorer(reader, queries[qi], clauses)
                cur = reader
            last = F(sc * qw)
            v = last
            if scorer is not None:
                t = doc - int(model.bases[reader])
                a = scorer.doc
                if a < t:
                    a = scorer.advance(t)
                if a == t:
                    v = combine(mode, last, F(scorer.score() * rw))
            new.append((doc, v))
        if isinstance(getattr(scorer, "req", None), ReqOpt):
            model.reqopt_skips += scorer.req.skips
        elif isinstance(scorer, ReqOpt):
            model.reqopt_skips += scorer.skips
        new = sort_hits(new)
        for i, (d, s) in enumerate(new):
            row[i]["doc"] = d
            row[i]["score"] = s
        for i in range(n, cnt):
            row[i]["score"] = F(F(row[i]["score"]) * qw)
    return out
