// orc_nested — one level of nested BooleanQuery (src/core/search/query/boolean_query.rs of zhihu/rucene): pure-SHOULD
// groups of TermQuerys as clauses of the oracle's BooleanQuery, beside terms and 1-D PointRangeQuerys.  TEST
// INFRASTRUCTURE: the parity reference of the device's group clauses (tests/nested_oracle.py binds it).
//
// It includes orc_points.cpp (which includes oracle/oracle.cpp unchanged), so the term scorers, ConjunctionScorer,
// DisjunctionSumScorer, ReqOptScorer, ReqNotScorer, the range scorer and the TopDocs collector are the oracle's.
// What is added is BooleanWeight::create_scorer (:196-279) applied recursively: a group clause is the group's own
// BooleanQuery::build + create_scorer —
//   - a group of one clause is that clause (build, :66-75);
//   - otherwise a DisjunctionSumScorer over the members that have a scorer in the leaf, even over one (the `1 =>` arm
//     is commented out), None when none has; its cost() is the sum of theirs (disjunction_scorer.rs:39);
//   - a group under FILTER or MUST_NOT is built with needs_scores = false: its members are non-scoring term scorers
//     and its score() is 0.0f (disjunction_scorer.rs:57-64).
#include "orc_points.cpp"

namespace {

constexpr int32_t kGroupBit = 0x200;  // orc_clause.occur: a group, term_id indexes the group array

struct NestedCtx {
    const orc_index& ix;
    const PointTable& pts;
    const orc_point_range* ranges;
    const orc_query* groups;
    const orc_clause* clauses;
    std::map<uint32_t, SimWeight> weights;  // absolute clause index -> TermWeight
};

ScorerPtr term_scorer(const SegmentData& seg, NestedCtx& cx, uint32_t ci, bool needs_scores) {
    const orc_clause& c = cx.clauses[ci];
    if (c.term_id >= seg.terms.size() || seg.terms[c.term_id].doc_freq <= 0) return nullptr;
    if (!needs_scores) return ScorerPtr(new FilterTermScorer(seg, seg.terms[c.term_id]));
    return ScorerPtr(new TermScorer(seg, seg.terms[c.term_id], &cx.weights.at(ci)));
}

// the scorer of one clause of the outer query in leaf seg_i; occ: the clause's occur
ScorerPtr clause_scorer(uint32_t seg_i, NestedCtx& cx, uint32_t ci, int32_t occ) {
    const SegmentData& seg = cx.ix.segs[seg_i];
    const orc_clause& c = cx.clauses[ci];
    const bool needs_scores = occ != ORC_FILTER && occ != ORC_MUST_NOT;
    if (c.occur & kRangeBit) return range_scorer(cx.pts, seg_i, seg, cx.ranges[c.term_id]);
    if (!(c.occur & kGroupBit)) return term_scorer(seg, cx, ci, needs_scores);
    const orc_query& g = cx.groups[c.term_id];
    if (g.n_clauses == 1) return term_scorer(seg, cx, g.clause_begin, needs_scores);
    std::vector<ScorerPtr> v;
    for (uint32_t j = 0; j < g.n_clauses; j++)
        if (ScorerPtr s = term_scorer(seg, cx, g.clause_begin + j, needs_scores)) v.push_back(std::move(s));
    if (v.empty()) return nullptr;
    return ScorerPtr(new DisjunctionSumScorer(std::move(v), needs_scores, g.min_should_match > 0 ? g.min_should_match : 1));
}

// create_scorer_r (orc_points.cpp) with group clauses
ScorerPtr create_scorer_n(uint32_t seg_i, const orc_query& q, NestedCtx& cx) {
    auto occur_of = [&](uint32_t i) { return cx.clauses[q.clause_begin + i].occur & ~(kRangeBit | kGroupBit); };
    auto sub = [&](uint32_t i) { return clause_scorer(seg_i, cx, q.clause_begin + i, occur_of(i)); };
    if (!q.is_boolean) return sub(0);
    if (q.is_boolean == 2) throw Error("DisjunctionMaxQuery with groups is not modelled");
    int32_t msm = q.min_should_match;
    std::vector<uint32_t> musts, shoulds, filters, must_nots;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const int occ = occur_of(i);
        (occ == ORC_MUST ? musts : occ == ORC_SHOULD ? shoulds : occ == ORC_FILTER ? filters : must_nots).push_back(i);
    }
    if (msm <= 0) msm = musts.empty() ? 1 : 0;
    if (musts.size() + shoulds.size() + filters.size() + must_nots.size() == 0)
        throw Error("boolean query should at least contain one inner query!");
    if (must_nots.empty() && musts.size() + shoulds.size() + filters.size() == 1) {
        const uint32_t i = musts.size() == 1 ? musts[0] : shoulds.size() == 1 ? shoulds[0] : filters[0];
        return sub(i);
    }
    const bool match_all = musts.size() + shoulds.size() + filters.size() == 0;
    musts.insert(musts.end(), filters.begin(), filters.end());
    ScorerPtr must_scorer, should_scorer, must_not_scorer;
    const SegmentData& seg = cx.ix.segs[seg_i];
    if (match_all) must_scorer.reset(new AllDocsScorer(seg.max_doc));
    if (!musts.empty()) {
        std::vector<ScorerPtr> v;
        for (uint32_t i : musts) {
            ScorerPtr s = sub(i);
            if (!s) return nullptr;
            v.push_back(std::move(s));
        }
        if (v.size() > 1) must_scorer.reset(new ConjunctionScorer(std::move(v)));
        else must_scorer = std::move(v[0]);
    }
    {
        std::vector<ScorerPtr> v;
        for (uint32_t i : shoulds)
            if (ScorerPtr s = sub(i)) v.push_back(std::move(s));
        if (!v.empty()) should_scorer.reset(new DisjunctionSumScorer(std::move(v), true, msm));
    }
    {
        std::vector<ScorerPtr> v;
        for (uint32_t i : must_nots)
            if (ScorerPtr s = sub(i)) v.push_back(std::move(s));
        if (v.size() == 1) must_not_scorer = std::move(v[0]);
        else if (v.size() > 1) must_not_scorer.reset(new DisjunctionSumScorer(std::move(v), false, msm));
    }
    if (must_scorer) {
        if (should_scorer) {
            ScorerPtr ro(new ReqOptScorer(std::move(must_scorer), std::move(should_scorer)));
            if (must_not_scorer) return ScorerPtr(new ReqNotScorer(std::move(ro), std::move(must_not_scorer)));
            return ro;
        }
        if (must_not_scorer) return ScorerPtr(new ReqNotScorer(std::move(must_scorer), std::move(must_not_scorer)));
        return must_scorer;
    }
    if (should_scorer) {
        if (must_not_scorer) return ScorerPtr(new ReqNotScorer(std::move(should_scorer), std::move(must_not_scorer)));
        return should_scorer;
    }
    return nullptr;
}

void search_one_n(NestedCtx& cx, const orc_query& q, uint32_t k, int parallel_mode, orc_hit* out, uint32_t* out_count,
                  uint64_t* out_total) {
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const uint32_t ci = q.clause_begin + i;
        const orc_clause& c = cx.clauses[ci];
        if (c.occur & kRangeBit) continue;
        if (c.occur & kGroupBit) {
            const orc_query& g = cx.groups[c.term_id];
            for (uint32_t j = 0; j < g.n_clauses; j++) {
                const orc_clause& m = cx.clauses[g.clause_begin + j];
                make_weight(cx.ix, m.term_id, m.boost, cx.weights[g.clause_begin + j]);
            }
        } else {
            make_weight(cx.ix, c.term_id, c.boost, cx.weights[ci]);
        }
    }
    TopDocsHeap main(k);
    for (uint32_t si = 0; si < cx.ix.segs.size(); si++) {
        const SegmentData& seg = cx.ix.segs[si];
        ScorerPtr scorer = create_scorer_n(si, q, cx);
        if (!scorer) continue;
        if (parallel_mode == 0) {
            bulk_score(*scorer, &seg, [&](int32_t doc, Scorer& s) { main.collect(doc + seg.doc_base, s.score()); });
        } else {
            TopDocsHeap leaf(k);
            bulk_score(*scorer, &seg, [&](int32_t doc, Scorer& s) { leaf.collect(doc + seg.doc_base, s.score()); });
            main.total_hits += leaf.total_hits;
            for (const orc_hit& h : leaf.data) main.add_doc(h.doc, h.score);
        }
    }
    *out_total = main.total_hits;
    std::vector<orc_hit> hits = main.top_docs();
    *out_count = (uint32_t)hits.size();
    for (size_t i = 0; i < hits.size(); i++) out[i] = hits[i];
}

}  // namespace

extern "C" {

int orc_search_batch_nested(orc_index* ix, void* p, const orc_query* queries, uint32_t n_queries,
                            const orc_clause* clauses, const orc_point_range* ranges, const orc_query* groups,
                            uint32_t n_groups, uint32_t k, int parallel_mode, int n_threads, orc_hit* out_hits,
                            uint32_t* out_counts, uint64_t* out_total) {
    ORC_TRY
    if (ix->segs.empty()) throw Error("index has no segments");
    for (uint32_t i = 0; i < n_queries; i++)
        for (uint32_t c = 0; c < queries[i].n_clauses; c++) {
            const orc_clause& cl = clauses[queries[i].clause_begin + c];
            if ((cl.occur & kGroupBit) && cl.term_id >= n_groups) throw Error("group index out of bounds");
        }
    const PointTable& pts = *static_cast<PointTable*>(p);
    parallel_for(n_queries, n_threads, [&](uint32_t i) {
        NestedCtx cx{*ix, pts, ranges, groups, clauses, {}};
        search_one_n(cx, queries[i], k, parallel_mode, out_hits + (size_t)i * k, out_counts + i, out_total + i);
    });
    return 0;
    ORC_CATCH(-1)
}

}  // extern "C"
