// orc_rescore_nested — QueryRescorer::rescore (src/core/search/scorer/rescorer.rs of zhihu/rucene) with rescoring
// queries that hold pure-SHOULD groups of TermQuerys and 1-D PointRangeQuerys.  TEST INFRASTRUCTURE: the parity
// reference of the device's nested and range rescoring (tests/rescore_nested_oracle.py binds it).
//
// It includes orc_nested.cpp (which includes orc_points.cpp and so oracle/oracle.cpp unchanged), so the scorer of
// a (query, leaf) is create_scorer_n's recursive BooleanWeight::create_scorer.  What is added is the rescorer over
// those trees, restated as orc_rescore.cpp restates it over the flat ones:
//   rescore             rescorer.rs:542-556   total_hits == 0 or no hits: nothing changes
//   query_rescore       rescorer.rs:300-354   truncate to window_size, stable sort by docid, iterative_rescore, sort()
//   iterative_rescore   rescorer.rs:229-298   one scorer per leaf; advance() when behind; matched iff doc == target
//   combine_score       rescorer.rs:356-373
//   combine_docs        rescorer.rs:375-417   the window replaces the first hits; the tail is scaled by query_weight
//   RescoreMode         rescorer.rs:96-115
//   ScoreDocHit's Ord   sort_field/collapse_top_docs.rs:180-201; Vec::sort is stable: std::stable_sort.
#include "orc_nested.cpp"

namespace {

enum { kAvg = 0, kMax = 1, kMin = 2, kTotal = 3, kMultiply = 4 };

float combine(int mode, float primary, float secondary) {  // rescorer.rs:105-114
    switch (mode) {
        case kAvg: return (primary + secondary) / 2.0f;
        case kMax: return std::fmax(primary, secondary);
        case kMin: return std::fmin(primary, secondary);
        case kTotal: return primary + secondary;
        default: return primary * secondary;
    }
}

// ScoreDocHit::partial_cmp == Less (a NaN compares as "not less")
bool score_doc_hit_less(const orc_hit& a, const orc_hit& b) {
    if (b.score < a.score) return true;
    if (a.score < b.score) return false;
    if (!(a.score == b.score)) return false;
    return a.doc < b.doc;
}

void rescore_one_n(NestedCtx& cx, const orc_query& q, uint32_t window, float query_weight, float rescore_weight,
                   int mode, orc_hit* row, uint32_t count, uint64_t total) {
    if (total == 0 || count == 0) return;  // :548-550
    std::vector<orc_hit> hits(row, row + std::min<uint32_t>(count, window));
    std::stable_sort(hits.begin(), hits.end(), [](const orc_hit& a, const orc_hit& b) { return a.doc < b.doc; });
    // req.query.create_weight (:329): a TermWeight per term clause and group member (as search_one_n makes them)
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
    // iterative_rescore (:229-298)
    int32_t end_doc = 0, doc_base = 0;
    int reader_idx = -1, current_reader_idx = -1;
    ScorerPtr scorer;
    for (orc_hit& h : hits) {
        const int32_t doc_id = h.doc;
        const float current_score = h.score;
        while (doc_id >= end_doc && reader_idx < (int)cx.ix.segs.size() - 1) {
            reader_idx++;
            end_doc = cx.ix.segs[(size_t)reader_idx].doc_base + cx.ix.segs[(size_t)reader_idx].max_doc;
        }
        if (reader_idx != current_reader_idx) {
            doc_base = cx.ix.segs[(size_t)reader_idx].doc_base;
            scorer = create_scorer_n((uint32_t)reader_idx, q, cx);
            current_reader_idx = reader_idx;
        }
        bool matched = false;
        float new_score = 0.0f;
        if (scorer) {
            const int32_t target_doc = doc_id - doc_base;
            int32_t actual_doc = scorer->doc_id();
            if (actual_doc < target_doc) actual_doc = scorer->advance(target_doc);
            if (actual_doc == target_doc) {
                matched = true;
                new_score = scorer->score();
            }
        }
        h.score = matched ? combine(mode, current_score * query_weight, new_score * rescore_weight)
                          : current_score * query_weight;
    }
    std::stable_sort(hits.begin(), hits.end(), score_doc_hit_less);
    const size_t rescore_len = hits.size();
    for (size_t i = 0; i < rescore_len; i++) row[i] = hits[i];
    for (size_t i = rescore_len; i < count; i++) row[i].score = row[i].score * query_weight;
}

}  // namespace

extern "C" {

// Every row i (hits[i * k, i * k + counts[i]), rewritten in place) rescored with queries[i], whose clauses may be
// groups (term_id into `groups`) and ranges (term_id into `ranges`, points of table p); n_threads as orc_rescore.
int orc_rescore_nested(orc_index* ix, void* p, const orc_query* queries, uint32_t n_queries, const orc_clause* clauses,
                       const orc_point_range* ranges, const orc_query* groups, uint32_t n_groups, uint32_t window,
                       float query_weight, float rescore_weight, int mode, uint32_t k, orc_hit* hits,
                       const uint32_t* counts, const uint64_t* total, int n_threads) {
    ORC_TRY
    if (ix->segs.empty()) throw Error("index has no segments");
    if (mode < kAvg || mode > kMultiply) throw Error("bad rescore mode");
    for (uint32_t i = 0; i < n_queries; i++)
        for (uint32_t c = 0; c < queries[i].n_clauses; c++) {
            const orc_clause& cl = clauses[queries[i].clause_begin + c];
            if ((cl.occur & kGroupBit) && cl.term_id >= n_groups) throw Error("group index out of bounds");
        }
    const PointTable& pts = *static_cast<PointTable*>(p);
    parallel_for(n_queries, n_threads, [&](uint32_t i) {
        NestedCtx cx{*ix, pts, ranges, groups, clauses, {}};
        rescore_one_n(cx, queries[i], window, query_weight, rescore_weight, mode, hits + (size_t)i * k,
                      std::min(counts[i], k), total[i]);
    });
    return 0;
    ORC_CATCH(-1)
}

}  // extern "C"
