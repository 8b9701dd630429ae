// orc_rescore — QueryRescorer::rescore (src/core/search/scorer/rescorer.rs of zhihu/rucene) over the oracle's own
// scorer trees.  TEST INFRASTRUCTURE: the parity reference of the device's rescoring (tests/rescore_oracle.py binds it).
//
// It includes oracle/oracle.cpp unchanged, so the index model, the BM25 weights (make_weight) and every scorer with its
// advance() / next() / score() (create_scorer, BooleanWeight::create_scorer) are the oracle's; what is added here is the
// rescorer itself, restated literally:
//   rescore             rescorer.rs:542-556   total_hits == 0 or no hits: nothing changes
//   query_rescore       rescorer.rs:300-354   truncate to window_size, stable sort by docid, iterative_rescore, sort()
//   iterative_rescore   rescorer.rs:229-298   one scorer per leaf; advance() when behind; matched iff doc == target
//   combine_score       rescorer.rs:356-373
//   combine_docs        rescorer.rs:375-417   the window replaces the first hits; the tail is scaled by query_weight
//   RescoreMode         rescorer.rs:96-115
//   ScoreDocHit's Ord   sort_field/collapse_top_docs.rs:180-201 (score reversed via partial_cmp, then docid);
//                       order_by_doc :161-170.  Vec::sort / sort_by are stable: std::stable_sort.
#include "../../oracle/oracle.cpp"

namespace {

enum { kAvg = 0, kMax = 1, kMin = 2, kTotal = 3, kMultiply = 4 };

float combine(int mode, float primary, float secondary) {  // rescorer.rs:105-114
    switch (mode) {
        case kAvg: return (primary + secondary) / 2.0f;
        case kMax: return std::fmax(primary, secondary);  // f32::max: the non-NaN argument
        case kMin: return std::fmin(primary, secondary);
        case kTotal: return primary + secondary;
        default: return primary * secondary;
    }
}

// ScoreDocHit::partial_cmp == Less.  A NaN makes the reference's unwrap() panic; here it compares as "not less".
bool score_doc_hit_less(const orc_hit& a, const orc_hit& b) {
    if (b.score < a.score) return true;   // score().partial_cmp(..).reverse() == Less
    if (a.score < b.score) return false;
    if (!(a.score == b.score)) return false;
    return a.doc < b.doc;
}

void rescore_one(const orc_index& ix, const orc_query& q, const orc_clause* clauses, uint32_t window, float query_weight,
                 float rescore_weight, int mode, orc_hit* row, uint32_t count, uint64_t total) {
    if (total == 0 || count == 0) return;  // :548-550
    // query_rescore (:300-306): the first window_size hits, stable-sorted by docid
    std::vector<orc_hit> hits(row, row + std::min<uint32_t>(count, window));
    std::stable_sort(hits.begin(), hits.end(), [](const orc_hit& a, const orc_hit& b) { return a.doc < b.doc; });
    // req.query.create_weight (:329): one weight per clause, as IndexSearcher::search builds them
    Plan plan;
    plan.weights.resize(q.n_clauses);
    for (uint32_t i = 0; i < q.n_clauses; i++)
        make_weight(ix, clauses[q.clause_begin + i].term_id, clauses[q.clause_begin + i].boost, plan.weights[i]);
    // iterative_rescore (:229-298)
    int32_t end_doc = 0, doc_base = 0;
    int reader_idx = -1, current_reader_idx = -1;
    ScorerPtr scorer;
    for (orc_hit& h : hits) {
        const int32_t doc_id = h.doc;
        const float current_score = h.score;
        while (doc_id >= end_doc && reader_idx < (int)ix.segs.size() - 1) {
            reader_idx++;
            end_doc = ix.segs[(size_t)reader_idx].doc_base + ix.segs[(size_t)reader_idx].max_doc;
        }
        if (reader_idx != current_reader_idx) {
            const SegmentData& seg = ix.segs[(size_t)reader_idx];
            doc_base = seg.doc_base;
            scorer = create_scorer(ix, seg, q, clauses, plan);
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
        // combine_score (:356-373)
        h.score = matched ? combine(mode, current_score * query_weight, new_score * rescore_weight)
                          : current_score * query_weight;
    }
    std::stable_sort(hits.begin(), hits.end(), score_doc_hit_less);  // hits.sort() (:351)
    // combine_docs (:375-417)
    const size_t rescore_len = hits.size();
    for (size_t i = 0; i < rescore_len; i++) row[i] = hits[i];
    for (size_t i = rescore_len; i < count; i++) row[i].score = row[i].score * query_weight;
}

}  // namespace

extern "C" {

// Every row i (hits[i * k, i * k + counts[i]), rewritten in place) rescored with queries[i]; n_threads: queries are
// independent, so they are spread over that many threads (the CPU rate of host-side rescoring).
int orc_rescore(orc_index* ix, const orc_query* queries, uint32_t n_queries, const orc_clause* clauses, uint32_t window,
                float query_weight, float rescore_weight, int mode, uint32_t k, orc_hit* hits, const uint32_t* counts,
                const uint64_t* total, int n_threads) {
    ORC_TRY
    if (ix->segs.empty()) throw Error("index has no segments");
    if (mode < kAvg || mode > kMultiply) throw Error("bad rescore mode");
    parallel_for(n_queries, n_threads, [&](uint32_t i) {
        rescore_one(*ix, queries[i], clauses, window, query_weight, rescore_weight, mode, hits + (size_t)i * k,
                    std::min(counts[i], k), total[i]);
    });
    return 0;
    ORC_CATCH(-1)
}

}  // extern "C"
