// searcher.hpp — C++ host mirror of the reference's search surface for the accelerated path,
// written over the C ABI (include/rucene_gpu.h).  The reference is Rust; its toolchain is absent
// here, so this header plays the role the Rust shim (INTEGRATION.md) plays in a Rucene build:
// same names, argument meaning and error behaviour as
//   search/searcher.rs:234-249         trait IndexSearcher (search)
//   search/query/term_query.rs:46-49   TermQuery::new(term, boost, ctx)
//   search/query/boolean_query.rs:40-87 BooleanQuery::build(musts, shoulds, filters, must_nots, msm)
//   search/collector/top_docs.rs:107-124 TopDocsCollector::new(k) / top_docs()
//   search/sort_field/collapse_top_docs.rs:22-68,288-326 ScoreDoc / TopDocs
//   search/similarity/bm25_similarity.rs:45-46,151-177 BM25Similarity, compute_weight
//   search/scorer/rescorer.rs:67-115,542-556 RescoreRequest, RescoreMode, QueryRescorer::rescore
//   search/query/point_range_query.rs  PointRangeQuery, IntPoint / LongPoint / FloatPoint / DoublePoint (1-D; the
//                                      sortable bytes of util/numeric.rs:163-220)
// (paths relative to src/core/ of zhihu/rucene).  Header-only; link librucene_gpu.so.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "bm25.hpp"
#include "rucene_gpu.h"

namespace rucene {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
struct IllegalArgument : Error {  // error::ErrorKind::IllegalArgument
    explicit IllegalArgument(const std::string& m) : Error(RG_EINVAL, m) {}
};
struct UnsupportedQuery : Error {  // caller falls back to DefaultIndexSearcher
    explicit UnsupportedQuery(const std::string& m) : Error(RG_EUNSUPPORTED, m) {}
};

struct Term {
    std::string field;
    std::string bytes;
    static Term create(std::string f, std::string b) { return Term{std::move(f), std::move(b)}; }
};

struct Query {
    virtual ~Query() = default;
};
using QueryPtr = std::shared_ptr<Query>;

struct TermQuery : Query {
    Term term;
    float boost;
    TermQuery(Term t, float b) : term(std::move(t)), boost(b) {}
    static QueryPtr create(Term t, float boost = 1.0f) { return std::make_shared<TermQuery>(std::move(t), boost); }
};

// A 1-D point range, bounds inclusive, as packed sortable bytes (4 or 8).  Scores 0f32: PointRangeWeight's weight is
// only set by normalize(), which the searcher never calls.
struct PointRangeQuery : Query {
    std::string field, lower, upper;
    PointRangeQuery(std::string f, std::string lo, std::string hi)
        : field(std::move(f)), lower(std::move(lo)), upper(std::move(hi)) {}
    static QueryPtr create(std::string field, std::string lower, std::string upper) {
        if (lower.size() != upper.size() || (lower.size() != 4 && lower.size() != 8))
            throw IllegalArgument("1-D points of 4 or 8 bytes: lower and upper must have the same length");
        return std::make_shared<PointRangeQuery>(std::move(field), std::move(lower), std::move(upper));
    }
};

namespace detail {
inline std::string be_bytes(uint64_t v, int n) {
    std::string out((size_t)n, '\0');
    for (int i = n - 1; i >= 0; i--, v >>= 8) out[(size_t)i] = (char)(v & 0xff);
    return out;
}
}  // namespace detail

// int_to_sortable_bytes / long_to_sortable_bytes: the sign bit flipped, big-endian
struct IntPoint {
    static std::string pack(int32_t v) { return detail::be_bytes((uint32_t)v ^ 0x80000000u, 4); }
    static QueryPtr new_range_query(std::string f, int32_t lo, int32_t hi) { return PointRangeQuery::create(std::move(f), pack(lo), pack(hi)); }
    static QueryPtr new_exact_query(std::string f, int32_t v) { return new_range_query(std::move(f), v, v); }
};
struct LongPoint {
    static std::string pack(int64_t v) { return detail::be_bytes((uint64_t)v ^ 0x8000000000000000ull, 8); }
    static QueryPtr new_range_query(std::string f, int64_t lo, int64_t hi) { return PointRangeQuery::create(std::move(f), pack(lo), pack(hi)); }
    static QueryPtr new_exact_query(std::string f, int64_t v) { return new_range_query(std::move(f), v, v); }
};
// sortable_float_bits / sortable_double_bits: -0.0 < +0.0, NaNs beyond the infinities
struct FloatPoint {
    static std::string pack(float f) {
        int32_t b;
        std::memcpy(&b, &f, 4);
        return IntPoint::pack(b ^ ((b >> 31) & 0x7fffffff));
    }
    static QueryPtr new_range_query(std::string fl, float lo, float hi) { return PointRangeQuery::create(std::move(fl), pack(lo), pack(hi)); }
    static QueryPtr new_exact_query(std::string fl, float v) { return new_range_query(std::move(fl), v, v); }
};
struct DoublePoint {
    static std::string pack(double d) {
        int64_t b;
        std::memcpy(&b, &d, 8);
        return LongPoint::pack(b ^ ((b >> 63) & 0x7fffffffffffffffll));
    }
    static QueryPtr new_range_query(std::string fl, double lo, double hi) { return PointRangeQuery::create(std::move(fl), pack(lo), pack(hi)); }
    static QueryPtr new_exact_query(std::string fl, double v) { return new_range_query(std::move(fl), v, v); }
};

// MatchAllDocsQuery (search/query/match_all_query.rs:28-116): every docid, score 0f32
struct MatchAllDocsQuery : Query {};
// ConstantScoreQuery::with_boost(query, boost) (match_all_query.rs:162-205)
struct ConstantScoreQuery : Query {
    QueryPtr query;
    float boost;
    ConstantScoreQuery(QueryPtr q, float b) : query(std::move(q)), boost(b) {}
    static QueryPtr with_boost(QueryPtr q, float b) { return std::make_shared<ConstantScoreQuery>(std::move(q), b); }
};

struct BooleanQuery : Query {
    std::vector<QueryPtr> must_queries, should_queries, filter_queries, must_not_queries;
    int32_t min_should_match = 0;
    // BooleanQuery::build — including the collapse of a single positive clause (:66-75)
    static QueryPtr build(std::vector<QueryPtr> musts, std::vector<QueryPtr> shoulds,
                          std::vector<QueryPtr> filters, std::vector<QueryPtr> must_nots,
                          int32_t min_should_match) {
        const int32_t msm = min_should_match > 0 ? min_should_match : (musts.empty() ? 1 : 0);
        if (musts.size() + shoulds.size() + filters.size() + must_nots.size() == 0)
            throw IllegalArgument("boolean query should at least contain one inner query!");
        if (must_nots.empty() && musts.size() + shoulds.size() + filters.size() == 1) {
            if (musts.size() == 1) return musts[0];
            if (shoulds.size() == 1) return shoulds[0];
            return ConstantScoreQuery::with_boost(filters[0], 0.0f);
        }
        if (musts.size() + shoulds.size() + filters.size() == 0)  // only must_not exists (:76-79)
            musts.push_back(std::make_shared<MatchAllDocsQuery>());
        auto q = std::make_shared<BooleanQuery>();
        q->must_queries = std::move(musts);
        q->should_queries = std::move(shoulds);
        q->filter_queries = std::move(filters);
        q->must_not_queries = std::move(must_nots);
        q->min_should_match = msm;
        return q;
    }
};

struct ScoreDoc {
    int32_t doc;
    float score;
    int32_t doc_id() const { return doc; }
};

class TopDocs {
public:
    TopDocs() = default;
    TopDocs(uint64_t total, std::vector<ScoreDoc> docs) : total_hits_(total), score_docs_(std::move(docs)) {}
    uint64_t total_hits() const { return total_hits_; }
    const std::vector<ScoreDoc>& score_docs() const { return score_docs_; }
    std::vector<ScoreDoc>& score_docs_mut() { return score_docs_; }

private:
    uint64_t total_hits_ = 0;
    std::vector<ScoreDoc> score_docs_;
};

class TopDocsCollector {
public:
    explicit TopDocsCollector(size_t estimated_hits) : estimated_hits_(estimated_hits) {
        if (estimated_hits == 0) throw IllegalArgument("estimated_hits must be >= 1");
    }
    bool needs_scores() const { return true; }
    size_t estimated_hits() const { return estimated_hits_; }
    const TopDocs& top_docs() const { return top_; }
    void fill(TopDocs t) { top_ = std::move(t); }  // called by the GPU searcher

private:
    size_t estimated_hits_;
    TopDocs top_;
};

struct BM25Similarity {
    float k1 = 1.2f, b = 0.75f;
};

// What the reader hands to the searcher per leaf (LeafReader::{postings,norm_values,live_docs} +
// the field's Terms statistics).
struct LeafData {
    const uint8_t* doc_file = nullptr;
    size_t doc_len = 0;
    const uint8_t* norms = nullptr;
    const uint64_t* live_docs = nullptr;
    const rg_term_state* terms = nullptr;
    uint32_t n_terms = 0;
    int32_t max_doc = 0;
    int64_t doc_count = 0, sum_total_term_freq = 0, sum_doc_freq = 0;
};

class GpuIndexSearcher {
public:
    // DefaultIndexSearcher::new(reader, None): uploads the leaves in order and takes the
    // collection statistics of the largest leaf (searcher.rs:306-363).
    GpuIndexSearcher(std::vector<LeafData> leaves, std::string field,
                     std::unordered_map<std::string, uint32_t> term_ids, BM25Similarity sim = {}, int device = -1)
        : leaves_(std::move(leaves)), field_(std::move(field)), term_ids_(std::move(term_ids)), sim_(sim) {
        if (leaves_.empty()) throw IllegalArgument("reader has no leaves");
        rg_config cfg{};
        cfg.device = device;
        check(rg_engine_create(&cfg, &engine_));
        int32_t base = 0;
        size_t best = 0;
        for (size_t i = 0; i < leaves_.size(); i++) {
            const LeafData& l = leaves_[i];
            check(rg_segment_upload(engine_, (uint32_t)i, base, l.max_doc, l.doc_file, l.doc_len, l.norms,
                                    l.live_docs, l.terms, l.n_terms));
            base += l.max_doc;
            if (l.max_doc > leaves_[best].max_doc) best = i;
        }
        max_doc_ = base;
        stats_ = best;
        const LeafData& s = leaves_[stats_];
        avgdl_ = bm25_avg_field_length(s.sum_total_term_freq, s.doc_count, max_doc_);
        float cache[256];
        bm25_norm_cache(sim_.k1, sim_.b, avgdl_, cache);
        check(rg_norm_cache_set(engine_, 0, cache));
    }
    ~GpuIndexSearcher() { rg_engine_destroy(engine_); }
    GpuIndexSearcher(const GpuIndexSearcher&) = delete;
    GpuIndexSearcher& operator=(const GpuIndexSearcher&) = delete;

    // The points of one 1-D point field of leaf `leaf` (what PointValues::intersect hands an accept-all visitor):
    // docs[i] has the packed sortable value packed[i * bytes_per_dim ..].  A field never uploaded has no points.
    void upload_points(uint32_t leaf, const std::string& field, uint32_t bytes_per_dim, const int32_t* docs,
                       const uint8_t* packed, size_t n) {
        auto it = point_fields_.emplace(field, (uint32_t)point_fields_.size()).first;
        check(rg_points_upload(engine_, leaf, it->second, bytes_per_dim, docs, packed, n));
    }

    // IndexSearcher::search(&query, &mut collector)
    void search(const Query& query, TopDocsCollector& collector) {
        std::vector<rg_clause> clauses;
        std::vector<rg_point_range> ranges;
        std::vector<rg_query> groups;
        rg_query q = compile(query, clauses, &ranges, &groups);
        const uint32_t k = (uint32_t)collector.estimated_hits();
        std::vector<rg_hit> hits(k);
        uint32_t count = 0;
        uint64_t total = 0;
        rg_search_params p{k, sim_.k1, RG_MODE_SEARCH, 0};
        if (!groups.empty())
            check(rg_search_batch_nested(engine_, &q, 1, clauses.data(), (uint32_t)clauses.size(), &p, ranges.data(),
                                         (uint32_t)ranges.size(), groups.data(), (uint32_t)groups.size(), hits.data(),
                                         &count, &total));
        else if (ranges.empty())
            check(rg_search_batch(engine_, &q, 1, clauses.data(), (uint32_t)clauses.size(), &p, hits.data(), &count, &total));
        else
            check(rg_search_batch_ranges(engine_, &q, 1, clauses.data(), (uint32_t)clauses.size(), &p, ranges.data(),
                                         (uint32_t)ranges.size(), hits.data(), &count, &total));
        std::vector<ScoreDoc> docs(count);
        for (uint32_t i = 0; i < count; i++) docs[i] = ScoreDoc{hits[i].doc, hits[i].score};
        collector.fill(TopDocs(total, std::move(docs)));
    }

    rg_engine* engine() { return engine_; }

    // The device side of QueryRescorer::rescore (below): rg_rescore_hits over top_docs as one row
    void rescore_top_docs(const Query& query, uint32_t window_size, float query_weight, float rescore_weight,
                          uint32_t mode, TopDocs& top_docs) {
        std::vector<ScoreDoc>& docs = top_docs.score_docs_mut();
        if (top_docs.total_hits() == 0 || docs.empty()) return;  // rescorer.rs:548-550
        std::vector<rg_clause> clauses;
        std::vector<rg_point_range> ranges;
        std::vector<rg_query> groups;
        rg_query q = compile(query, clauses, &ranges, &groups);
        std::vector<rg_hit> hits(docs.size());
        for (size_t i = 0; i < docs.size(); i++) hits[i] = rg_hit{docs[i].doc, docs[i].score};
        const uint32_t count = (uint32_t)docs.size();
        const uint64_t total = top_docs.total_hits();
        rg_rescore_params p{window_size, query_weight, rescore_weight, mode, sim_.k1, 0};
        if (groups.empty() && ranges.empty())
            check(rg_rescore_hits(engine_, &q, 1, clauses.data(), (uint32_t)clauses.size(), &p, count, hits.data(),
                                  &count, &total));
        else
            check(rg_rescore_hits_nested(engine_, &q, 1, clauses.data(), (uint32_t)clauses.size(), ranges.data(),
                                         (uint32_t)ranges.size(), groups.data(), (uint32_t)groups.size(), &p, count,
                                         hits.data(), &count, &total));
        for (size_t i = 0; i < docs.size(); i++) docs[i] = ScoreDoc{hits[i].doc, hits[i].score};
    }

private:
    void check(int rc) {
        if (rc == RG_OK) return;
        const std::string msg = rg_last_error(engine_);
        if (rc == RG_EUNSUPPORTED) throw UnsupportedQuery(msg);
        throw Error(rc, msg);
    }
    // TermQuery::create_weight -> BM25Similarity::compute_weight (idf from the statistics leaf)
    rg_clause clause_of(const TermQuery& tq, int32_t occur) const {
        rg_clause c{};
        c.occur = occur;
        c.term_id = 0xffffffffu;  // absent everywhere
        int64_t df = 0;
        const LeafData& s = leaves_[stats_];
        if (tq.term.field == field_) {
            auto it = term_ids_.find(tq.term.bytes);
            if (it != term_ids_.end()) {
                c.term_id = it->second;
                if (c.term_id < s.n_terms) df = s.terms[c.term_id].doc_freq;
            }
        }
        const int64_t doc_count = s.doc_count == -1 ? max_doc_ : s.doc_count;
        c.weight = bm25_idf(df, doc_count) * tq.boost;
        c.cache_id = 0;
        return c;
    }
    using Pending = std::vector<std::pair<size_t, const BooleanQuery*>>;  // (group index, nested query)
    // a TermQuery, (ranges != null) a PointRangeQuery or (groups != null) a nested pure-SHOULD BooleanQuery of
    // TermQuerys as one clause; a group's members are written after the query's own clauses (compile)
    void add_clause(const Query& leaf, int32_t occur, std::vector<rg_clause>& clauses,
                    std::vector<rg_point_range>* ranges, std::vector<rg_query>* groups = nullptr,
                    Pending* pending = nullptr) const {
        if (auto tq = dynamic_cast<const TermQuery*>(&leaf)) {
            clauses.push_back(clause_of(*tq, occur));
            return;
        }
        if (auto bq = dynamic_cast<const BooleanQuery*>(&leaf); bq && groups) {
            bool pure = bq->must_queries.empty() && bq->filter_queries.empty() && bq->must_not_queries.empty();
            for (const QueryPtr& m : bq->should_queries) pure = pure && dynamic_cast<const TermQuery*>(m.get());
            if (!pure) throw UnsupportedQuery("only pure-SHOULD groups of TermQuerys are accelerated");
            clauses.push_back(rg_clause{occur | RG_CLAUSE_GROUP, (uint32_t)groups->size(), 0.0f, 0u});
            pending->emplace_back(groups->size(), bq);
            groups->push_back(rg_query{0u, 0u, bq->min_should_match, RG_Q_BOOLEAN});
            return;
        }
        auto pq = dynamic_cast<const PointRangeQuery*>(&leaf);
        if (!pq) throw UnsupportedQuery("only TermQuery and PointRangeQuery leaves are accelerated");
        if (!ranges) throw UnsupportedQuery("PointRangeQuery is not accelerated here");
        rg_point_range r{};
        auto it = point_fields_.find(pq->field);
        r.field = it == point_fields_.end() ? 0xffffffffu : it->second;  // no leaf has points of it: no scorer anywhere
        r.bytes_per_dim = (uint32_t)pq->lower.size();
        std::memcpy(r.lower, pq->lower.data(), pq->lower.size());
        std::memcpy(r.upper, pq->upper.data(), pq->upper.size());
        clauses.push_back(rg_clause{occur | RG_CLAUSE_RANGE, (uint32_t)ranges->size(), 0.0f, 0u});
        ranges->push_back(r);
    }
    rg_query compile(const Query& query, std::vector<rg_clause>& clauses, std::vector<rg_point_range>* ranges = nullptr,
                     std::vector<rg_query>* groups = nullptr) const {
        Pending pending;
        const rg_query q = compile_one(query, clauses, ranges, groups, &pending);
        for (const auto& g : pending) {
            rg_query& gq = (*groups)[g.first];
            gq.clause_begin = (uint32_t)clauses.size();
            gq.n_clauses = (uint32_t)g.second->should_queries.size();
            for (const QueryPtr& m : g.second->should_queries)
                clauses.push_back(clause_of(static_cast<const TermQuery&>(*m), RG_SHOULD));
        }
        return q;
    }
    rg_query compile_one(const Query& query, std::vector<rg_clause>& clauses, std::vector<rg_point_range>* ranges,
                         std::vector<rg_query>* groups, Pending* pending) const {
        rg_query q{};
        q.clause_begin = (uint32_t)clauses.size();
        if (dynamic_cast<const TermQuery*>(&query) || dynamic_cast<const PointRangeQuery*>(&query)) {
            add_clause(query, RG_SHOULD, clauses, ranges);
            q.n_clauses = 1;
            return q;
        }
        if (auto cq = dynamic_cast<const ConstantScoreQuery*>(&query)) {  // the lone FILTER clause of build()
            if (!cq->query || cq->boost != 0.0f) throw UnsupportedQuery("only ConstantScoreQuery(leaf, 0) is accelerated");
            add_clause(*cq->query, RG_FILTER, clauses, ranges, groups, pending);
            q.n_clauses = 1;
            q.flags = RG_Q_BOOLEAN;
            return q;
        }
        auto bq = dynamic_cast<const BooleanQuery*>(&query);
        if (!bq) throw UnsupportedQuery("query type is not accelerated");
        std::vector<QueryPtr> musts = bq->must_queries;
        if (musts.size() == 1 && dynamic_cast<const MatchAllDocsQuery*>(musts[0].get()) && bq->should_queries.empty() &&
            bq->filter_queries.empty() && !bq->must_not_queries.empty())
            musts.clear();  // the engine reads "only MUST_NOT clauses" as MatchAllDocsQuery minus those terms
        auto add = [&](const std::vector<QueryPtr>& v, int32_t occur) {
            for (const QueryPtr& c : v) add_clause(*c, occur, clauses, ranges, groups, pending);
        };
        add(musts, RG_MUST);
        add(bq->filter_queries, RG_FILTER);
        add(bq->should_queries, RG_SHOULD);
        add(bq->must_not_queries, RG_MUST_NOT);
        q.n_clauses = (uint32_t)clauses.size() - q.clause_begin;
        q.min_should_match = bq->min_should_match;
        q.flags = RG_Q_BOOLEAN;
        return q;
    }

    std::vector<LeafData> leaves_;
    std::string field_;
    std::unordered_map<std::string, uint32_t> term_ids_;
    std::map<std::string, uint32_t> point_fields_;  // point field name -> engine-wide id, in upload order
    BM25Similarity sim_;
    rg_engine* engine_ = nullptr;
    int32_t max_doc_ = 0;
    size_t stats_ = 0;
    float avgdl_ = 1.0f;
};

// RescoreMode / RescoreRequest / QueryRescorer (search/scorer/rescorer.rs:67-115,542-556) for score TopDocs:
// the first window_size hits are rescored by request.query on the GPU and sorted again, the rest are scaled by
// query_weight.  More than 1024 hits, or a rescoring query outside the accelerated shapes, throws UnsupportedQuery
// (the caller then uses the CPU rescorer).
enum class RescoreMode : uint32_t {
    Avg = RG_RESCORE_AVG,
    Max = RG_RESCORE_MAX,
    Min = RG_RESCORE_MIN,
    Total = RG_RESCORE_TOTAL,
    Multiply = RG_RESCORE_MULTIPLY,
};

struct RescoreRequest {
    QueryPtr query;
    float query_weight = 1.0f;
    float rescore_weight = 1.0f;
    RescoreMode rescore_mode = RescoreMode::Total;
    size_t window_size = 10;
};

class QueryRescorer {
public:
    void rescore(GpuIndexSearcher& searcher, const RescoreRequest& req, TopDocs& top_docs) const {
        if (!req.query) throw IllegalArgument("RescoreRequest without a query");
        const uint32_t window = (uint32_t)std::min<size_t>(req.window_size, 0xffffffffu);
        searcher.rescore_top_docs(*req.query, window, req.query_weight, req.rescore_weight,
                                  (uint32_t)req.rescore_mode, top_docs);
    }
};

}  // namespace rucene
