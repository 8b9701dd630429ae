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
// (paths relative to src/core/ of zhihu/rucene).  Header-only; link librucene_gpu.so.
#pragma once
#include <cstdint>
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

    // IndexSearcher::search(&query, &mut collector)
    void search(const Query& query, TopDocsCollector& collector) {
        std::vector<rg_clause> clauses;
        rg_query q = compile(query, clauses);
        const uint32_t k = (uint32_t)collector.estimated_hits();
        std::vector<rg_hit> hits(k);
        uint32_t count = 0;
        uint64_t total = 0;
        rg_search_params p{k, sim_.k1, RG_MODE_SEARCH, 0};
        check(rg_search_batch(engine_, &q, 1, clauses.data(), (uint32_t)clauses.size(), &p, hits.data(), &count, &total));
        std::vector<ScoreDoc> docs(count);
        for (uint32_t i = 0; i < count; i++) docs[i] = ScoreDoc{hits[i].doc, hits[i].score};
        collector.fill(TopDocs(total, std::move(docs)));
    }

    rg_engine* engine() { return engine_; }

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
    rg_query compile(const Query& query, std::vector<rg_clause>& clauses) const {
        rg_query q{};
        q.clause_begin = (uint32_t)clauses.size();
        if (auto tq = dynamic_cast<const TermQuery*>(&query)) {
            clauses.push_back(clause_of(*tq, RG_SHOULD));
            q.n_clauses = 1;
            return q;
        }
        if (auto cq = dynamic_cast<const ConstantScoreQuery*>(&query)) {  // the lone FILTER clause of build()
            auto tq = dynamic_cast<const TermQuery*>(cq->query.get());
            if (!tq || cq->boost != 0.0f) throw UnsupportedQuery("only ConstantScoreQuery(TermQuery, 0) is accelerated");
            clauses.push_back(clause_of(*tq, RG_FILTER));
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
            for (const QueryPtr& c : v) {
                auto tq = dynamic_cast<const TermQuery*>(c.get());
                if (!tq) throw UnsupportedQuery("only TermQuery leaves are accelerated");
                clauses.push_back(clause_of(*tq, occur));
            }
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
    BM25Similarity sim_;
    rg_engine* engine_ = nullptr;
    int32_t max_doc_ = 0;
    size_t stats_ = 0;
    float avgdl_ = 1.0f;
};

}  // namespace rucene
