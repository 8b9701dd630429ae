// search.cu — batch planning and the search entry points of include/rucene_gpu.h.
//
// Host side of IndexSearcher::search for a batch (search/searcher.rs:487-525): what
// BooleanQuery::build / BooleanWeight::create_scorer decide per (query, leaf)
// (search/query/boolean_query.rs:40-87,196-279) becomes a list of work items
// (query, segment, docid range) evaluated by k_eval_or / k_eval_and, followed by the exact
// TopDocsCollector replay.  Plan shapes outside the accelerated path return RG_EUNSUPPORTED so
// the caller can fall through to DefaultIndexSearcher, exactly like an unsupported Query would.
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>

#include "engine.hpp"

using namespace rg;

// A typed window into the batch's device slab.
template <class T>
struct Span {
    T* p = nullptr;
    size_t n = 0;
    size_t bytes() const { return n * sizeof(T); }
};

// The kernel routes of work items: each route is one launch list of rg_batch_run.
enum Route : uint32_t {
    kRouteOr,            // k_eval_or over block streams (any disjunction k_eval_or_ms and the decode-free one do not take)
    kRouteMs,            // k_eval_or_ms: plain sums with presence bitmaps; non-essential clauses are only counted
    kRouteLean,          // the decode-free k_eval_or: every clause a score column or a scored list
    kRouteDpq,           // k_eval_dpq: >= 10 clauses in the leaf (DisiPriorityQueue), one item per (query, leaf)
    kRouteAnd,           // k_eval_and: conjunctions
    kRouteReqOpt,        // k_eval_and<REQOPT>: MUST + SHOULD (ReqOptScorer)
    kRouteAndRanges,     // k_eval_and_ranges: conjunctions with a point-range clause
    kRouteReqOptRanges,
    kRouteAndNested,     // k_eval_and_nested: conjunctions with a group member (ranges or not)
    kRouteReqOptNested,
    kRoutes
};
// Routes whose items launch range-major (all first docid ranges, then all second ones, ...: see plan_batch); the
// others launch in item order (their items mostly cover a whole leaf: a ReqOptScorer's running mean, the
// DisiPriorityQueue).
constexpr bool kRouteByRank[kRoutes] = {true, true, true, false, true, false, true, false, true, false};

struct rg_batch {
    uint32_t n_queries = 0, k = 0, mode = 0;
    float k1 = 1.2f;
    uint32_t n_items = 0, n_groups = 0, n_leaves = 0;
    uint64_t generation = 0;  // engine->generation at prepare time
    // One device allocation per batch (cudaMalloc/cudaFree cost milliseconds each next to a
    // multi-GB index image; the engine keeps the last slab for the next batch).  Layout:
    // [plan arrays copied from the host][item_head: 0xff per run][everything zeroed per run].
    DevBuf<uint8_t> slab;
    Span<WorkItem> items;
    Span<ItemClause> clauses;
    Span<uint32_t> ids[kRoutes];     // the work items of each route, in launch order
    uint32_t n_ids[kRoutes] = {};
    uint32_t width[kRoutes] = {};    // widest item of k_eval_or / k_eval_dpq (clauses) and k_eval_or_ms (block streams)
    Span<uint4> local_lists;         // batch-local scored lists (choose_local_lists), built by rg_batch_prepare
    bool uses_planes = false;        // some column / bitmap reference of this batch carries tf-norm planes
    Span<ColRef> col_refs;           // score columns this batch reads (ItemClause.term_id indexes it)
    std::vector<std::shared_ptr<ColEntry>> cols;  // keeps them alive (the engine's LRU may drop them meanwhile)
    std::vector<std::shared_ptr<ColEntry>> lists; // scored posting lists this batch streams, likewise
    uint32_t n_cols_built = 0;       // columns materialised by this rg_batch_prepare (the others were cached)
    uint32_t n_lists_built = 0;
    uint64_t col_floats = 0, list_floats = 0;
    Span<uint32_t> group_item_begin, group_out;
    Span<uint32_t> item_head, item_matches, item_theta, item_topk_n;
    Span<float> item_topk;  // [n_items][kcap] (not zeroed: item_topk_n says what is valid)
    uint32_t topk_cap = 0;
    Span<uint2> deep_map;   // k > 1024 only: per query the (base, shift) of its theta bucket map (deep_bucket_maps)
    Span<unsigned long long> arena_next;  // [0] bump pointer, [1] error flag (as u32 view)
    Span<unsigned long long> dbg;         // RG_CFG_STATS counters (zeroed per run)
    Span<rg_hit> out_hits;
    Span<uint32_t> out_counts;
    Span<unsigned long long> out_total;
    Span<uint8_t> leaf_records;
    uint8_t* zero_begin = nullptr;
    size_t zero_bytes = 0;
    uint64_t postings = 0, algo_bytes = 0, h2d_bytes = 0;
    uint32_t kernels_per_run = 0;
    bool or_has_not = false, or_has_msm = false, or_has_dmax = false, or_nonpos = false;
    bool ran = false;
    bool local_built = false;  // batch-local scored lists were launched into the slab
    // two batches may be in flight (prepare the next while one runs): the plan goes up on the engine's copy stream,
    // the run waits for `uploaded`, the fetch waits for `done` on the copy stream; timing events are the batch's own
    cudaEvent_t uploaded = nullptr, done = nullptr, ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool synced = false;  // the host has waited for `done`
    DevBuf<uint8_t> rescore_plan;  // the last rg_batch_rescore's plan (read by its k_rescore)
    // point ranges: RangeRef per (leaf, range) and the range kernels' block counters (zeroed per run)
    Span<RangeRef> range_refs;
    Span<unsigned long long> range_stats;
    Span<unsigned long long> group_stats;  // group-lead counters of k_eval_and_nested (zeroed per run)
    ~rg_batch() {
        for (cudaEvent_t x : {uploaded, done, ev[0], ev[1], ev[2], ev[3]})
            if (x) cudaEventDestroy(x);
    }
};

namespace {

// RG_PLAN_TIMING=1: where rg_batch_prepare's host time goes, one line per call on stderr
struct PlanTimer {
    bool on = getenv("RG_PLAN_TIMING") != nullptr;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    std::string line;
    void mark(const char* what) {
        if (!on) return;
        const auto t1 = std::chrono::steady_clock::now();
        char buf[96];
        snprintf(buf, sizeof buf, " %s=%.2f", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
        line += buf;
        t0 = t1;
    }
    ~PlanTimer() {
        if (on && !line.empty()) fprintf(stderr, "[rg plan ms]%s\n", line.c_str());
    }
};

struct HostPlan {
    std::vector<WorkItem> items;
    std::vector<ItemClause> clauses;
    std::vector<uint32_t> ids[kRoutes];   // the work items of each route
    std::vector<uint32_t> rank[kRoutes];  // kRouteByRank routes: the launch-order key of each id
    uint32_t width[kRoutes] = {};
    std::vector<RangeRef> range_refs;     // point ranges: RangeRef per (leaf, range)
    // batch-local scored lists: build jobs whose dst is an offset (in floats) into the batch's list region, and the
    // col_refs entries to point there once the slab exists
    std::vector<ColumnJob> local_jobs;
    std::vector<std::pair<uint32_t, uint64_t>> local_refs;  // (col_refs index, offset in floats)
    uint64_t local_floats = 0;
    uint32_t local_units = 0;
    std::vector<ColRef> col_refs;
    std::map<std::tuple<uint32_t, uint32_t, uint32_t>, uint32_t> bitmap_refs;  // (leaf, term, cache) -> col_refs entry {null, bits, hi}
    std::vector<std::shared_ptr<ColEntry>> cols, lists;
    uint32_t n_cols_built = 0, n_lists_built = 0;
    uint64_t col_floats = 0, list_floats = 0;
    std::vector<uint32_t> group_item_begin, group_out;
    uint64_t postings = 0, algo_bytes = 0;
    bool or_has_not = false, or_has_msm = false, or_has_dmax = false, or_nonpos = false;
    // back to the empty plan, keeping the vectors' storage (a plan is tens of MB: fresh vectors would be page-faulted
    // in by every rg_batch_prepare)
    void reset() {
        items.clear(); clauses.clear(); local_jobs.clear(); local_refs.clear(); range_refs.clear();
        for (uint32_t r = 0; r < kRoutes; r++) {
            ids[r].clear();
            rank[r].clear();
            width[r] = 0;
        }
        local_floats = 0;
        local_units = 0;
        col_refs.clear(); bitmap_refs.clear(); cols.clear(); lists.clear();
        group_item_begin.clear(); group_out.clear();
        n_cols_built = n_lists_built = 0;
        col_floats = list_floats = postings = algo_bytes = 0;
        or_has_not = or_has_msm = or_has_dmax = or_nonpos = false;
    }
};
// the engine keeps one of these between calls (rg_engine::plan_scratch)
struct PlanScratch {
    HostPlan hp;
    std::vector<HostPlan> parts;
    std::vector<uint32_t> sort_tmp;
};

struct QShape {
    int type = -1;  // kTypeOr / kTypeAnd
    std::vector<uint32_t> clause_idx;  // scoring clauses (indices into the caller's array), evaluation order
    std::vector<uint32_t> not_idx;     // MUST_NOT clauses (ReqNotScorer)
    uint32_t msm = 0;                  // min_should_match when > 1 on a pure-SHOULD shape, else 0
    bool dismax = false;               // DisjunctionMaxQuery: score = max + (sum - max) * tie
    float tie = 0.0f;
    std::vector<uint32_t> opt_idx;     // SHOULD clauses beside a MUST (ReqOptScorer's optional side), clause order
    bool match_all = false;            // only MUST_NOT clauses: BooleanQuery::build adds MatchAllDocsQuery (score 0)
    // point ranges (RG_CLAUSE_RANGE, only from the *_ranges entry points): required (MUST / FILTER, or the one clause
    // a query collapses to) and MUST_NOT ones.  A shape with ranges is always kTypeAnd or kTypeReqOpt.
    std::vector<uint32_t> req_rng, not_rng;
    // What a kTypeAnd / kTypeReqOpt shape is planned from: the required side (MUST then FILTER) and the optional side,
    // in clause order, terms and nested groups (RG_CLAUSE_GROUP, only from the *_nested entry points) mixed.
    // clause_idx / opt_idx list the terms among them (columns are chosen from those); not_idx holds MUST_NOT groups
    // flattened.
    struct Entry {
        uint32_t begin, n;  // its clauses [begin, begin + n): a term's one clause, or a group's members
        bool group;
        bool filter;        // a FILTER group: needs_scores = false, it scores exactly 0.0f
    };
    std::vector<Entry> req_seq, opt_seq;
    // a shape without groups: every required / optional clause is a term entry
    void term_entries() {
        for (uint32_t ci : clause_idx) req_seq.push_back(Entry{ci, 1, false, false});
        for (uint32_t ci : opt_idx) opt_seq.push_back(Entry{ci, 1, false, false});
    }
};

// MUST_NOT clauses never score, but the kernels still form cache pointers from the id
void check_caches(const QShape& s, const rg_clause* clauses, uint32_t n_caches) {
    for (const auto* idx : {&s.clause_idx, &s.opt_idx, &s.not_idx})
        for (uint32_t ci : *idx)
            if (clauses[ci].cache_id >= n_caches) throw ArgError("clause refers to an unset norm cache");
}

inline bool is_range_clause(const rg_clause& c, const rg_point_range* ranges) {
    return ranges && (c.occur & RG_CLAUSE_RANGE);
}

void check_range_clause(const rg_clause& c, const rg_point_range* ranges, uint32_t n_ranges) {
    if (c.term_id >= n_ranges) throw ArgError("range clause: term_id outside the range array");
    const rg_point_range& r = ranges[c.term_id];
    if (r.bytes_per_dim != 4 && r.bytes_per_dim != 8) throw ArgError("range: bytes_per_dim must be 4 or 8");
    uint32_t wbits;
    memcpy(&wbits, &c.weight, 4);
    if (wbits != 0u) throw Unsupported("a boosted PointRangeQuery (weight != +0.0f)");
}

// BooleanQuery::build with PointRangeQuery clauses.  A PointRangeWeight scores 0f32 (its weight is only set by
// normalize(), which the searcher never calls), so a range is a docid predicate that adds +0.0f: in a conjunction
// ConjunctionScorer's cost order decides nothing (x + 0.0f == x for every x except -0.0f, which becomes +0.0f
// wherever the addition happens), and on the required side of a ReqOptScorer made of ranges only the running mean
// stays 0 and never skips.  Shapes outside that (a range on a disjunction, in a dismax, beside only MUST_NOT
// clauses) are refused.  Returns false when the query has no range clause (the term-only classify applies).
bool classify_ranges(const rg_query& q, const rg_clause* clauses, const rg_point_range* ranges, uint32_t n_ranges,
                     QShape& s) {
    bool any = false;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const rg_clause& c = clauses[q.clause_begin + i];
        if (!is_range_clause(c, ranges)) continue;
        any = true;
        check_range_clause(c, ranges, n_ranges);
    }
    if (!any) return false;
    if (q.flags & RG_Q_DISMAX) throw Unsupported("a PointRangeQuery in a DisjunctionMaxQuery");
    if (!(q.flags & RG_Q_BOOLEAN)) {
        if (q.n_clauses != 1) throw ArgError("a bare query has exactly one clause");
        s.type = kTypeAnd;
        s.req_rng.push_back(q.clause_begin);
        return true;
    }
    if (q.n_clauses > (uint32_t)kMaxTerms) throw Unsupported("more than 9 clauses with a PointRangeQuery");
    std::vector<uint32_t> musts, shoulds, must_nots, should_rng;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const uint32_t ci = q.clause_begin + i;
        const rg_clause& c = clauses[ci];
        const bool rng = is_range_clause(c, ranges);
        const int32_t occ = rng ? (c.occur & ~RG_CLAUSE_RANGE) : c.occur;
        if (occ == RG_MUST || occ == RG_FILTER) (rng ? s.req_rng : musts).push_back(ci);
        else if (occ == RG_SHOULD) (rng ? should_rng : shoulds).push_back(ci);
        else if (occ == RG_MUST_NOT) (rng ? s.not_rng : must_nots).push_back(ci);
        else throw ArgError("unknown occur");
    }
    // FILTER terms follow the MUST terms (must_weights, :96-125): keep that order among the terms
    std::vector<uint32_t> req_terms;
    for (uint32_t ci : musts)
        if (clauses[ci].occur == RG_MUST) req_terms.push_back(ci);
    for (uint32_t ci : musts)
        if (clauses[ci].occur == RG_FILTER) req_terms.push_back(ci);
    const size_t n_pos = req_terms.size() + s.req_rng.size() + shoulds.size() + should_rng.size();
    if (must_nots.empty() && s.not_rng.empty() && n_pos == 1) {  // collapses to the one range (:66-75)
        s.type = kTypeAnd;
        if (s.req_rng.empty()) s.req_rng = should_rng;
        return true;
    }
    if (req_terms.empty() && s.req_rng.empty())
        throw Unsupported("a PointRangeQuery on a disjunction or beside only MUST_NOT clauses");
    if (!should_rng.empty()) throw Unsupported("a SHOULD PointRangeQuery beside a required clause");
    s.type = shoulds.empty() ? kTypeAnd : kTypeReqOpt;
    s.clause_idx = req_terms;
    s.opt_idx = shoulds;
    s.not_idx = must_nots;
    s.term_entries();
    return true;
}

// what a clause scores with: a FILTER clause is a required clause with NonScoringSimilarity, i.e. exactly 0f32
// (= BM25 with weight +0: 0 * (k1+1) * f / (f + norm) = +0 for any finite norm)
inline float clause_weight(const rg_clause& c) { return c.occur == RG_FILTER ? 0.0f : c.weight; }

// BooleanQuery::build + BooleanWeight::create_scorer wiring for the accelerated shapes.  rescore: the shape is a
// rescoring query (rg_batch_rescore), scored through advance() only: shapes whose scorer is a DisiPriorityQueue are
// refused (its f32 summation order depends on the heap's history), and a pure SHOULD query with
// min_should_match > 1 (SimpleQueue at any width) is taken up to kDpqMaxTerms clauses.
QShape classify(const rg_query& q, const rg_clause* clauses, uint32_t n_clauses_total, bool rescore = false) {
    if ((uint64_t)q.clause_begin + q.n_clauses > n_clauses_total) throw ArgError("query clause range out of bounds");
    QShape s;
    if (q.flags & RG_Q_DISMAX) {
        // DisjunctionMaxQuery::build (search/query/disjunction_max_query.rs:51-68) over TermQuerys;
        // DisjunctionMaxScorer::new (disjunction_scorer.rs:118-139): SimpleQueue below 10 disjuncts
        if (q.n_clauses == 0) throw ArgError("DisjunctionMaxQuery: sub query should not be empty!");
        if (q.n_clauses > (uint32_t)kDpqMaxTerms) throw Unsupported("more than 32 disjuncts");
        if (rescore && q.n_clauses > (uint32_t)kMaxTerms)
            throw Unsupported("rescoring with a DisjunctionMaxQuery of 10 or more disjuncts (DisiPriorityQueue order)");
        s.type = kTypeOr;
        for (uint32_t i = 0; i < q.n_clauses; i++) s.clause_idx.push_back(q.clause_begin + i);
        if (q.n_clauses > 1) {  // a single disjunct is the disjunct itself
            s.dismax = true;
            memcpy(&s.tie, &q.min_should_match, 4);
        }
        return s;
    }
    if (!(q.flags & RG_Q_BOOLEAN)) {
        if (q.n_clauses != 1) throw ArgError("a bare TermQuery has exactly one clause");
        s.type = kTypeOr;  // TermScorer == one-clause disjunction: 0.0f + s == s
        s.clause_idx.push_back(q.clause_begin);
        return s;
    }
    std::vector<uint32_t> musts, shoulds, filters, must_nots;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const rg_clause& c = clauses[q.clause_begin + i];
        if (c.occur == RG_MUST) musts.push_back(q.clause_begin + i);
        else if (c.occur == RG_SHOULD) shoulds.push_back(q.clause_begin + i);
        else if (c.occur == RG_MUST_NOT) must_nots.push_back(q.clause_begin + i);
        else if (c.occur == RG_FILTER) filters.push_back(q.clause_begin + i);
        else throw ArgError("unknown occur");
    }
    int32_t msm = q.min_should_match > 0 ? q.min_should_match : (musts.empty() ? 1 : 0);
    if (musts.size() + shoulds.size() + filters.size() + must_nots.size() == 0)
        throw ArgError("boolean query should at least contain one inner query!");
    // up to 9 clauses of any mix; wider queries only as pure SHOULD disjunctions (DisiPriorityQueue kernel)
    const size_t n_all = musts.size() + shoulds.size() + filters.size() + must_nots.size();
    if (n_all > (size_t)kMaxTerms) {
        const bool pure_should = musts.empty() && filters.empty() && must_nots.empty();
        if (rescore) {
            if (!pure_should || n_all > (size_t)kDpqMaxTerms)
                throw Unsupported("more than 9 clauses (only pure SHOULD disjunctions of up to 32 clauses go wider)");
            if (msm <= 1)
                throw Unsupported("rescoring with a disjunction of 10 or more clauses and min_should_match <= 1 (DisiPriorityQueue order)");
        } else if (!pure_should || n_all > (size_t)kDpqMaxTerms || msm > 1) {
            throw Unsupported("more than 9 clauses (only pure SHOULD disjunctions of up to 32 clauses with min_should_match <= 1 go wider)");
        }
    }
    // BooleanQuery::create_weight (:96-125): must_weights = the MUST clauses, then the FILTER clauses
    // (needs_scores = false); BooleanWeight::create_scorer treats them alike from there on
    musts.insert(musts.end(), filters.begin(), filters.end());
    if (musts.empty() && shoulds.empty()) {
        // only MUST_NOT clauses (:76-79): musts.push(MatchAllDocsQuery) -> ReqNotScorer(all docs with score 0, ...)
        s.type = kTypeOr;
        s.match_all = true;
        s.not_idx = must_nots;
        return s;
    }
    // BooleanWeight::create_scorer (:253-278): ReqNotScorer(must | should, must_not); the excluded
    // set is the union of the MUST_NOT clauses (DisjunctionSumScorer with needs_scores = false)
    s.not_idx = must_nots;
    if (must_nots.empty() && musts.size() + shoulds.size() == 1) {  // collapses to the clause (:66-75)
        s.type = kTypeOr;
        s.clause_idx = musts.empty() ? shoulds : musts;
        return s;
    }
    if (!musts.empty()) {
        // one MUST + MUST_NOTs also takes the lead-list kernel; SHOULDs beside a MUST are the
        // optional side of a ReqOptScorer (:253-262) — per leaf, if any of them exists there
        s.type = shoulds.empty() ? kTypeAnd : kTypeReqOpt;
        s.clause_idx = musts;
        s.opt_idx = shoulds;
        s.term_entries();
        return s;
    }
    s.type = kTypeOr;
    s.clause_idx = shoulds;
    // min_should_match > 1 only ever filters a disjunction that is iterated with next(): the
    // top-level SHOULD side.  Beside a MUST it sits behind ReqOptScorer::score -> advance(), which
    // does not look at it (disjunction_scorer.rs:350-363), so those shapes ignore it above.
    s.msm = msm > 1 ? (uint32_t)msm : 0u;
    if (s.msm > 15u && !rescore) throw Unsupported("min_should_match > 15");
    return s;
}

// BooleanQuery::build with groups: pure-SHOULD BooleanQuerys of TermQuerys as clauses (RG_CLAUSE_GROUP).  `ext` is
// the planner's copy of the clause array; clauses the collapses make (a one-member group as its term under the
// group's occur, a lone FILTER group's members as FILTER terms) are appended to it.  Returns false when the query has
// no group clause.
//   - A group of one clause is that clause (build, :66-75); a query whose only positive clause is a group and that has
//     no MUST_NOT clause is the group: a disjunction.  `+(a | b) -c` is ReqNotScorer(DSS(a, b), c), the tree of the
//     disjunction `a b -c`, and runs there too.
//   - MUST_NOT groups are flattened into MUST_NOT terms: ReqNotScorer only calls advance() and doc_id() on its
//     excluded side (req_not_scorer.rs:46-118), and a DisjunctionSumScorer's advance() never looks at
//     min_should_match (disjunction_scorer.rs:350-364), so excluding (a | b) is excluding a and excluding b.
//   - Everything else needs a MUST / FILTER clause: a conjunction, or the required side of a ReqOptScorer.
bool classify_groups(const rg_query& q, std::vector<rg_clause>& ext, uint32_t n_clauses, const rg_point_range* ranges,
                     uint32_t n_ranges, const rg_query* groups, uint32_t n_groups, uint32_t n_caches, QShape& s) {
    bool any = false;
    for (uint32_t i = 0; i < q.n_clauses; i++) any = any || (ext[q.clause_begin + i].occur & RG_CLAUSE_GROUP) != 0;
    if (!any) return false;
    if (q.flags & RG_Q_DISMAX) throw Unsupported("a group in a DisjunctionMaxQuery");
    if (!(q.flags & RG_Q_BOOLEAN) && q.n_clauses != 1) throw ArgError("a bare query has exactly one clause");
    // member ranges: inside the array, apart from the query's own clauses and from the query's other groups
    std::vector<std::pair<uint32_t, uint32_t>> spans{{q.clause_begin, q.clause_begin + q.n_clauses}};
    std::vector<uint32_t> seen;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const rg_clause& c = ext[q.clause_begin + i];
        if (!(c.occur & RG_CLAUSE_GROUP)) continue;
        if (c.occur & RG_CLAUSE_RANGE) throw ArgError("unknown occur");
        if (c.term_id >= n_groups) throw ArgError("group clause: term_id outside the group array");
        if (std::find(seen.begin(), seen.end(), c.term_id) != seen.end()) continue;
        seen.push_back(c.term_id);
        const rg_query& g = groups[c.term_id];
        if ((uint64_t)g.clause_begin + g.n_clauses > n_clauses) throw ArgError("group clause range out of bounds");
        for (const auto& sp : spans)
            if (g.clause_begin < sp.second && sp.first < g.clause_begin + g.n_clauses)
                throw ArgError("group clause range overlaps the query's clauses or another group");
        spans.emplace_back(g.clause_begin, g.clause_begin + g.n_clauses);
        if (g.flags & RG_Q_DISMAX) throw Unsupported("a DisjunctionMaxQuery inside a BooleanQuery");
        if (!(g.flags & RG_Q_BOOLEAN)) throw ArgError("a group is a BooleanQuery (RG_Q_BOOLEAN)");
        if (g.n_clauses == 0) throw ArgError("boolean query should at least contain one inner query!");
        if (g.min_should_match > 1) throw Unsupported("a group with min_should_match > 1");
        for (uint32_t j = 0; j < g.n_clauses; j++) {
            const rg_clause& m = ext[g.clause_begin + j];
            if (m.occur & RG_CLAUSE_GROUP) throw Unsupported("a group inside a group");
            if (m.occur & RG_CLAUSE_RANGE) throw Unsupported("a PointRangeQuery inside a group");
            if (m.occur == RG_MUST || m.occur == RG_FILTER || m.occur == RG_MUST_NOT)
                throw Unsupported("a group member that is not a SHOULD TermQuery");
            if (m.occur != RG_SHOULD) throw ArgError("unknown occur");
            if (m.cache_id >= n_caches) throw ArgError("clause refers to an unset norm cache");
        }
    }
    using Entry = QShape::Entry;
    std::vector<Entry> musts, filters, shoulds;
    std::vector<uint32_t> nots, should_rng;
    size_t n_flat = 0;  // clauses of an item after flattening
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const uint32_t ci = q.clause_begin + i;
        const rg_clause c = ext[ci];
        const bool grp = (c.occur & RG_CLAUSE_GROUP) != 0;
        const bool rng = !grp && ranges && (c.occur & RG_CLAUSE_RANGE);
        const int32_t occ = c.occur & ~(RG_CLAUSE_GROUP | (rng ? RG_CLAUSE_RANGE : 0));
        if (occ != RG_MUST && occ != RG_SHOULD && occ != RG_MUST_NOT && occ != RG_FILTER) throw ArgError("unknown occur");
        if (rng) {
            check_range_clause(c, ranges, n_ranges);
            n_flat++;
            (occ == RG_MUST_NOT ? s.not_rng : occ == RG_SHOULD ? should_rng : s.req_rng).push_back(ci);
            continue;
        }
        Entry e{ci, 1, false, false};
        if (grp) {
            const rg_query& g = groups[c.term_id];
            if (g.n_clauses == 1) {  // a group of one clause is that clause
                const rg_clause& m = ext[g.clause_begin];
                e.begin = (uint32_t)ext.size();
                ext.push_back(rg_clause{occ, m.term_id, m.weight, m.cache_id});
            } else {
                e = Entry{g.clause_begin, g.n_clauses, true, occ == RG_FILTER};
            }
        }
        n_flat += e.n;
        if (occ == RG_MUST_NOT) {
            for (uint32_t j = 0; j < e.n; j++) nots.push_back(e.begin + j);
        } else {
            (occ == RG_MUST ? musts : occ == RG_FILTER ? filters : shoulds).push_back(e);
        }
    }
    auto lone_group = [&](const Entry& e) {  // the query is the group: a disjunction of its members
        if (e.n > (uint32_t)kDpqMaxTerms || (e.n + nots.size() > (size_t)kMaxTerms && !nots.empty()))
            throw Unsupported("more than 9 clauses (only pure SHOULD disjunctions of up to 32 clauses go wider)");
        s.type = kTypeOr;
        for (uint32_t j = 0; j < e.n; j++) {
            if (e.filter) {  // ConstantScoreQuery(.., 0) of the group: members that score 0
                const rg_clause& m = ext[e.begin + j];
                s.clause_idx.push_back((uint32_t)ext.size());
                ext.push_back(rg_clause{RG_FILTER, m.term_id, 0.0f, m.cache_id});
            } else {
                s.clause_idx.push_back(e.begin + j);
            }
        }
    };
    const size_t n_pos = musts.size() + filters.size() + shoulds.size() + s.req_rng.size() + should_rng.size();
    if (n_pos == 0 && !s.req_rng.empty()) throw ArgError("internal: range bookkeeping");
    if (nots.empty() && s.not_rng.empty() && n_pos == 1) {  // collapses to the one positive clause (:66-75)
        if (!s.req_rng.empty() || !should_rng.empty()) {
            s.type = kTypeAnd;
            if (s.req_rng.empty()) s.req_rng = should_rng;
            return true;
        }
        const Entry& e = !musts.empty() ? musts[0] : !filters.empty() ? filters[0] : shoulds[0];
        if (e.group) {
            lone_group(e);
        } else {
            s.type = kTypeOr;
            s.clause_idx.push_back(e.begin);
        }
        return true;
    }
    if (n_flat > (size_t)kMaxTerms) throw Unsupported("more than 9 clauses after flattening the groups");
    if (n_pos == 0) {  // only MUST_NOT clauses: MatchAllDocsQuery beside them (:76-79)
        if (!s.not_rng.empty()) throw Unsupported("a PointRangeQuery on a disjunction or beside only MUST_NOT clauses");
        s.type = kTypeOr;
        s.match_all = true;
        s.not_idx = nots;
        return true;
    }
    if (musts.empty() && filters.empty() && s.req_rng.empty())
        throw Unsupported("a group in a disjunction (no MUST / FILTER clause)");
    if (!should_rng.empty()) throw Unsupported("a SHOULD PointRangeQuery beside a required clause");
    if (musts.size() == 1 && musts[0].group && filters.empty() && shoulds.empty() && s.req_rng.empty() &&
        s.not_rng.empty()) {
        lone_group(musts[0]);  // ReqNotScorer(DSS(members), MUST_NOT side)
        s.not_idx = nots;
        return true;
    }
    s.type = shoulds.empty() ? kTypeAnd : kTypeReqOpt;
    s.req_seq = musts;
    s.req_seq.insert(s.req_seq.end(), filters.begin(), filters.end());
    s.opt_seq = shoulds;
    for (const Entry& e : s.req_seq)
        if (!e.group) s.clause_idx.push_back(e.begin);
    for (const Entry& e : s.opt_seq)
        if (!e.group) s.opt_idx.push_back(e.begin);
    s.not_idx = nots;
    return true;
}

// BooleanWeight::create_scorer / DisjunctionMaxWeight::create_scorer for one (query, leaf): which clauses of the
// shape have a scorer in the leaf.  present: the scoring clauses (a conjunction's required ones), a conjunction's
// stably sorted by cost() = doc_freq (ConjunctionScorer::new, :30); nots: the MUST_NOT clauses (:236-251); opts:
// the SHOULD clauses beside a MUST (:217-234).  False when the scorer is None: a required clause is absent
// (:201-206), no clause exists, or fewer SHOULD clauses than min_should_match exist.
bool resolve_leaf(const QShape& shape, const Segment& seg, const rg_clause* clauses, std::vector<uint32_t>& present,
                  std::vector<uint32_t>& nots, std::vector<uint32_t>& opts) {
    present.clear();
    nots.clear();
    opts.clear();
    bool dead = false;
    for (uint32_t ci : shape.clause_idx) {
        const uint32_t t = clauses[ci].term_id;
        const int32_t df = t < seg.host_terms.size() ? seg.host_terms[t].doc_freq : 0;
        if (df > 0) present.push_back(ci);
        else if (shape.type != kTypeOr) dead = true;  // create_scorer -> None (:201-206)
    }
    if (dead || (present.empty() && !shape.match_all && shape.req_rng.empty())) return false;
    if (shape.type == kTypeOr && shape.msm > present.size()) return false;  // nothing can reach msm here
    for (uint32_t ci : shape.not_idx) {
        const uint32_t t = clauses[ci].term_id;
        if (t < seg.host_terms.size() && seg.host_terms[t].doc_freq > 0) nots.push_back(ci);
    }
    for (uint32_t ci : shape.opt_idx) {
        const uint32_t t = clauses[ci].term_id;
        if (t < seg.host_terms.size() && seg.host_terms[t].doc_freq > 0) opts.push_back(ci);
    }
    if (shape.type != kTypeOr) {
        // ConjunctionScorer::new: stable sort by cost() = doc_freq (:30)
        std::stable_sort(present.begin(), present.end(), [&](uint32_t a, uint32_t b) {
            return seg.host_terms[clauses[a].term_id].doc_freq < seg.host_terms[clauses[b].term_id].doc_freq;
        });
    }
    return true;
}

const PointField* point_field(const Segment& seg, const rg_point_range& r) {
    const auto it = seg.points.find(r.field);
    if (it == seg.points.end()) return nullptr;
    if (it->second.bytes_per_dim != r.bytes_per_dim)
        throw ArgError("range: the field was uploaded with another bytes_per_dim");  // as PointRangeWeight bails
    return &it->second;
}

uint64_t be_key(const uint8_t* b, uint32_t n) {
    uint64_t v = 0;
    for (uint32_t j = 0; j < n; j++) v = v << 8 | b[j];
    return v;
}

// PointRangeWeight::create_scorer per leaf: None when the leaf has no points of the field.  req: the required ranges
// with their point counts in the leaf (a required range with no points, or none inside it, leaves the leaf without a
// match: false); nots: the MUST_NOT ranges that can exclude something.
bool resolve_ranges(const QShape& shape, const Segment& seg, const rg_clause* clauses, const rg_point_range* ranges,
                    std::vector<std::pair<uint64_t, uint32_t>>& req, std::vector<uint32_t>& nots) {
    req.clear();
    nots.clear();
    for (uint32_t ci : shape.req_rng) {
        const rg_point_range& r = ranges[clauses[ci].term_id];
        const PointField* pf = point_field(seg, r);
        const uint64_t n = pf ? pf->count(be_key(r.lower, r.bytes_per_dim), be_key(r.upper, r.bytes_per_dim)) : 0;
        if (n == 0) return false;
        req.emplace_back(n, ci);
    }
    for (uint32_t ci : shape.not_rng) {
        const rg_point_range& r = ranges[clauses[ci].term_id];
        const PointField* pf = point_field(seg, r);
        if (pf && pf->count(be_key(r.lower, r.bytes_per_dim), be_key(r.upper, r.bytes_per_dim))) nots.push_back(ci);
    }
    std::stable_sort(req.begin(), req.end(),
                     [](const std::pair<uint64_t, uint32_t>& a, const std::pair<uint64_t, uint32_t>& b) { return a.first < b.first; });
    return true;
}

// BooleanWeight::create_scorer of a conjunction / ReqOpt shape (kTypeAnd / kTypeReqOpt) in one leaf, for the first pass
// (plan_batch) and rescoring (plan_rescore) alike.  A term's cost() is its doc_freq.  A group is a
// DisjunctionSumScorer over its members present here (even over one: the `1 =>` arm is commented out,
// boolean_query.rs:196-279), None when it has none; its cost() is the sum of those members' doc_freq
// (disjunction_scorer.rs:39).  A required clause that is None leaves the leaf without a scorer (:201-206), an optional
// one is left out (:217-234).  MUST_NOT groups arrive flattened (classify_groups).
struct ConjLeaf {
    // a required / optional clause in this leaf: its clauses here are members[begin, begin + n)
    struct Req {
        uint64_t cost;
        uint32_t begin, n;
        bool group, filter;
    };
    std::vector<Req> req, opt;    // req: ConjunctionScorer's cost order (stable); opt: clause order
    std::vector<uint32_t> members, nots, rnots;  // nots: MUST_NOT terms present here; rnots: MUST_NOT ranges
    std::vector<std::pair<uint64_t, uint32_t>> rreq;  // required ranges with their point counts, cheapest first
    bool range_lead = false;      // a range leads (cheaper than every term and group)
    uint32_t leaf_type = 0;       // kTypeReqOpt only when some optional clause has a scorer here
    uint64_t cost = 0;            // the lead's

    // false: the leaf has no scorer
    bool resolve(const QShape& shape, const Segment& seg, const rg_clause* clauses, const rg_point_range* ranges) {
        auto df_of = [&](uint32_t ci) -> uint64_t {
            const uint32_t t = clauses[ci].term_id;
            return t < seg.host_terms.size() && seg.host_terms[t].doc_freq > 0 ? (uint64_t)seg.host_terms[t].doc_freq : 0;
        };
        auto entry = [&](const QShape::Entry& en) {
            Req r{0, (uint32_t)members.size(), 0, en.group, en.filter};
            for (uint32_t j = 0; j < en.n; j++)
                if (const uint64_t df = df_of(en.begin + j)) {
                    members.push_back(en.begin + j);
                    r.cost += df;
                }
            r.n = (uint32_t)members.size() - r.begin;
            return r;
        };
        req.clear();
        opt.clear();
        members.clear();
        nots.clear();
        rreq.clear();
        rnots.clear();
        bool dead = shape.req_seq.empty() && shape.req_rng.empty();
        for (const QShape::Entry& en : shape.req_seq) {
            req.push_back(entry(en));
            dead = dead || req.back().n == 0;
        }
        if (dead) return false;
        for (const QShape::Entry& en : shape.opt_seq) {
            const Req r = entry(en);
            if (r.n) opt.push_back(r);
        }
        for (uint32_t ci : shape.not_idx)
            if (df_of(ci)) nots.push_back(ci);
        // point ranges: the required ones with their point counts (cheapest first) and the MUST_NOT ones
        if ((!shape.req_rng.empty() || !shape.not_rng.empty()) && !resolve_ranges(shape, seg, clauses, ranges, rreq, rnots))
            return false;
        // ConjunctionScorer::new: stable sort by cost() (:30); the score is lead1 + lead2 + the others in that
        // order, each group one f32 value
        std::stable_sort(req.begin(), req.end(), [](const Req& a, const Req& b) { return a.cost < b.cost; });
        range_lead = !rreq.empty() && (req.empty() || rreq[0].first < req[0].cost);
        // no SHOULD scorer in this leaf -> the MUST side alone, no ReqOptScorer (:259-266)
        leaf_type = shape.type == kTypeReqOpt && opt.empty() ? (uint32_t)kTypeAnd : (uint32_t)shape.type;
        cost = range_lead ? rreq[0].first : req[0].cost;
        return true;
    }
};

// Score columns: which (leaf, term, weight, norm cache, k1) clauses of the batch's disjunctions are read
// from a materialised f32 column (k_build_columns) instead of their block stream.  Only terms with a
// presence bitmap (df >= max_doc/64, chosen at upload) qualify.  Columns are persistent: a key that is
// already in the engine's cache is used as is; a new one is built when at least two clauses of the
// batch share it (RG_CFG_EAGER_COLUMNS: one), most valuable (uses x df) first, evicting least recently
// used columns no batch references while over the HBM budget.  RG_CFG_NO_COLUMNS turns the feature off.
constexpr uint32_t kMatchAllTerm = 0xffffffffu;  // ColKey term of a leaf's MatchAllDocsQuery column

// the score column / scored list of a clause in leaf si
ColKey col_key(uint32_t si, const rg_clause& c, uint32_t k1bits) {
    const float w = clause_weight(c);
    uint32_t wbits;
    memcpy(&wbits, &w, 4);
    return ColKey(si, c.term_id, wbits, c.cache_id, k1bits);
}

// the col_refs entry of a clause's score column in leaf si, -1: none
int64_t col_of(const std::map<ColKey, uint32_t>& columns, uint32_t si, const rg_clause& c, uint32_t k1bits) {
    if (columns.empty()) return -1;
    const auto it = columns.find(col_key(si, c, k1bits));
    return it == columns.end() ? -1 : (int64_t)it->second;
}

// the build job of a column or list: its work units (blocks and tail) start at unit_begin of the launch
ColumnJob column_job(const ColKey& key, void* dst, uint32_t unit_begin) {
    ColumnJob job{};
    job.seg = std::get<0>(key);
    job.term_id = std::get<1>(key);
    const uint32_t wbits = std::get<2>(key);
    memcpy(&job.weight, &wbits, 4);
    job.cache_id = std::get<3>(key);
    job.dst = dst;
    job.unit_begin = unit_begin;
    return job;
}

// tf-norm planes of a bitmap term for one (norm cache, k1) — see TfPlanes: built for ALL bitmap terms of the leaf the
// first time a batch asks (a histogram pass over a sample of their blocks picks tau1/tau2, one more pass sets the
// bits), kept until the cache changes.  Fills ref.hi1/hi2/tau1/tau2; leaves them null when there is none (flag, no
// bitmap, no memory) — the kernel then bounds the clause by presence alone.
void tf_planes_of(rg_engine* e, uint32_t si, uint32_t term, uint32_t cache_id, float k1, ColRef& ref) {
    ref.hi1 = ref.hi2 = nullptr;
    ref.tau1 = ref.tau2 = 1.0f;
    if ((e->cfg.flags & (RG_CFG_TFPLANES | RG_CFG_MAXSCORE)) != (RG_CFG_TFPLANES | RG_CFG_MAXSCORE)) return;
    Segment& seg = e->segs[si];
    if (term >= seg.bitmap_slot.size() || seg.bitmap_slot[term] < 0) return;
    uint32_t k1bits;
    memcpy(&k1bits, &k1, 4);
    const auto key = std::make_pair(cache_id, k1bits);
    auto it = seg.tf_planes.find(key);
    const size_t n_bm = seg.bitmap_terms.size();
    const size_t stride = n_bm * seg.bitmap_words;
    if (it == seg.tf_planes.end()) {
        TfPlanes tp;
        if (cudaMalloc(reinterpret_cast<void**>(&tp.bits.p), 2 * stride * sizeof(uint32_t)) != cudaSuccess) {
            cudaGetLastError();
            tp.bits.p = nullptr;
            seg.tf_planes.emplace(key, std::move(tp));  // remembered as "none": do not retry every batch
            return;
        }
        tp.bits.n = 2 * stride;
        cudaStream_t st = e->stream;
        RG_CUDA_CHECK(cudaMemsetAsync(tp.bits.p, 0, tp.bits.bytes(), st));
        std::vector<ColumnJob> jobs(n_bm);
        uint32_t units = 0;
        for (size_t i = 0; i < n_bm; i++) {
            const uint32_t t = seg.bitmap_terms[i];
            jobs[i] = ColumnJob{si, t, cache_id, 1.0f, tp.bits.p + i * seg.bitmap_words, units, 0u};
            units += seg.host_terms[t].n_blocks + (seg.host_terms[t].tail_n ? 1u : 0u);
        }
        DevBuf<ColumnJob> d_jobs;
        DevBuf<uint32_t> d_hist;
        d_jobs.alloc(n_bm);
        d_hist.alloc(n_bm * 256);
        RG_CUDA_CHECK(cudaMemsetAsync(d_hist.p, 0, d_hist.bytes(), st));
        RG_CUDA_CHECK(cudaMemcpyAsync(d_jobs.p, jobs.data(), n_bm * sizeof(ColumnJob), cudaMemcpyHostToDevice, st));
        launch_build_tf_planes(st, e->d_segs.p, d_jobs.p, (uint32_t)n_bm, units, e->d_caches.p, k1, d_hist.p, 0);
        RG_CUDA_CHECK(cudaGetLastError());
        std::vector<uint32_t> hist(n_bm * 256);
        RG_CUDA_CHECK(cudaMemcpyAsync(hist.data(), d_hist.p, hist.size() * 4, cudaMemcpyDeviceToHost, st));
        RG_CUDA_CHECK(cudaStreamSynchronize(st));
        tp.tau1.assign(n_bm, 1.0f);
        tp.tau2.assign(n_bm, 1.0f);
        for (size_t i = 0; i < n_bm; i++) {  // 90th / 99th percentile bin edges of the sampled factor
            uint64_t total = 0, cum = 0;
            for (int b = 0; b < 256; b++) total += hist[i * 256 + b];
            bool have1 = false;
            for (int b = 0; b < 256 && total; b++) {
                cum += hist[i * 256 + b];
                if (!have1 && cum * 10 >= total * 9) {
                    tp.tau1[i] = (float)(b + 1) / 256.0f;
                    have1 = true;
                }
                if (cum * 100 >= total * 99) {
                    tp.tau2[i] = (float)(b + 1) / 256.0f;
                    break;
                }
            }
            uint32_t t2bits;
            memcpy(&t2bits, &tp.tau2[i], 4);
            jobs[i].weight = tp.tau1[i];
            jobs[i].pad = t2bits;
        }
        RG_CUDA_CHECK(cudaMemcpyAsync(d_jobs.p, jobs.data(), n_bm * sizeof(ColumnJob), cudaMemcpyHostToDevice, st));
        launch_build_tf_planes(st, e->d_segs.p, d_jobs.p, (uint32_t)n_bm, units, e->d_caches.p, k1, nullptr, stride);
        RG_CUDA_CHECK(cudaGetLastError());
        RG_CUDA_CHECK(cudaStreamSynchronize(st));
        e->launches += 2;
        it = seg.tf_planes.emplace(key, std::move(tp)).first;
    }
    if (!it->second.bits.p) return;
    const size_t slot = (size_t)seg.bitmap_slot[term];
    ref.hi1 = it->second.bits.p + slot * seg.bitmap_words;
    ref.hi2 = ref.hi1 + stride;
    ref.tau1 = it->second.tau1[slot];
    ref.tau2 = it->second.tau2[slot];
}

// Every BM25 contribution w*(k1+1)*f / (f + cache[norm]) of the clause is a finite-or-infinite f32 > 0 (no zero, no
// negative, no NaN): weight well inside the normal range, 0 <= k1 <= 1e6, the norm cache entries
// that norm bytes of the leaf select in [0, 1e10] (Segment::cache_small).  Score columns store
// +0.0f for "no posting", and the plain-sum disjunction kernel tells a match from its non-zero sum.
static bool scores_positive(const Segment& seg, float w, uint32_t cache_id, float k1) {
    return w >= 1e-20f && w <= 1e30f && k1 >= 0.0f && k1 <= 1e6f && cache_id < seg.cache_small.size() && seg.cache_small[cache_id];
}

static void ensure_budget(rg_engine* e) {
    if (e->col_budget_floats) return;  // once per index state (cudaMemGetInfo costs milliseconds)
    size_t free_b = 0, total_b = 0;
    RG_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    e->col_budget_floats = std::max<uint64_t>(1, ((uint64_t)free_b / sizeof(float) + e->col_floats) / 3);
}

// Job table of a column / list build: uploaded on the copy stream (the engine stream may be busy with a running
// batch) into one of four grow-only device tables; the build kernel is launched on the engine stream — ordered before
// the run of the batch being prepared — and the caller records list_jobs_done[slot] behind it, which is what the
// table's next reuse waits for.  No stream is synchronised beyond the copy itself.
static const ColumnJob* stage_jobs(rg_engine* e, const std::vector<ColumnJob>& jobs, uint32_t& slot) {
    slot = e->list_jobs_next;
    e->list_jobs_next = (e->list_jobs_next + 1u) & 3u;
    RG_CUDA_CHECK(cudaEventSynchronize(e->list_jobs_done[slot]));  // the build that last read this table has finished
    if (e->list_jobs[slot].n < jobs.size()) e->list_jobs[slot].alloc(jobs.size() + jobs.size() / 2 + 64);
    RG_CUDA_CHECK(cudaMemcpyAsync(e->list_jobs[slot].p, jobs.data(), jobs.size() * sizeof(ColumnJob), cudaMemcpyHostToDevice,
                                  e->copy_stream));
    RG_CUDA_CHECK(cudaStreamSynchronize(e->copy_stream));
    return e->list_jobs[slot].p;
}

// Drop the least recently used score columns no batch references until `len` more floats fit the column budget.
// (cudaFree synchronises, which also orders it after running kernels.)
static bool make_room(rg_engine* e, uint64_t len) {
    while (e->col_floats + len > e->col_budget_floats) {
        auto victim = e->col_cache.end();
        for (auto it = e->col_cache.begin(); it != e->col_cache.end(); ++it)
            if (it->second.use_count() == 1 && (victim == e->col_cache.end() || it->second->last_use < victim->second->last_use))
                victim = it;
        if (victim == e->col_cache.end()) return false;
        e->col_floats -= victim->second->len;
        e->col_cache.erase(victim);
    }
    return true;
}

// The scored lists' arena: one cudaMalloc at first need (a sixth of the free HBM, at most 24 GiB), used as a ring of
// slabs — one per rg_batch_prepare that built lists.  Space is reclaimed oldest slab first and only when no batch
// still references one of its lists; a list that is evicted while still popular is simply rebuilt by the next batch
// that shares it (one pass over its postings).  Returns the offset of `len` contiguous floats, or ~0 if there is none.
static uint64_t list_arena_alloc(rg_engine* e, uint64_t len) {
    constexpr uint64_t kNoRoom = ~0ull;
    if (!e->list_arena.p) {
        if (e->list_arena_tried) return kNoRoom;
        e->list_arena_tried = true;
        size_t free_b = 0, total_b = 0;
        RG_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
        uint64_t want = std::min<uint64_t>((uint64_t)free_b / 6, 24ull << 30) / sizeof(float);
        uint64_t least = 16ull << 20;
        if (const char* v = getenv("RG_LIST_ARENA_KB")) {  // tests: a small arena, so that the ring wraps and reclaims
            want = std::max<uint64_t>(64, strtoull(v, nullptr, 10)) * 1024 / sizeof(float);
            least = want;
        }
        for (; want >= least; want /= 2) {
            float* p = nullptr;
            if (cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(float)) == cudaSuccess) {
                e->list_arena.p = p;
                e->list_arena.n = want;
                break;
            }
            cudaGetLastError();
        }
        if (!e->list_arena.p) return kNoRoom;
    }
    const uint64_t size = e->list_arena.n;
    if (len > size / 2) return kNoRoom;
    auto evict_front = [&]() {
        auto& sl = e->list_slabs.front();
        auto cached = [&](const std::shared_ptr<ColEntry>& ent) {
            const auto it = e->list_cache.find(ent->key);
            return it != e->list_cache.end() && it->second == ent;
        };
        for (const auto& ent : sl.entries)
            if (ent.use_count() > (cached(ent) ? 2 : 1)) return false;  // a prepared batch still streams it
        for (const auto& ent : sl.entries)
            if (cached(ent)) {
                e->list_floats -= ent->len;
                e->list_cache.erase(ent->key);
            }
        e->list_slabs.pop_front();
        return true;
    };
    for (;;) {
        if (e->list_slabs.empty()) {
            e->list_head = 0;
            break;
        }
        const uint64_t tail = e->list_slabs.front().off, head = e->list_head;
        if (head > tail) {  // in use: [tail, head)
            if (size - head >= len) break;
            if (tail >= len) {  // wrap around; [head, size) stays unused until the ring comes round again
                e->list_head = 0;
                break;
            }
        } else if (tail - head >= len) {  // in use: [tail, end) and [0, head)
            break;
        }
        if (!evict_front()) return kNoRoom;
    }
    const uint64_t off = e->list_head;
    e->list_head += len;
    return off;
}

std::map<ColKey, uint32_t> choose_columns(rg_engine* e, const std::vector<QShape>& shapes, const rg_clause* clauses,
                                          float k1, HostPlan& hp, PlanTimer& tm) {
    std::map<ColKey, uint32_t> chosen;
    const bool cols_off = (e->cfg.flags & (RG_CFG_NO_COLUMNS | RG_CFG_NO_BITMAPS)) != 0;  // (a match-all column is not optional)
    const bool eager = (e->cfg.flags & RG_CFG_EAGER_COLUMNS) != 0;
    const uint32_t min_uses = eager ? 1u : 2u;
    uint32_t k1bits;
    memcpy(&k1bits, &k1, 4);
    std::unordered_map<ColKey, uint32_t, ColKeyHash> uses;
    bool any_match_all = false;
    for (const QShape& sh : shapes) {
        any_match_all = any_match_all || sh.match_all;
        if (cols_off) continue;
        for (uint32_t si = 0; si < e->segs.size(); si++) {
            const Segment& seg = e->segs[si];
            // a column pays where it is read: the exhaustive disjunction kernel scans it docid by docid (df >= max_doc/8),
            // k_eval_or_ms and the conjunction kernel gather single cells (df >= max_doc/64)
            auto count = [&](uint32_t ci, uint64_t den) {
                const rg_clause& c = clauses[ci];
                if (c.term_id >= seg.host_terms.size() || seg.bitmap_slot[c.term_id] < 0) return;
                if ((uint64_t)seg.host_terms[c.term_id].doc_freq * den < (uint64_t)seg.max_doc) return;
                if (!scores_positive(seg, clause_weight(c), c.cache_id, k1)) return;  // a column cell of +0.0f means "no posting"
                uses[col_key(si, c, k1bits)]++;
            };
            const uint64_t or_den = ((e->cfg.flags & RG_CFG_MAXSCORE) || eager) ? (uint64_t)kColumnDen : (uint64_t)e->or_col_den;
            for (uint32_t ci : sh.clause_idx) count(ci, sh.type == kTypeOr ? or_den : (uint64_t)kColumnDen);
            // conjunctions probe the columns of their non-lead clauses (which clause leads depends on the leaf;
            // the lead's use is counted too and simply stays unused)
            for (uint32_t ci : sh.opt_idx) count(ci, (uint64_t)kColumnDen);
        }
    }
    tm.mark("col_uses");
    if (uses.empty() && !any_match_all) return chosen;
    ensure_budget(e);
    tm.mark("col_budget");
    auto add_ref = [&](const ColKey& key, const std::shared_ptr<ColEntry>& ent) {
        ent->last_use = ++e->col_tick;
        chosen[key] = (uint32_t)hp.col_refs.size();
        ColRef ref{ent->col, ent->bits, nullptr, nullptr, 1.0f, 1.0f, e->column_sweep ? nullptr : ent->bmax};
        if (std::get<1>(key) != kMatchAllTerm) tf_planes_of(e, std::get<0>(key), std::get<1>(key), std::get<3>(key), k1, ref);
        hp.col_refs.push_back(ref);
        hp.cols.push_back(ent);
        hp.col_floats += ent->len;
    };
    std::vector<std::pair<uint64_t, ColKey>> to_build;
    for (const auto& kv : uses) {
        const auto it = e->col_cache.find(kv.first);
        if (it != e->col_cache.end()) {
            e->col_hits++;
            add_ref(kv.first, it->second);
        } else if (kv.second >= min_uses) {
            const Segment& seg = e->segs[std::get<0>(kv.first)];
            to_build.emplace_back((uint64_t)kv.second * (uint64_t)seg.host_terms[std::get<1>(kv.first)].doc_freq, kv.first);
        }
    }
    std::sort(to_build.begin(), to_build.end(), [](const auto& x, const auto& y) { return x.first != y.first ? x.first > y.first : x.second < y.second; });
    tm.mark("col_cached");
    std::vector<ColumnJob> jobs;
    std::vector<std::shared_ptr<ColEntry>> built;
    uint32_t n_units = 0;
    cudaStream_t st = e->stream;
    if (any_match_all) {
        // MatchAllDocsQuery (query/match_all_query.rs:28-116) as a column: every docid of the leaf, score 0f32
        for (uint32_t si = 0; si < e->segs.size(); si++) {
            const ColKey key(si, kMatchAllTerm, 0u, 0u, 0u);
            auto it = e->col_cache.find(key);
            if (it == e->col_cache.end()) {
                auto ent = std::make_shared<ColEntry>();
                ent->key = key;
                ent->len = ((uint64_t)e->segs[si].max_doc + 1024 + 3) & ~3ull;
                if (cudaMalloc(reinterpret_cast<void**>(&ent->col), ent->len * sizeof(float)) != cudaSuccess) {
                    cudaGetLastError();
                    ent->col = nullptr;
                    continue;
                }
                RG_CUDA_CHECK(cudaMemsetAsync(ent->col, 0, ent->len * sizeof(float), st));
                e->col_floats += ent->len;
                it = e->col_cache.emplace(key, ent).first;
            }
            add_ref(key, it->second);
        }
    }
    for (const auto& r : to_build) {
        if (hp.col_refs.size() >= 4096) break;
        const Segment& seg = e->segs[std::get<0>(r.second)];
        // windows read past max_doc; the block-maximum table follows the cells
        const uint64_t col_len = ((uint64_t)seg.max_doc + 1024 + kColBlk - 1) / kColBlk * kColBlk;
        const uint64_t len = col_len + ((col_len / kColBlk + 3) & ~3ull);
        if (!make_room(e, len)) break;
        auto ent = std::make_shared<ColEntry>();
        ent->key = r.second;
        ent->len = len;
        if (cudaMalloc(reinterpret_cast<void**>(&ent->col), len * sizeof(float)) != cudaSuccess) {
            cudaGetLastError();
            ent->col = nullptr;
            break;
        }
        const TermHost& th = seg.host_terms[std::get<1>(r.second)];
        ent->bits = seg.bitmaps.p + (size_t)seg.bitmap_slot[std::get<1>(r.second)] * seg.bitmap_words;
        ent->bmax = reinterpret_cast<uint32_t*>(ent->col + col_len);
        built.push_back(ent);
        RG_CUDA_CHECK(cudaMemsetAsync(ent->col, 0, len * sizeof(float), st));
        jobs.push_back(column_job(r.second, ent->col, n_units));
        n_units += th.n_blocks + (th.tail_n ? 1u : 0u);
        e->col_cache[r.second] = ent;
        e->col_floats += len;
        e->col_builds++;
        add_ref(r.second, ent);
    }
    tm.mark("col_alloc");
    if (!jobs.empty()) {
        uint32_t jb = 0;
        const ColumnJob* d_jobs = stage_jobs(e, jobs, jb);
        tm.mark("col_stage");
        launch_build_columns(st, e->d_segs.p, d_jobs, (uint32_t)jobs.size(), n_units, e->d_caches.p, k1);
        RG_CUDA_CHECK(cudaGetLastError());
        RG_CUDA_CHECK(cudaEventRecord(e->list_jobs_done[jb], st));
        e->launches++;
        for (const auto& ent : built) {
            launch_col_block_max(st, ent->col, ent->bmax, (uint32_t)((reinterpret_cast<float*>(ent->bmax) - ent->col) / kColBlk));
            RG_CUDA_CHECK(cudaGetLastError());
            e->launches++;
        }
        hp.n_cols_built = (uint32_t)jobs.size();
    }
    return chosen;
}

// Scored posting lists.  A disjunction clause that stays a block stream costs, per query that carries it: unpack the
// doc and freq blocks, a warp scan, one norm-byte gather + one cache load + one IEEE division per posting.  None of
// that depends on the query beyond (term, weight, norm cache, k1) — so a clause two queries of a batch share (or that
// an earlier batch left behind) is decoded and scored ONCE into (docid, f32 score) pairs, 1 KB per 128-posting block in
// block order, and k_eval_or streams those: two 16-byte loads per lane and block.  Exactly the values stream_refill
// would compute (same instructions, same order), so the results do not change.  8 bytes per posting: the whole
// 100 M-doc benchmark index would be 10.7 GB; they live in the engine's list arena (list_arena_alloc).
// RG_CFG_NO_LISTS turns the feature off.
constexpr uint32_t kListMinDf = 4096;  // shorter lists are a few blocks per query: not worth a cache entry (eager: 256)
std::map<ColKey, uint32_t> choose_lists(rg_engine* e, const std::vector<QShape>& shapes, const rg_clause* clauses, float k1,
                                        const std::map<ColKey, uint32_t>& columns, HostPlan& hp) {
    std::map<ColKey, uint32_t> chosen;
    if (e->cfg.flags & (RG_CFG_NO_LISTS | RG_CFG_MAXSCORE)) return chosen;  // (k_eval_or_ms seeks inside blocks: not wired)
    const bool eager = (e->cfg.flags & RG_CFG_EAGER_COLUMNS) != 0;
    const uint32_t min_uses = eager ? 1u : 2u;
    const uint64_t min_df = eager ? 256u : kListMinDf;
    uint32_t k1bits;
    memcpy(&k1bits, &k1, 4);
    std::unordered_map<ColKey, uint32_t, ColKeyHash> uses;
    for (const QShape& sh : shapes) {
        if (sh.type != kTypeOr || sh.match_all || sh.clause_idx.size() >= 10) continue;  // (>= 10: k_eval_dpq)
        for (uint32_t si = 0; si < e->segs.size(); si++) {
            const Segment& seg = e->segs[si];
            for (uint32_t ci : sh.clause_idx) {
                const rg_clause& c = clauses[ci];
                if (c.term_id >= seg.host_terms.size()) continue;
                const uint64_t df = (uint64_t)seg.host_terms[c.term_id].doc_freq;
                if (df < min_df) continue;
                const ColKey key = col_key(si, c, k1bits);
                if (df * e->or_col_den >= (uint64_t)seg.max_doc && columns.count(key)) continue;  // read from its score column
                uses[key]++;
            }
        }
    }
    if (uses.empty()) return chosen;
    auto add_ref = [&](const ColKey& key, const std::shared_ptr<ColEntry>& ent) {
        if (hp.col_refs.size() >= 65536) return;  // ItemClause.flags carries the reference in 16 bits
        ent->last_use = ++e->col_tick;
        chosen[key] = (uint32_t)hp.col_refs.size();
        hp.col_refs.push_back(ColRef{ent->col, nullptr, nullptr, nullptr, 1.0f, 1.0f});
        hp.lists.push_back(ent);
        hp.list_floats += ent->len;
    };
    std::vector<std::pair<uint64_t, ColKey>> to_build;
    for (const auto& kv : uses) {
        const auto it = e->list_cache.find(kv.first);
        if (it != e->list_cache.end()) {
            e->list_hits++;
            add_ref(kv.first, it->second);
        } else if (kv.second >= min_uses) {
            const Segment& seg = e->segs[std::get<0>(kv.first)];
            to_build.emplace_back((uint64_t)kv.second * (uint64_t)seg.host_terms[std::get<1>(kv.first)].doc_freq, kv.first);
        }
    }
    std::sort(to_build.begin(), to_build.end(), [](const auto& x, const auto& y) { return x.first != y.first ? x.first > y.first : x.second < y.second; });
    // one piece of the arena for everything this call builds
    struct Pick { ColKey key; uint64_t len, off; uint32_t units; };
    std::vector<Pick> picks;
    uint64_t total = 0, n_units64 = 0;
    const uint64_t room = e->list_arena.p ? e->list_arena.n / 2 : (e->list_arena_tried ? 0 : ~0ull);
    for (const auto& r : to_build) {
        if (hp.col_refs.size() + picks.size() >= 65536) break;
        const Segment& seg = e->segs[std::get<0>(r.second)];
        const TermHost& th = seg.host_terms[std::get<1>(r.second)];
        const uint32_t units = th.n_blocks + 1u;  // + the vint tail (or an unused unit the last block's prefetch may touch)
        const uint64_t len = (uint64_t)units * 256u;
        if (n_units64 + units > 0x7fffffffu) break;
        if (total + len > room) continue;  // does not fit next to the more valuable ones: it stays a decoded stream
        picks.push_back(Pick{r.second, len, total, th.n_blocks + (th.tail_n ? 1u : 0u)});
        total += len;
        n_units64 += units;
    }
    if (picks.empty()) return chosen;
    uint64_t at = list_arena_alloc(e, total);
    while (at == ~0ull && picks.size() > 1) {  // (first call: the arena turned out smaller than hoped) build the most valuable half
        picks.resize(picks.size() / 2);
        total = picks.back().off + picks.back().len;
        at = list_arena_alloc(e, total);
    }
    if (at == ~0ull) return chosen;
    float* base = e->list_arena.p + at;
    e->list_slabs.push_back(rg_engine::ListSlab{at, total, {}});
    std::vector<ColumnJob> jobs;
    uint32_t n_units = 0;
    cudaStream_t st = e->stream;
    for (const Pick& pk : picks) {
        auto ent = std::make_shared<ColEntry>();
        ent->key = pk.key;
        ent->len = pk.len;
        ent->col = base + pk.off;
        ent->in_arena = true;
        e->list_slabs.back().entries.push_back(ent);
        jobs.push_back(column_job(pk.key, ent->col, n_units));
        n_units += pk.units;
        e->list_cache[pk.key] = ent;
        e->list_floats += pk.len;
        e->list_builds++;
        add_ref(pk.key, ent);
    }
    uint32_t jb = 0;
    const ColumnJob* d_jobs = stage_jobs(e, jobs, jb);
    launch_build_lists(st, e->d_segs.p, d_jobs, (uint32_t)jobs.size(), n_units, e->d_caches.p, k1);
    RG_CUDA_CHECK(cudaEventRecord(e->list_jobs_done[jb], st));
    RG_CUDA_CHECK(cudaGetLastError());
    e->launches++;
    hp.n_lists_built = (uint32_t)jobs.size();
    return chosen;
}

// Batch-local scored lists.  In a plain-sum disjunction (every clause score > 0, no MUST_NOT, min_should_match or
// dismax) a clause that is neither read from a score column nor given a persistent list above — rare, or used once —
// gets a scored list for this batch only, whatever its df: then every clause of the item is a column or a list and
// the item runs in the decode-free k_eval_or, which needs fewer registers and no stream cache in shared memory.
// Same layout and values as a persistent list (k_build_columns<4>); they live in the batch's slab, are freed with it
// and never enter the list arena or its LRU.  They are taken smallest first within local_list_budget_floats; a clause
// over the budget stays a block stream and its items stay on the stream variant.  RG_CFG_NO_LISTS / RG_CFG_MAXSCORE:
// none.
//
// The budget per batch is a sixteenth of the HBM free when first needed (after the candidate and list arenas, less
// what the score columns may still take): a batch's slab can be held by two batches in flight and three idle spare
// slabs, each with 1/8 headroom, so local lists hold at most about a third of that memory.  Recomputed after an
// upload.  RG_LOCAL_LISTS_KB sets it (tests).
static uint64_t local_list_budget_floats(rg_engine* e) {
    if (!e->local_budget_floats) {
        if (const char* v = getenv("RG_LOCAL_LISTS_KB")) {
            e->local_budget_floats = std::max<uint64_t>(1, strtoull(v, nullptr, 10) * 1024 / sizeof(float));
        } else {
            size_t free_b = 0, total_b = 0;
            RG_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
            const uint64_t col_room = e->col_budget_floats > e->col_floats ? (e->col_budget_floats - e->col_floats) * sizeof(float) : 0;
            const uint64_t avail = free_b > col_room ? free_b - col_room : 0;
            e->local_budget_floats = std::max<uint64_t>(1, avail / 16 / sizeof(float));
        }
    }
    return e->local_budget_floats;
}

void choose_local_lists(rg_engine* e, const std::vector<QShape>& shapes, const rg_clause* clauses, float k1,
                        const std::map<ColKey, uint32_t>& columns, std::map<ColKey, uint32_t>& lists, HostPlan& hp) {
    if (e->cfg.flags & (RG_CFG_NO_LISTS | RG_CFG_MAXSCORE)) return;
    uint32_t k1bits;
    memcpy(&k1bits, &k1, 4);
    std::map<ColKey, uint64_t> want;  // clause -> list length in floats: a unit of 256 per block and tail
    for (const QShape& sh : shapes) {
        if (sh.type != kTypeOr || sh.match_all || sh.clause_idx.size() >= 10 || sh.msm || sh.dismax || !sh.not_idx.empty())
            continue;
        for (uint32_t si = 0; si < e->segs.size(); si++) {
            const Segment& seg = e->segs[si];
            auto df_of = [&](const rg_clause& c) -> uint64_t {
                return c.term_id < seg.host_terms.size() ? (uint64_t)seg.host_terms[c.term_id].doc_freq : 0u;
            };
            bool pos = true;  // as plan_batch's item_pos
            for (uint32_t ci : sh.clause_idx)
                if (df_of(clauses[ci])) pos = pos && scores_positive(seg, clause_weight(clauses[ci]), clauses[ci].cache_id, k1);
            if (!pos) continue;
            for (uint32_t ci : sh.clause_idx) {
                const rg_clause& c = clauses[ci];
                const uint64_t df = df_of(c);
                if (!df) continue;
                const ColKey key = col_key(si, c, k1bits);
                if ((df * e->or_col_den >= (uint64_t)seg.max_doc && columns.count(key)) || lists.count(key)) continue;
                // + one unit: stream_refill prefetches the block after a full block, and a list whose item keeps a
                // block stream (budget) is read by the stream variant
                want.emplace(key, (uint64_t)(seg.host_terms[c.term_id].n_blocks + 1u) * 256u);
            }
        }
    }
    if (want.empty()) return;
    std::vector<std::pair<uint64_t, ColKey>> order;
    order.reserve(want.size());
    for (const auto& kv : want) order.emplace_back(kv.second, kv.first);
    std::sort(order.begin(), order.end());
    const uint64_t budget = local_list_budget_floats(e);
    for (const auto& r : order) {
        const ColKey& key = r.second;
        const TermHost& th = e->segs[std::get<0>(key)].host_terms[std::get<1>(key)];
        // sorted by length: once one does not fit, none of the rest does.  ItemClause.flags carries the reference in
        // 16 bits; the build launch counts units in 31.
        if (hp.local_floats + r.first > budget || hp.col_refs.size() >= 65536 ||
            (uint64_t)hp.local_units + th.n_blocks + 1u > 0x7fffffffu)
            break;
        lists[key] = (uint32_t)hp.col_refs.size();
        hp.local_refs.emplace_back((uint32_t)hp.col_refs.size(), hp.local_floats);
        hp.col_refs.push_back(ColRef{nullptr, nullptr, nullptr, nullptr, 1.0f, 1.0f});
        // dst is an offset in floats, rebased in rg_batch_prepare
        hp.local_jobs.push_back(column_job(key, reinterpret_cast<void*>((uintptr_t)hp.local_floats), hp.local_units));
        hp.local_units += th.n_blocks + (th.tail_n ? 1u : 0u);
        hp.local_floats += r.first;
    }
}

// The shape of every query of a batch: classify_groups where the entry point passes groups, classify_ranges where it
// passes ranges, else classify (rescore: with the refusals of rescoring queries).  With groups, `ext` is the planner's copy of the
// clause array plus what the collapses append; returns the clause array the shapes index.
const rg_clause* classify_batch(const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                                uint32_t n_clauses, const rg_point_range* ranges, uint32_t n_ranges,
                                const rg_query* groups, uint32_t n_groups, uint32_t n_caches, bool rescore,
                                std::vector<rg_clause>& ext, std::vector<QShape>& shapes) {
    shapes.assign(n_queries, QShape{});
    if (groups) ext.assign(clauses, clauses + n_clauses);
    for (uint32_t qi = 0; qi < n_queries; qi++) {
        if (ranges && (uint64_t)queries[qi].clause_begin + queries[qi].n_clauses > n_clauses)
            throw ArgError("query clause range out of bounds");
        if (groups && classify_groups(queries[qi], ext, n_clauses, ranges, n_ranges, groups, n_groups, n_caches, shapes[qi])) {
        } else if (ranges && classify_ranges(queries[qi], groups ? ext.data() : clauses, ranges, n_ranges, shapes[qi])) {
        } else {
            shapes[qi] = classify(queries[qi], groups ? ext.data() : clauses, n_clauses, rescore);
        }
        if (groups) clauses = ext.data();  // (ext may have moved)
        const QShape& sh = shapes[qi];
        // ReqNotScorer moves past an excluded hit with next(), and a SHOULD disjunction with min_should_match > 1
        // then skips to the next doc that reaches min_should_match: whether a later hit matches depends on the walk
        if (rescore && sh.msm > 1 && !sh.not_idx.empty())
            throw Unsupported("rescoring with a min_should_match > 1 disjunction beside MUST_NOT clauses");
        // a query that is a group of 10 or more members scores through a DisiPriorityQueue (classify refuses the
        // flat shapes of that width)
        if (rescore && sh.type == kTypeOr && sh.msm == 0 && sh.clause_idx.size() > (size_t)kMaxTerms)
            throw Unsupported("rescoring with a disjunction of 10 or more clauses and min_should_match <= 1 (DisiPriorityQueue order)");
        check_caches(sh, clauses, n_caches);
    }
    return clauses;
}

// RangeRef per (leaf, range), leaf-major: the range clauses of leaf si point at entry si * n_ranges + range
void fill_range_refs(const rg_engine* e, const rg_point_range* ranges, uint32_t n_ranges, std::vector<RangeRef>& refs) {
    const uint32_t n_segs = (uint32_t)e->segs.size();
    refs.assign((size_t)n_segs * n_ranges, RangeRef{});
    for (uint32_t si = 0; si < n_segs; si++)
        for (uint32_t ri = 0; ri < n_ranges; ri++) {
            const rg_point_range& r = ranges[ri];
            const PointField* pfp = point_field(e->segs[si], r);  // a bytes_per_dim mismatch is RG_EINVAL here
            if (!pfp) continue;
            const PointField& pf = *pfp;
            refs[(size_t)si * n_ranges + ri] = RangeRef{pf.offsets.p, pf.keys.p, pf.blocks.p, be_key(r.lower, r.bytes_per_dim),
                                                        be_key(r.upper, r.bytes_per_dim), pf.bytes_per_dim == 8 ? 1u : 0u, 0u};
        }
}

bool has_ranges(const std::vector<QShape>& shapes) {
    for (const QShape& sh : shapes)
        if (!sh.req_rng.empty() || !sh.not_rng.empty()) return true;
    return false;
}

void plan_batch(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                uint32_t n_clauses, uint32_t mode, float k1, HostPlan& hp, PlanTimer& tm, PlanScratch& scratch,
                const rg_point_range* ranges, uint32_t n_ranges, const rg_query* groups = nullptr,
                uint32_t n_groups = 0) {
    const uint32_t n_caches = (uint32_t)(e->h_caches.size() / 256);
    const uint32_t n_segs = (uint32_t)e->segs.size();
    std::vector<QShape> shapes;
    std::vector<rg_clause> ext;  // groups: the clause array grows by what the collapses make (classify_groups)
    clauses = classify_batch(queries, n_queries, clauses, n_clauses, ranges, n_ranges, groups, n_groups, n_caches, false,
                             ext, shapes);
    // Docid ranges (= work items) per (query, leaf).  A caller's rg_config.range_postings is taken as is: ~that many
    // postings per range.  By default conjunction items (one CTA each) get 32 K postings; disjunctions (one warp each)
    // are cut on a GRID THE WHOLE BATCH SHARES: per leaf a power of two R_leaf <= 256 of equal docid ranges, sized so that
    // an average query's range holds ~128 K postings (longer ranges cost less setup and keep theta chains short) but the
    // batch still has ~32 K items; an inexpensive query takes R_leaf / 2^j of them (>= 8 K postings each).  Items are
    // launched in order of their range's start on that grid, so the warps in flight read the same region of the
    // columns, lists and norms through L2 — measured on C4 (one 100 M-doc leaf, one H100 at 400 W, columns for
    // df >= max_doc/8): 128 equal ranges 670 ms, 256 627, 512 627.
    static const uint64_t max_ranges = getenv("RG_MAX_RANGES") ? std::max(1, atoi(getenv("RG_MAX_RANGES"))) : 256;  // tuning knob
    uint64_t and_rp = e->cfg.range_postings, or_rp = e->cfg.range_postings;
    std::vector<uint32_t> or_grid(n_segs, 0);  // R_leaf; 0 = per-query ranges of or_rp postings (explicit range_postings)
    if (!e->range_postings_set) {
        and_rp = 1u << 15;
        uint64_t n_or = 0;
        std::vector<uint64_t> leaf_cost(n_segs, 0);
        for (const QShape& sh : shapes)
            if (sh.type == kTypeOr) {
                n_or++;
                for (uint32_t si = 0; si < n_segs; si++)
                    for (uint32_t ci : sh.clause_idx)
                        if (clauses[ci].term_id < e->segs[si].host_terms.size())
                            leaf_cost[si] += (uint64_t)e->segs[si].host_terms[clauses[ci].term_id].doc_freq;
            }
        uint64_t total = 0;
        for (uint64_t c : leaf_cost) total += c;
        const uint64_t per_range = std::min<uint64_t>(1u << 17, std::max<uint64_t>(1u << 13, total >> 15));
        for (uint32_t si = 0; si < n_segs; si++) {
            const uint64_t mean = n_or ? leaf_cost[si] / n_or : 0;
            uint32_t g = 1;
            while (g < max_ranges && (uint64_t)g * per_range < mean) g <<= 1;
            or_grid[si] = std::min<uint32_t>(g, (uint32_t)max_ranges);
        }
    }
    if (has_ranges(shapes)) fill_range_refs(e, ranges, n_ranges, hp.range_refs);
    tm.mark("classify");
    const std::map<ColKey, uint32_t> columns = choose_columns(e, shapes, clauses, k1, hp, tm);
    tm.mark("columns");
    std::map<ColKey, uint32_t> lists = choose_lists(e, shapes, clauses, k1, columns, hp);
    tm.mark("lists");
    choose_local_lists(e, shapes, clauses, k1, columns, lists, hp);
    tm.mark("local_lists");
    uint32_t k1bits;
    memcpy(&k1bits, &k1, 4);
    const bool no_ms = (e->cfg.flags & RG_CFG_MAXSCORE) == 0;
    const bool lists_on = (e->cfg.flags & (RG_CFG_NO_LISTS | RG_CFG_MAXSCORE)) == 0;
    // Queries are planned in parallel: contiguous chunks, one HostPlan each, concatenated in query order (item order
    // is collection order, so the result equals the serial plan).
    std::mutex refs_mutex;
    const uint32_t n_threads = n_queries >= 512 ? std::min<uint32_t>(16u, std::max(1u, std::thread::hardware_concurrency())) : 1u;
    auto plan_range = [&](uint32_t q_begin, uint32_t q_end, HostPlan& lp) {
    using Req = ConjLeaf::Req;
    // scratch of every (query, leaf) this thread plans
    ConjLeaf cl;
    std::vector<uint32_t> present, nots, opts;
    for (uint32_t qi = q_begin; qi < q_end; qi++) {
        const QShape& shape = shapes[qi];
        bool group_open = false;
        uint32_t chain_pos = 0;
        for (uint32_t si = 0; si < n_segs; si++) {
            const Segment& seg = e->segs[si];
            const uint64_t n_blocks = (uint64_t)(seg.max_doc + kBlock - 1) / kBlock;
            // The (query, leaf) as R work items, the docid ranges of [0, max_doc) cut evenly (on 128-doc block edges
            // when a range leads: it walks whole blocks), the next links of the query's heap chain, appended to the
            // route's launch list; range r gets the launch-order key r * rank_step.
            auto emit = [&](Route route, uint32_t type, uint32_t n_terms, uint32_t clause_begin, uint32_t width, uint64_t R,
                            uint32_t rank_step, bool block_edges) {
                const bool new_group = mode == RG_MODE_SEARCH_PARALLEL || !group_open;
                if (new_group) {
                    // SEARCH: one heap per query over all its leaves; SEARCH_PARALLEL: one per leaf
                    lp.group_out.push_back(mode == RG_MODE_SEARCH_PARALLEL ? si * n_queries + qi : qi);
                    group_open = true;
                }
                for (uint64_t r = 0; r < R; r++) {
                    WorkItem it{};
                    it.query = qi;
                    it.seg = (uint16_t)si;
                    it.type = (uint8_t)type;
                    it.n_terms = (uint8_t)n_terms;
                    it.lo = (int32_t)((uint64_t)seg.max_doc * r / R);
                    it.hi = (int32_t)((uint64_t)seg.max_doc * (r + 1) / R);
                    if (block_edges) {
                        it.lo = (int32_t)(n_blocks * r / R * kBlock);
                        it.hi = r + 1 == R ? seg.max_doc : (int32_t)(n_blocks * (r + 1) / R * kBlock);
                    }
                    it.clause_begin = clause_begin;
                    it.chain_pos = (r == 0 && new_group) ? 0u : chain_pos;
                    chain_pos = it.chain_pos + 1;
                    lp.ids[route].push_back((uint32_t)lp.items.size());
                    if (kRouteByRank[route]) lp.rank[route].push_back((uint32_t)r * rank_step);
                    lp.items.push_back(it);
                }
                lp.width[route] = std::max(lp.width[route], width);
            };
            auto range_clause = [&](uint32_t ci, uint32_t not_flag) {
                return ItemClause{si * n_ranges + clauses[ci].term_id, 0.0f, 0u, kClauseRange | not_flag};
            };
            const uint32_t clause_begin = (uint32_t)lp.clauses.size();
            if (shape.type != kTypeOr) {
                // BooleanWeight::create_scorer of a conjunction / ReqOpt in this leaf
                if (!cl.resolve(shape, seg, clauses, ranges)) continue;
                const std::vector<Req>& req = cl.req;
                const std::vector<Req>& opt = cl.opt;
                const std::vector<uint32_t>& members = cl.members;
                const auto& rreq = cl.rreq;
                const bool range_lead = cl.range_lead;
                const uint32_t leaf_type = cl.leaf_type;
                const uint64_t cost = cl.cost;
                // bytes: the lead's postings (a range lead: its block table and keys, and every clause's list); each
                // probed term at most one block per lead doc; a group counts as its members
                auto enc = [&](uint32_t ci) -> uint64_t { return seg.host_terms[clauses[ci].term_id].enc_bytes; };
                auto probed = [&](uint32_t ci) -> uint64_t {
                    if (range_lead) return enc(ci);
                    const TermHost& th = seg.host_terms[clauses[ci].term_id];
                    const uint64_t per_block = th.n_blocks ? th.enc_bytes / th.n_blocks : th.enc_bytes;
                    return std::min<uint64_t>(th.enc_bytes, cost * per_block);
                };
                uint64_t bytes = range_lead ? 24ull * n_blocks + 8ull * cost : cost;
                for (size_t i = 0; i < req.size(); i++)
                    for (uint32_t j = 0; j < req[i].n; j++) {
                        const uint32_t ci = members[req[i].begin + j];
                        bytes += i == 0 ? enc(ci) : probed(ci);
                    }
                for (const Req& r : opt)
                    for (uint32_t j = 0; j < r.n; j++) bytes += probed(members[r.begin + j]);
                for (uint32_t ci : cl.nots) bytes += enc(ci);
                lp.postings += cost;
                lp.algo_bytes += bytes;
                // The lead is a block stream; every other term that has a score column is probed by one gather per
                // lead doc instead of skip search + block decode (a MUST_NOT term: any column of the term will do).  A
                // group's members are contiguous, in member order, and always block streams (a group that leads is
                // merged from its members' blocks).  A range that leads comes first; the other required ranges are
                // probed after the terms (each adds +0.0f, so where it is added does not change the sum).
                auto put = [&](const Req& r, bool lead, uint32_t side) {
                    for (uint32_t j = 0; j < r.n; j++) {
                        const rg_clause& c = clauses[members[r.begin + j]];
                        if (r.group) {
                            const uint32_t last = j + 1 == r.n ? kClauseGroupLast : 0u;
                            lp.clauses.push_back(ItemClause{c.term_id, r.filter ? 0.0f : c.weight, c.cache_id,
                                                            (side == kClauseOpt ? kClauseOptGroup : kClauseReqGroup) | last});
                            continue;
                        }
                        const int64_t col = lead ? -1 : col_of(columns, si, c, k1bits);
                        if (col >= 0) lp.clauses.push_back(ItemClause{(uint32_t)col, clause_weight(c), c.cache_id, side | kClauseColumn});
                        else lp.clauses.push_back(ItemClause{c.term_id, clause_weight(c), c.cache_id, side});
                    }
                };
                if (range_lead) lp.clauses.push_back(range_clause(rreq[0].second, 0u));
                for (size_t i = 0; i < req.size(); i++) put(req[i], i == 0 && !range_lead, 0u);
                for (size_t i = range_lead ? 1 : 0; i < rreq.size(); i++) lp.clauses.push_back(range_clause(rreq[i].second, 0u));
                for (uint32_t ci : cl.nots) {
                    const int64_t col = col_of(columns, si, clauses[ci], k1bits);
                    if (col >= 0) lp.clauses.push_back(ItemClause{(uint32_t)col, 0.0f, clauses[ci].cache_id, kClauseNot | kClauseColumn});
                    else lp.clauses.push_back(ItemClause{clauses[ci].term_id, 0.0f, clauses[ci].cache_id, kClauseNot});
                }
                for (uint32_t ci : cl.rnots) lp.clauses.push_back(range_clause(ci, kClauseNot));
                for (const Req& r : opt) put(r, false, kClauseOpt);
                const uint32_t n_item_terms = (uint32_t)(lp.clauses.size() - clause_begin);
                if (n_item_terms > (uint32_t)kMaxTerms || (!range_lead && req[0].group && req[0].n > 8u))  // a leading group: one warp of k_eval_and_nested per member
                    throw Unsupported("a conjunction item wider than k_eval_and takes");  // (the classifiers keep this unreachable)
                // Ranges of ~range_postings postings, at most max_ranges per (query, leaf).  A ReqOptScorer with a
                // required term or group keeps its running mean over the whole leaf: one item.  One whose required
                // side is only ranges scores +0.0f there, so scores_sum stays 0, 2 * 0 < 0 never holds and the running
                // mean never skips the optional side: its docid ranges are independent.
                uint64_t R = std::min<uint64_t>((cost + and_rp - 1) / and_rp, max_ranges);
                R = std::max<uint64_t>(1, std::min<uint64_t>(R, n_blocks));
                if (leaf_type == kTypeReqOpt && !req.empty()) R = 1;
                bool grouped = false;
                for (const Req& r : req) grouped = grouped || r.group;
                for (const Req& r : opt) grouped = grouped || r.group;
                const bool ro = leaf_type == kTypeReqOpt;
                const Route route = grouped                             ? (ro ? kRouteReqOptNested : kRouteAndNested)
                                    : !rreq.empty() || !cl.rnots.empty() ? (ro ? kRouteReqOptRanges : kRouteAndRanges)
                                                                      : (ro ? kRouteReqOpt : kRouteAnd);
                emit(route, leaf_type, n_item_terms, clause_begin, 0u, R, 1u, range_lead);
                continue;
            }
            // disjunctions: present = the scoring clauses, nots = the MUST_NOT ones
            if (!resolve_leaf(shape, seg, clauses, present, nots, opts)) continue;
            // ten or more sub-scorers in this leaf: DisjunctionSumScorer / DisjunctionMaxScorer switch to the
            // DisiPriorityQueue (disjunction_scorer.rs:41-45,118-139), whose summation order only k_eval_dpq reproduces
            const bool leaf_dpq = !shape.match_all && present.size() >= 10;
            uint64_t cost = 0, bytes = 0;
            if (shape.match_all) {
                cost = (uint64_t)seg.max_doc;  // AllDocsIterator: every docid of the leaf
            } else {
                for (uint32_t ci : present) {
                    const TermHost& th = seg.host_terms[clauses[ci].term_id];
                    cost += (uint64_t)th.doc_freq;
                    bytes += th.enc_bytes + 12ull * th.n_blocks;  // + skip table / descriptors
                }
                bytes += cost;  // one norm byte per scored posting
            }
            for (uint32_t ci : nots) bytes += seg.host_terms[clauses[ci].term_id].enc_bytes;
            lp.postings += cost;
            lp.algo_bytes += bytes;
            auto df_of = [&](uint32_t ci) { return (uint64_t)seg.host_terms[clauses[ci].term_id].doc_freq; };
            bool use_ms = false;
            uint32_t n_streams = 0;
            bool item_pos = !shape.match_all;  // every clause score > 0: the plain-sum kernel variant applies
            for (uint32_t ci : present) item_pos = item_pos && scores_positive(seg, clause_weight(clauses[ci]), clauses[ci].cache_id, k1);
            if (shape.match_all) {
                // the leaf's match-all column (every docid present, score 0) + the MUST_NOT streams: k_eval_or<NOT>
                const auto it = columns.find(ColKey(si, kMatchAllTerm, 0u, 0u, 0u));
                if (it == columns.end()) throw Unsupported("no memory for the MatchAllDocsQuery column");
                lp.clauses.push_back(ItemClause{it->second, 0.0f, 0u, kClauseColumn | kClauseNoBound | kClauseAllDocs});
            } else if (leaf_dpq) {
                for (uint32_t ci : present) lp.clauses.push_back(ItemClause{clauses[ci].term_id, clause_weight(clauses[ci]), clauses[ci].cache_id, 0});
            } else {
                // A disjunction goes to k_eval_or_ms (presence bitmaps, non-essential clauses are only counted)
                // when it is a plain sum of SHOULD clauses, reads at least one score column, and none of its
                // other clauses is dense (a dense block stream would cut its windows to a few docids).
                uint32_t n_bitmap = 0;
                bool dense_stream = false;
                for (uint32_t ci : present) {
                    if (seg.bitmap_slot[clauses[ci].term_id] >= 0) n_bitmap++;
                    else if (df_of(ci) * 32u >= (uint64_t)seg.max_doc) dense_stream = true;  // (bitmap budget ran out)
                }
                use_ms = !no_ms && n_bitmap > 0 && !dense_stream && nots.empty() && !shape.msm && !(shape.dismax && present.size() > 1);
                for (uint32_t ci : present) {
                    const rg_clause& c = clauses[ci];
                    const int64_t col = col_of(columns, si, c, k1bits);
                    const float w = clause_weight(c);
                    // the score bound w*(k1+1) needs weight >= 0 and cache entries >= 0
                    const bool boundable = w >= 0.0f && w < INFINITY && k1 >= 0.0f &&
                                           c.cache_id < e->cache_nonneg.size() && e->cache_nonneg[c.cache_id];
                    const uint32_t bound = boundable ? 0u : kClauseNoBound;
                    // the exhaustive kernel scans a column docid by docid: that only pays for df >= max_doc/8
                    if (col >= 0 && (use_ms || df_of(ci) * e->or_col_den >= (uint64_t)seg.max_doc)) {
                        lp.clauses.push_back(ItemClause{(uint32_t)col, w, c.cache_id, kClauseColumn | bound});
                        continue;
                    }
                    n_streams++;
                    uint32_t flags = 0;
                    if (!use_ms && !lists.empty()) {  // a scored list of this clause: streamed instead of decoded
                        const auto lt = lists.find(col_key(si, c, k1bits));
                        if (lt != lists.end()) flags = kClauseList | (lt->second << kClauseRefShift);
                    }
                    if (use_ms && seg.bitmap_slot[c.term_id] >= 0) {  // a block stream whose presence comes from its bitmap
                        const auto key = std::make_tuple(si, c.term_id, c.cache_id);
                        std::lock_guard<std::mutex> lock(refs_mutex);  // the reference table is shared by the planner threads
                        auto it = hp.bitmap_refs.find(key);
                        if (it == hp.bitmap_refs.end()) {
                            it = hp.bitmap_refs.emplace(key, (uint32_t)hp.col_refs.size()).first;
                            ColRef ref{nullptr, seg.bitmaps.p + (size_t)seg.bitmap_slot[c.term_id] * seg.bitmap_words, nullptr, nullptr,
                                       1.0f, 1.0f};
                            tf_planes_of(e, si, c.term_id, c.cache_id, k1, ref);
                            hp.col_refs.push_back(ref);
                        }
                        if (it->second < 65536u) flags = kClauseBitmap | bound | (it->second << kClauseRefShift);
                    }
                    lp.clauses.push_back(ItemClause{c.term_id, w, c.cache_id, flags});
                }
            }
            for (uint32_t ci : nots) lp.clauses.push_back(ItemClause{clauses[ci].term_id, 0.0f, clauses[ci].cache_id, kClauseNot});
            const uint32_t n_item_terms = (uint32_t)(present.size() + (shape.match_all ? 1 : 0) + nots.size());
            // DisjunctionMaxWeight::create_scorer (disjunction_max_query.rs:135-155): one scorer in this
            // leaf is that scorer; otherwise the tie breaker rides in a meta clause after the item's
            const bool leaf_dismax = shape.dismax && present.size() > 1;
            // the decode-free k_eval_or: a plain sum whose every clause is a score column or a scored list
            bool lean = lists_on && !leaf_dpq && !use_ms && item_pos && nots.empty() && !shape.msm && !leaf_dismax;
            for (uint32_t i = clause_begin; lean && i < lp.clauses.size(); i++)
                lean = (lp.clauses[i].flags & (kClauseColumn | kClauseList)) != 0;
            if (leaf_dismax) lp.clauses.push_back(ItemClause{0u, shape.tie, 0u, kClauseTie});
            // ranges of ~range_postings postings, at most max_ranges per (query, leaf): long lists get
            // longer ranges (a range is one warp's sequential job; there are thousands of warps)
            uint64_t R = std::min<uint64_t>((cost + or_rp - 1) / or_rp, max_ranges);
            uint32_t rank_step = 1;  // launch-order key of range r = r * rank_step (its start on the leaf's grid)
            if (or_grid[si]) {
                R = or_grid[si];
                while (R > 1 && cost / R < (1u << 13)) {
                    R >>= 1;
                    rank_step <<= 1;
                }
            }
            R = std::max<uint64_t>(1, std::min<uint64_t>(R, n_blocks));
            if (leaf_dpq) R = 1;  // sequential scorer state: one item per leaf
            const Route route = leaf_dpq ? kRouteDpq : use_ms ? kRouteMs : lean ? kRouteLean : kRouteOr;
            if (route == kRouteOr) {  // the k_eval_or variant the batch needs
                lp.or_has_not = lp.or_has_not || !nots.empty();
                lp.or_nonpos = lp.or_nonpos || !item_pos;
                lp.or_has_msm = lp.or_has_msm || shape.msm;
                lp.or_has_dmax = lp.or_has_dmax || leaf_dismax;
            }
            const uint32_t type = (leaf_dpq ? kTypeDpq : kTypeOr) | shape.msm << kItemMsmShift | (leaf_dismax ? kItemDismax : 0u);
            emit(route, type, n_item_terms, clause_begin, route == kRouteMs ? n_streams : n_item_terms, R, rank_step, false);
        }
    }
    };
    if (n_threads <= 1) {
        plan_range(0, n_queries, hp);
        tm.mark("plan");
    } else {
        std::vector<HostPlan>& parts = scratch.parts;
        parts.resize(n_threads);
        for (HostPlan& lp : parts) lp.reset();
        std::vector<std::exception_ptr> errs(n_threads);
        std::vector<std::thread> ths;
        for (uint32_t t = 0; t < n_threads; t++)
            ths.emplace_back([&, t] {
                try {
                    plan_range((uint32_t)((uint64_t)n_queries * t / n_threads), (uint32_t)((uint64_t)n_queries * (t + 1) / n_threads), parts[t]);
                } catch (...) {
                    errs[t] = std::current_exception();
                }
            });
        for (auto& th : ths) th.join();
        tm.mark("plan_threads");
        for (auto& ep : errs)
            if (ep) std::rethrow_exception(ep);
        // concatenate in query order: offsets first, then every part is copied by its own thread
        struct Off { size_t items, clauses, groups, ids[kRoutes]; };
        std::vector<Off> off(n_threads + 1, Off{});
        for (uint32_t t = 0; t < n_threads; t++) {
            const HostPlan& lp = parts[t];
            off[t + 1].items = off[t].items + lp.items.size();
            off[t + 1].clauses = off[t].clauses + lp.clauses.size();
            off[t + 1].groups = off[t].groups + lp.group_out.size();
            for (uint32_t r = 0; r < kRoutes; r++) {
                off[t + 1].ids[r] = off[t].ids[r] + lp.ids[r].size();
                hp.width[r] = std::max(hp.width[r], lp.width[r]);
            }
            hp.postings += lp.postings;
            hp.algo_bytes += lp.algo_bytes;
            hp.or_has_not = hp.or_has_not || lp.or_has_not;
            hp.or_nonpos = hp.or_nonpos || lp.or_nonpos;
            hp.or_has_msm = hp.or_has_msm || lp.or_has_msm;
            hp.or_has_dmax = hp.or_has_dmax || lp.or_has_dmax;
        }
        const Off& end = off[n_threads];
        hp.items.resize(end.items);
        hp.clauses.resize(end.clauses);
        hp.group_out.resize(end.groups);
        for (uint32_t r = 0; r < kRoutes; r++) {
            hp.ids[r].resize(end.ids[r]);
            if (kRouteByRank[r]) hp.rank[r].resize(end.ids[r]);
        }
        ths.clear();
        for (uint32_t t = 0; t < n_threads; t++)
            ths.emplace_back([&, t] {
                const HostPlan& lp = parts[t];
                const Off& o = off[t];
                const uint32_t item_off = (uint32_t)o.items, clause_off = (uint32_t)o.clauses;
                for (size_t i = 0; i < lp.items.size(); i++) {
                    WorkItem it = lp.items[i];
                    it.clause_begin += clause_off;
                    hp.items[o.items + i] = it;
                }
                std::copy(lp.clauses.begin(), lp.clauses.end(), hp.clauses.begin() + o.clauses);
                for (uint32_t r = 0; r < kRoutes; r++) {
                    for (size_t i = 0; i < lp.ids[r].size(); i++) hp.ids[r][o.ids[r] + i] = lp.ids[r][i] + item_off;
                    std::copy(lp.rank[r].begin(), lp.rank[r].end(), hp.rank[r].begin() + o.ids[r]);
                }
                std::copy(lp.group_out.begin(), lp.group_out.end(), hp.group_out.begin() + o.groups);
            });
        for (auto& th : ths) th.join();
    }
    tm.mark("merge");
    // Launch order: all first ranges, then all second ranges, ... so that by the time range r of a
    // query starts, its range r-1 has (almost always) finished and published theta; candidate
    // lists then stay ~k*ln(n) per query instead of per range.  Item order itself is untouched.
    auto by_rank = [&scratch](std::vector<uint32_t>& ids, const std::vector<uint32_t>& rank) {
        // stable counting sort on the range index (<= 256 distinct values)
        uint32_t max_rank = 0;
        for (uint32_t r : rank) max_rank = std::max(max_rank, r);
        std::vector<uint32_t> start(max_rank + 2, 0);
        for (uint32_t r : rank) start[r + 1]++;
        for (uint32_t r = 0; r <= max_rank; r++) start[r + 1] += start[r];
        std::vector<uint32_t>& out = scratch.sort_tmp;
        out.resize(ids.size());
        for (size_t i = 0; i < ids.size(); i++) out[start[rank[i]]++] = ids[i];
        ids.swap(out);
    };
    for (uint32_t r = 0; r < kRoutes; r++)
        if (kRouteByRank[r]) by_rank(hp.ids[r], hp.rank[r]);
    // heap groups = contiguous item runs starting at chain-start items
    for (uint32_t i = 0; i < hp.items.size(); i++)
        if (hp.items[i].chain_pos == 0) hp.group_item_begin.push_back(i);
    hp.group_item_begin.push_back((uint32_t)hp.items.size());
    if (hp.group_item_begin.size() != hp.group_out.size() + 1) throw ArgError("internal: group bookkeeping mismatch");
    tm.mark("order");
}

// The rescoring query's scorer per (query, leaf) for k_rescore (RescoreLeaf, engine.hpp), from the same shape
// classification and per-leaf resolution as the first pass (classify_batch, then ConjLeaf or resolve_leaf).  Plans
// every query before anything is launched, so a refused shape leaves the rows untouched.
struct RescorePlan {
    std::vector<RescoreLeaf> leaves;  // [n_queries][n_segs]
    std::vector<ItemClause> clauses;
    std::vector<RangeRef> range_refs;  // per (leaf, range), when a query has ranges
    bool nested = false;               // some clause is a group member or a range: k_rescore<true>
};

void plan_rescore(const rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                  uint32_t n_clauses, const rg_point_range* ranges, uint32_t n_ranges, const rg_query* groups,
                  uint32_t n_groups, RescorePlan& rp) {
    const uint32_t n_caches = (uint32_t)(e->h_caches.size() / 256);
    const uint32_t n_segs = (uint32_t)e->segs.size();
    std::vector<QShape> shapes;
    std::vector<rg_clause> ext;
    clauses = classify_batch(queries, n_queries, clauses, n_clauses, ranges, n_ranges, groups, n_groups, n_caches, true,
                             ext, shapes);
    rp.leaves.assign((size_t)n_queries * n_segs, RescoreLeaf{0u, kRsNone, 0, 0, 0, 0.0f});
    rp.clauses.clear();
    rp.range_refs.clear();
    rp.nested = false;
    if (has_ranges(shapes)) fill_range_refs(e, ranges, n_ranges, rp.range_refs);
    std::vector<uint32_t> present, nots, opts;
    ConjLeaf cl;
    for (uint32_t qi = 0; qi < n_queries; qi++) {
        QShape& shape = shapes[qi];
        // advance() never counts clauses (disjunction_scorer.rs:350-364), and BooleanWeight::create_scorer builds the
        // DisjunctionSumScorer over whatever SHOULD clauses exist in the leaf, however few: min_should_match plays
        // no part in rescoring
        shape.msm = 0;
        // a bare TermQuery, or what BooleanQuery::build / DisjunctionMaxQuery::build collapse to one clause: the
        // TermScorer itself (a DisjunctionSumScorer would add it to 0.0f)
        const bool single = shape.type == kTypeOr && !shape.match_all && !shape.dismax && shape.clause_idx.size() == 1 &&
                            shape.not_idx.empty();
        for (uint32_t si = 0; si < n_segs; si++) {
            const Segment& seg = e->segs[si];
            RescoreLeaf& L = rp.leaves[(size_t)qi * n_segs + si];
            if (shape.type != kTypeOr) {
                // a conjunction / ReqOptScorer, as the first pass resolves it: the required side in cost order (a
                // range that leads first, the other required ranges after the terms and groups: each adds +0.0f), then
                // the optional side in clause order, then the MUST_NOT terms and ranges
                if (!cl.resolve(shape, seg, clauses, ranges)) continue;
                L.clause_begin = (uint32_t)rp.clauses.size();
                L.kind = kRsConj;
                L.tie = shape.tie;
                auto put = [&](const ConjLeaf::Req& r, uint32_t side) {
                    for (uint32_t j = 0; j < r.n; j++) {
                        const rg_clause& c = clauses[cl.members[r.begin + j]];
                        if (r.group) {
                            const uint32_t last = j + 1 == r.n ? kClauseGroupLast : 0u;
                            rp.clauses.push_back(ItemClause{c.term_id, r.filter ? 0.0f : c.weight, c.cache_id,
                                                            (side == kClauseOpt ? kClauseOptGroup : kClauseReqGroup) | last});
                            rp.nested = true;
                        } else {
                            rp.clauses.push_back(ItemClause{c.term_id, clause_weight(c), c.cache_id, side});
                        }
                    }
                };
                auto range = [&](uint32_t ci, uint32_t not_flag) {
                    rp.clauses.push_back(ItemClause{si * n_ranges + clauses[ci].term_id, 0.0f, 0u, kClauseRange | not_flag});
                    rp.nested = true;
                };
                if (cl.range_lead) range(cl.rreq[0].second, 0u);
                for (const ConjLeaf::Req& r : cl.req) put(r, 0u);
                for (size_t i = cl.range_lead ? 1 : 0; i < cl.rreq.size(); i++) range(cl.rreq[i].second, 0u);
                const size_t n_req = rp.clauses.size() - L.clause_begin;
                for (const ConjLeaf::Req& r : cl.opt) put(r, kClauseOpt);
                const size_t n_opt = rp.clauses.size() - L.clause_begin - n_req;
                for (uint32_t ci : cl.nots) rp.clauses.push_back(ItemClause{clauses[ci].term_id, 0.0f, clauses[ci].cache_id, kClauseNot});
                for (uint32_t ci : cl.rnots) range(ci, kClauseNot);
                L.n_req = (uint8_t)n_req;
                L.n_opt = (uint8_t)n_opt;
                L.n_not = (uint8_t)(rp.clauses.size() - L.clause_begin - n_req - n_opt);
                continue;
            }
            if (!resolve_leaf(shape, seg, clauses, present, nots, opts)) continue;
            L.clause_begin = (uint32_t)rp.clauses.size();
            if (shape.match_all) L.kind = kRsAll;
            else if (shape.dismax) L.kind = present.size() > 1 ? kRsMax : kRsTerm;  // one scorer: that scorer (:135-155)
            else L.kind = single ? kRsTerm : kRsSum;
            L.tie = shape.tie;
            L.n_req = (uint8_t)present.size();
            L.n_not = (uint8_t)nots.size();
            for (uint32_t ci : present) rp.clauses.push_back(ItemClause{clauses[ci].term_id, clause_weight(clauses[ci]), clauses[ci].cache_id, 0u});
            for (uint32_t ci : nots) rp.clauses.push_back(ItemClause{clauses[ci].term_id, 0.0f, clauses[ci].cache_id, kClauseNot});
        }
    }
}

void check_rescore_params(const rg_rescore_params* p) {
    if (p->mode > RG_RESCORE_MULTIPLY) throw ArgError("rescore mode out of range");
    if (p->reserved != 0) throw ArgError("rg_rescore_params.reserved must be 0");
}

// Upload the plan into `buf` and queue k_rescore over device rows of stride k, both on the engine stream, timed by
// the engine's rescore events.  No host wait: the copy is ordered behind any earlier k_rescore that reads `buf` (a
// buffer that has to grow is freed by cudaFree, which waits for the device), and a copy from pageable memory returns
// once the host vectors have been staged.
void queue_rescore(rg_engine* e, const RescorePlan& rp, DevBuf<uint8_t>& buf, const rg_rescore_params* p,
                   uint32_t n_queries, uint32_t k, rg_hit* d_hits, const uint32_t* d_counts,
                   const unsigned long long* d_totals) {
    cudaStream_t st = e->stream;
    const size_t leaves_b = (rp.leaves.size() * sizeof(RescoreLeaf) + 255) & ~(size_t)255;
    const size_t clauses_b = (std::max<size_t>(1, rp.clauses.size()) * sizeof(ItemClause) + 255) & ~(size_t)255;
    const size_t total = leaves_b + clauses_b + rp.range_refs.size() * sizeof(RangeRef);
    if (buf.n < total) buf.alloc(total);
    if (!rp.leaves.empty())
        RG_CUDA_CHECK(cudaMemcpyAsync(buf.p, rp.leaves.data(), rp.leaves.size() * sizeof(RescoreLeaf), cudaMemcpyHostToDevice,
                                      st));
    if (!rp.clauses.empty())
        RG_CUDA_CHECK(cudaMemcpyAsync(buf.p + leaves_b, rp.clauses.data(), rp.clauses.size() * sizeof(ItemClause),
                                      cudaMemcpyHostToDevice, st));
    if (!rp.range_refs.empty())
        RG_CUDA_CHECK(cudaMemcpyAsync(buf.p + leaves_b + clauses_b, rp.range_refs.data(),
                                      rp.range_refs.size() * sizeof(RangeRef), cudaMemcpyHostToDevice, st));
    RescoreParams rs{};
    rs.segs = e->d_segs.p;
    rs.n_segs = (uint32_t)e->segs.size();
    rs.leaves = reinterpret_cast<const RescoreLeaf*>(buf.p);
    rs.clauses = reinterpret_cast<const ItemClause*>(buf.p + leaves_b);
    rs.caches = e->d_caches.p;
    rs.k1 = p->k1;
    rs.hits = d_hits;
    rs.counts = d_counts;
    rs.totals = d_totals;
    rs.n_queries = n_queries;
    rs.k = k;
    rs.window = p->window_size;
    rs.mode = p->mode;
    rs.query_weight = p->query_weight;
    rs.rescore_weight = p->rescore_weight;
    uint32_t ncap = 32;
    while (ncap < std::min(k, p->window_size)) ncap <<= 1;
    rs.ncap = ncap;
    rs.ranges = reinterpret_cast<const RangeRef*>(buf.p + leaves_b + clauses_b);
    RG_CUDA_CHECK(cudaEventRecord(e->rescore_ev[0], st));
    launch_rescore(st, rs, rp.nested);
    RG_CUDA_CHECK(cudaGetLastError());
    RG_CUDA_CHECK(cudaEventRecord(e->rescore_ev[1], st));
    e->rescore_timed = true;
    if (n_queries) e->launches++;
}

template <class T>
void up(Span<T>& d, const std::vector<T>& h, cudaStream_t st) {
    if (!h.empty()) RG_CUDA_CHECK(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st));
}

void ensure_arena(rg_engine* e) {
    if (e->cand_arena.p) return;
    size_t free_b = 0, total_b = 0;
    RG_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    uint64_t want = e->cfg.cand_arena_bytes ? e->cfg.cand_arena_bytes : std::min<uint64_t>(8ull << 30, free_b / 6);
    want = std::min<uint64_t>(want, (uint64_t)0xfffffff0u * sizeof(rg_hit));
    want = std::max<uint64_t>(want, 1ull << 20);
    e->cand_arena.alloc(want / sizeof(rg_hit));
}

// k > 1024: the (base, shift) of every query's theta bucket map (eval_shared.cuh: deep_key).  The map only sets the
// resolution of theta, never its validity.  With a finite positive bound U on the query's scores, the top bucket starts
// at U and the 255 below it are 1/32 octave wide (shift 18: 2^18 ordered steps, a float octave being 2^23), covering
// 8 octaves; else (negative or zero weights, norm caches with negative entries) the absolute map base 0, shift 24.
// U is the largest over the query's work items of the round-up sum of its scoring clauses' nextafter(weight*(k1+1))
// (BM25's tf-norm factor is < 1 for norms >= 0); ranges, MUST_NOT, match-all and zero-weight clauses add nothing, a
// group's members each add their own.
static std::vector<uint2> deep_bucket_maps(const rg_engine* e, const HostPlan& hp, uint32_t n_queries, float k1) {
    std::vector<float> ub(n_queries, 0.0f);
    for (const WorkItem& it : hp.items) {
        float u = 0.0f;
        for (uint32_t c = 0; c < it.n_terms; c++) {
            const ItemClause& ic = hp.clauses[it.clause_begin + c];
            if (ic.flags & (kClauseNot | kClauseTie | kClauseAllDocs | kClauseRange)) continue;
            const float w1 = ic.weight * (k1 + 1.0f);
            if (w1 == 0.0f) continue;  // scores +-0 only (FILTER): an all-zero query keeps the absolute map, whose edge 128 is +0
            const bool nonneg = ic.cache_id < e->cache_nonneg.size() && e->cache_nonneg[ic.cache_id];
            if (!(w1 >= 0.0f) || !(w1 < INFINITY) || !(k1 >= 0.0f) || !nonneg) {
                u = INFINITY;
                break;
            }
            u = nextafterf(u + nextafterf(w1, INFINITY), INFINITY);
        }
        ub[it.query] = std::max(ub[it.query], u);
    }
    std::vector<uint2> maps(n_queries);
    for (uint32_t q = 0; q < n_queries; q++) {
        const float u = ub[q];
        if (u > 0.0f && u < INFINITY) {
            uint32_t bits;
            memcpy(&bits, &u, 4);
            maps[q] = uint2{(bits | 0x80000000u) - ((uint32_t)(kDeepBuckets - 1) << 18), 18u};
        } else {
            maps[q] = uint2{0u, 24u};
        }
    }
    return maps;
}

// The range / group array of a *_ranges / *_nested entry point: NULL with a non-zero count is a null argument;
// otherwise a non-null array (even of length 0) makes the range / group clauses readable.
template <class T>
bool readable(const T*& a, uint32_t n) {
    static const T none{};
    if (n && !a) return false;
    if (!a) a = &none;
    return true;
}

int null_argument(rg_batch** out) {
    if (out) *out = nullptr;
    g_last_error = "null argument";
    return RG_EINVAL;
}

}  // namespace

#define RG_TRY try {
#define RG_CATCH \
    }            \
    catch (...) { return translate_exception(); }

extern "C" {

static int batch_prepare(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                         uint32_t n_clauses, const rg_search_params* p, const rg_point_range* ranges, uint32_t n_ranges,
                         rg_batch** out, const rg_query* groups = nullptr, uint32_t n_groups = 0) {
    RG_TRY
    if (!e || !p || !out || (n_queries && !queries) || (n_clauses && !clauses)) throw ArgError("null argument");
    *out = nullptr;
    if (p->k == 0) throw ArgError("k must be >= 1");
    if (p->k > kDeepMaxK) throw Unsupported("k > 16384 is not accelerated");
    if (p->mode != RG_MODE_SEARCH && p->mode != RG_MODE_SEARCH_PARALLEL) throw ArgError("bad mode");
    if (e->segs.empty()) throw ArgError("no segment uploaded");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    PlanTimer tm;
    e->sync_tables();
    ensure_arena(e);
    tm.mark("tables");
    if (!e->plan_scratch) e->plan_scratch = std::make_shared<PlanScratch>();
    PlanScratch& scratch = *static_cast<PlanScratch*>(e->plan_scratch.get());
    HostPlan& hp = scratch.hp;
    hp.reset();
    plan_batch(e, queries, n_queries, clauses, n_clauses, p->mode, p->k1, hp, tm, scratch, ranges, n_ranges, groups,
               n_groups);
    std::unique_ptr<rg_batch> b(new rg_batch());
    b->generation = e->generation;
    b->cols = std::move(hp.cols);
    b->lists = std::move(hp.lists);
    b->n_cols_built = hp.n_cols_built;
    b->n_lists_built = hp.n_lists_built;
    b->list_floats = hp.list_floats;
    b->col_floats = hp.col_floats;
    for (const ColRef& r : hp.col_refs) b->uses_planes = b->uses_planes || r.hi1 != nullptr;
    b->n_queries = n_queries;
    b->k = p->k;
    b->mode = p->mode;
    b->k1 = p->k1;
    b->n_items = (uint32_t)hp.items.size();
    for (uint32_t r = 0; r < kRoutes; r++) {
        b->n_ids[r] = (uint32_t)hp.ids[r].size();
        b->width[r] = hp.width[r];
    }
    b->n_groups = (uint32_t)hp.group_out.size();
    b->or_has_not = hp.or_has_not;
    b->or_nonpos = hp.or_nonpos;
    b->or_has_msm = hp.or_has_msm;
    b->or_has_dmax = hp.or_has_dmax;
    b->n_leaves = (uint32_t)e->segs.size();
    const bool deep = p->k > 1024u;
    std::vector<uint2> deep_maps;
    if (deep) deep_maps = deep_bucket_maps(e, hp, n_queries, p->k1);
    b->postings = hp.postings;
    b->algo_bytes = hp.algo_bytes + (uint64_t)n_queries * p->k * sizeof(rg_hit);
    cudaStream_t st = e->stream;
    tm.mark("fields");
    // carve the slab
    size_t off = 0;
    auto carve = [&](auto& span, size_t count) {
        using T = std::remove_reference_t<decltype(*span.p)>;
        span.n = std::max<size_t>(1, count);
        span.p = reinterpret_cast<T*>(off);  // offset for now; rebased below
        off = (off + span.n * sizeof(T) + 255) & ~(size_t)255;
    };
    carve(b->items, hp.items.size());
    carve(b->clauses, hp.clauses.size());
    for (uint32_t r = 0; r < kRoutes; r++) carve(b->ids[r], hp.ids[r].size());
    carve(b->col_refs, hp.col_refs.size());
    carve(b->local_lists, hp.local_floats / 4);
    carve(b->group_item_begin, hp.group_item_begin.size());
    carve(b->group_out, hp.group_out.size());
    carve(b->range_refs, hp.range_refs.size());
    // running top-k scores of every OR work item (theta inheritance along a heap chain); skipped when it would
    // not fit comfortably (huge batches with k near 1024): theta then falls back to the per-range bound.  Deep
    // batches keep a score histogram of every item there instead (1 KB each)
    b->topk_cap = deep ? (uint32_t)kDeepBuckets : (std::min<uint32_t>(p->k, 1024u) + 31u) & ~31u;
    if (deep) carve(b->deep_map, n_queries);
    const size_t topk_floats = (size_t)b->n_items * b->topk_cap;
    const bool keep_topk = topk_floats * sizeof(float) <= (2ull << 30);
    carve(b->item_topk, keep_topk ? topk_floats : 1);
    carve(b->item_head, b->n_items);
    const size_t zero_off = off;
    carve(b->item_matches, b->n_items);
    carve(b->item_theta, b->n_items);
    carve(b->item_topk_n, b->n_items);
    carve(b->arena_next, 2);
    carve(b->dbg, 16);
    carve(b->range_stats, 3);
    carve(b->group_stats, 3);
    carve(b->out_hits, (size_t)std::max<uint32_t>(1, n_queries) * p->k);
    carve(b->out_counts, n_queries);
    carve(b->out_total, n_queries);
    if (p->mode == RG_MODE_SEARCH_PARALLEL)
        carve(b->leaf_records, (size_t)b->n_leaves * std::max<uint32_t>(1, n_queries) * leaf_record_bytes(p->k));
    {   // the smallest spare slab that fits, else a new one (a cudaMalloc + cudaFree per batch costs milliseconds)
        int best = -1;
        for (size_t i = 0; i < e->spare_slabs.size(); i++)
            if (e->spare_slabs[i].n >= off && (best < 0 || e->spare_slabs[i].n < e->spare_slabs[best].n)) best = (int)i;
        if (best >= 0) {
            b->slab = std::move(e->spare_slabs[best]);
            e->spare_slabs.erase(e->spare_slabs.begin() + best);
        } else {
            if (e->spare_slabs.size() >= 3) {  // none fits: drop the smallest to bound what idle slabs hold
                size_t sm = 0;
                for (size_t i = 1; i < e->spare_slabs.size(); i++)
                    if (e->spare_slabs[i].n < e->spare_slabs[sm].n) sm = i;
                e->spare_slabs.erase(e->spare_slabs.begin() + sm);
            }
            b->slab.alloc(off + off / 8);  // some headroom: the next batch of the same shape will fit
        }
    }
    auto rebase = [&](auto& span) {
        using T = std::remove_reference_t<decltype(*span.p)>;
        span.p = reinterpret_cast<T*>(b->slab.p + reinterpret_cast<size_t>(span.p));
    };
    rebase(b->items); rebase(b->clauses); rebase(b->col_refs); rebase(b->local_lists);
    for (Span<uint32_t>& ids : b->ids) rebase(ids);
    rebase(b->group_item_begin); rebase(b->group_out); rebase(b->item_head); rebase(b->item_matches);
    rebase(b->item_theta); rebase(b->item_topk_n); rebase(b->item_topk); rebase(b->arena_next); rebase(b->dbg); rebase(b->out_hits); rebase(b->out_counts);
    rebase(b->out_total);
    rebase(b->range_refs); rebase(b->range_stats); rebase(b->group_stats);
    if (p->mode == RG_MODE_SEARCH_PARALLEL) rebase(b->leaf_records);
    if (deep) rebase(b->deep_map);
    b->zero_begin = b->slab.p + zero_off;
    b->zero_bytes = off - zero_off;
    float* local_base = reinterpret_cast<float*>(b->local_lists.p);
    for (const auto& r : hp.local_refs) hp.col_refs[r.first].col = local_base + r.second;
    cudaStream_t cs = e->copy_stream;
    up(b->items, hp.items, cs);
    up(b->clauses, hp.clauses, cs);
    for (uint32_t r = 0; r < kRoutes; r++) up(b->ids[r], hp.ids[r], cs);
    up(b->col_refs, hp.col_refs, cs);
    up(b->group_item_begin, hp.group_item_begin, cs);
    up(b->group_out, hp.group_out, cs);
    up(b->range_refs, hp.range_refs, cs);
    if (deep) up(b->deep_map, deep_maps, cs);
    RG_CUDA_CHECK(cudaEventCreateWithFlags(&b->uploaded, cudaEventDisableTiming));
    RG_CUDA_CHECK(cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming));
    for (auto& x : b->ev) RG_CUDA_CHECK(cudaEventCreate(&x));
    RG_CUDA_CHECK(cudaEventRecord(b->uploaded, cs));
    if (!hp.local_jobs.empty()) {
        // on the engine stream, ahead of this batch's run; `done` is recorded behind it so that the slab is not handed
        // to another batch while the build may still write it (rg_batch_destroy of a batch that never ran)
        for (ColumnJob& j : hp.local_jobs) j.dst = local_base + reinterpret_cast<uintptr_t>(j.dst);
        uint32_t jb = 0;
        const ColumnJob* d_jobs = stage_jobs(e, hp.local_jobs, jb);
        launch_build_lists(st, e->d_segs.p, d_jobs, (uint32_t)hp.local_jobs.size(), hp.local_units, e->d_caches.p, p->k1);
        RG_CUDA_CHECK(cudaEventRecord(e->list_jobs_done[jb], st));
        RG_CUDA_CHECK(cudaGetLastError());
        RG_CUDA_CHECK(cudaEventRecord(b->done, st));
        b->local_built = true;
        e->launches++;
        tm.mark("local_lists_build");
    }
    b->h2d_bytes = (hp.items.size() * sizeof(WorkItem)) + hp.clauses.size() * sizeof(ItemClause) +
                   4 * (hp.group_item_begin.size() + hp.group_out.size()) + hp.col_refs.size() * sizeof(ColRef) +
                   hp.range_refs.size() * sizeof(RangeRef);
    b->kernels_per_run = (b->n_groups ? 1 : 0) + (p->mode == RG_MODE_SEARCH_PARALLEL ? 1 : 0);
    for (uint32_t r = 0; r < kRoutes; r++) {
        b->h2d_bytes += 4 * hp.ids[r].size();
        b->kernels_per_run += b->n_ids[r] ? 1 : 0;
    }
    tm.mark("alloc_copy_issue");
    RG_CUDA_CHECK(cudaStreamSynchronize(cs));  // the host vectors go out of scope (a running batch is not waited for)
    tm.mark("sync");
    *out = b.release();
    return RG_OK;
    RG_CATCH
}

int rg_batch_prepare(rg_engine* e, const rg_query* queries, uint32_t n_queries,
                     const rg_clause* clauses, uint32_t n_clauses, const rg_search_params* p,
                     rg_batch** out) {
    return batch_prepare(e, queries, n_queries, clauses, n_clauses, p, nullptr, 0, out);
}

int rg_batch_prepare_ranges(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                            uint32_t n_clauses, const rg_search_params* p, const rg_point_range* ranges,
                            uint32_t n_ranges, rg_batch** out) {
    if (!readable(ranges, n_ranges)) return null_argument(out);
    return batch_prepare(e, queries, n_queries, clauses, n_clauses, p, ranges, n_ranges, out);
}

int rg_batch_prepare_nested(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                            uint32_t n_clauses, const rg_search_params* p, const rg_point_range* ranges,
                            uint32_t n_ranges, const rg_query* groups, uint32_t n_groups, rg_batch** out) {
    if (!readable(ranges, n_ranges) || !readable(groups, n_groups)) return null_argument(out);
    return batch_prepare(e, queries, n_queries, clauses, n_clauses, p, ranges, n_ranges, out, groups, n_groups);
}

int rg_batch_run(rg_engine* e, rg_batch* b) {
    RG_TRY
    if (!e || !b) throw ArgError("null argument");
    if (b->generation != e->generation)
        throw ArgError("stale batch: a segment was uploaded or a norm cache changed after rg_batch_prepare");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    RG_CUDA_CHECK(cudaStreamWaitEvent(st, b->uploaded, 0));
    RG_CUDA_CHECK(cudaEventRecord(b->ev[0], st));
    RG_CUDA_CHECK(cudaMemsetAsync(b->item_head.p, 0xff, b->item_head.bytes(), st));
    RG_CUDA_CHECK(cudaMemsetAsync(b->zero_begin, 0, b->zero_bytes, st));
    EvalParams ep{};
    ep.segs = e->d_segs.p;
    ep.items = b->items.p;
    ep.clauses = b->clauses.p;
    ep.caches = e->d_caches.p;
    ep.n_items = b->n_items;
    ep.k = b->k;
    ep.k1 = b->k1;
    ep.cand_arena = e->cand_arena.p;
    ep.arena_slots = (uint32_t)std::min<size_t>(e->cand_arena.n, 0xfffffff0u);
    ep.arena_next = b->arena_next.p;
    ep.item_head = b->item_head.p;
    ep.item_matches = b->item_matches.p;
    ep.item_theta = b->item_theta.p;
    ep.item_topk = b->item_topk.n > 1 ? b->item_topk.p : nullptr;
    ep.item_topk_n = b->item_topk_n.p;
    ep.error_flag = reinterpret_cast<uint32_t*>(b->arena_next.p + 1);
    ep.dbg = (e->cfg.flags & RG_CFG_STATS) ? b->dbg.p : nullptr;
    ep.touched = b->dbg.p + 15;
    ep.deep_map = b->k > 1024u ? b->deep_map.p : nullptr;
    RG_CUDA_CHECK(cudaEventRecord(b->ev[2], st));
    ep.cols = b->col_refs.p;
    bool has_live = false, has_other = false;
    for (const Segment& sg : e->segs) {
        has_live = has_live || sg.live.p != nullptr;
        has_other = has_other || sg.has_other_enc;
    }
    launch_eval_or_lean(st, ep, b->ids[kRouteLean].p, b->n_ids[kRouteLean], has_live);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_or_ms(st, ep, b->ids[kRouteMs].p, b->n_ids[kRouteMs], b->width[kRouteMs], has_live, b->uses_planes);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_or(st, ep, b->ids[kRouteOr].p, b->n_ids[kRouteOr], std::max(1u, b->width[kRouteOr]), has_live, b->or_has_not,
                   b->or_has_msm, b->or_has_dmax, !b->or_nonpos);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_dpq(st, ep, b->ids[kRouteDpq].p, b->n_ids[kRouteDpq], b->width[kRouteDpq], has_live);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and(st, ep, b->ids[kRouteAnd].p, b->n_ids[kRouteAnd], false, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and(st, ep, b->ids[kRouteReqOpt].p, b->n_ids[kRouteReqOpt], true, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    const RangeParams rgp{b->range_refs.p, b->range_stats.p};
    launch_eval_and_ranges(st, ep, rgp, b->ids[kRouteAndRanges].p, b->n_ids[kRouteAndRanges], false, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and_ranges(st, ep, rgp, b->ids[kRouteReqOptRanges].p, b->n_ids[kRouteReqOptRanges], true, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and_nested(st, ep, rgp, b->group_stats.p, b->ids[kRouteAndNested].p, b->n_ids[kRouteAndNested], false, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and_nested(st, ep, rgp, b->group_stats.p, b->ids[kRouteReqOptNested].p, b->n_ids[kRouteReqOptNested], true, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    RG_CUDA_CHECK(cudaEventRecord(b->ev[3], st));
    ReplayParams rp{};
    rp.cand_arena = e->cand_arena.p;
    rp.item_head = b->item_head.p;
    rp.item_matches = b->item_matches.p;
    rp.group_item_begin = b->group_item_begin.p;
    rp.group_query = b->group_out.p;
    rp.n_groups = b->n_groups;
    rp.k = b->k;
    rp.out_hits = b->out_hits.p;
    rp.out_counts = b->out_counts.p;
    rp.out_total = b->out_total.p;
    rp.leaf_records = b->mode == RG_MODE_SEARCH_PARALLEL ? b->leaf_records.p : nullptr;
    launch_heap_replay(st, rp);
    RG_CUDA_CHECK(cudaGetLastError());
    if (b->mode == RG_MODE_SEARCH_PARALLEL && b->n_leaves >= 1) {
        launch_merge_leaf_records(st, b->leaf_records.p, b->n_leaves, b->n_queries, b->k, b->out_hits.p,
                                  b->out_counts.p, b->out_total.p);
        RG_CUDA_CHECK(cudaGetLastError());
    }
    e->launches += b->kernels_per_run;
    RG_CUDA_CHECK(cudaEventRecord(b->ev[1], st));
    RG_CUDA_CHECK(cudaEventRecord(b->done, st));
    b->ran = true;
    b->synced = false;
    return RG_OK;
    RG_CATCH
}

int rg_batch_fetch(rg_engine* e, rg_batch* b, rg_hit* out_hits, uint32_t* out_counts,
                   uint64_t* out_total_hits) {
    RG_TRY
    if (!e || !b || !out_hits || !out_counts || !out_total_hits) throw ArgError("null argument");
    if (!b->ran) throw ArgError("rg_batch_fetch before rg_batch_run");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    cudaStream_t st = e->copy_stream;  // not the engine stream: the next batch may already be running there
    RG_CUDA_CHECK(cudaStreamWaitEvent(st, b->done, 0));
    unsigned long long flags[2] = {0, 0};
    RG_CUDA_CHECK(cudaMemcpyAsync(out_hits, b->out_hits.p, (size_t)b->n_queries * b->k * sizeof(rg_hit), cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(out_counts, b->out_counts.p, (size_t)b->n_queries * 4, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(out_total_hits, b->out_total.p, (size_t)b->n_queries * 8, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(flags, b->arena_next.p, sizeof(flags), cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    b->synced = true;
    cudaEventElapsedTime(&e->last_run_ms, b->ev[0], b->ev[1]);
    cudaEventElapsedTime(&e->last_eval_ms, b->ev[2], b->ev[3]);
    cudaEventElapsedTime(&e->last_replay_ms, b->ev[3], b->ev[1]);
    cudaGetLastError();
    if (flags[1] & 1ull) throw OutOfArena("candidate arena exhausted: split the batch or raise cand_arena_bytes");
    return RG_OK;
    RG_CATCH
}

void rg_batch_destroy(rg_engine* e, rg_batch* b) {
    if (!b) return;
    // hand the slab back for the next batch — whose plan goes up on the copy stream, so this batch's kernels must be over
    if (e && (b->ran || b->local_built) && !b->synced) cudaEventSynchronize(b->done);
    if (e && b->slab.p) {
        if (e->spare_slabs.size() < 3) {
            e->spare_slabs.push_back(std::move(b->slab));
        } else {
            size_t sm = 0;
            for (size_t i = 1; i < e->spare_slabs.size(); i++)
                if (e->spare_slabs[i].n < e->spare_slabs[sm].n) sm = i;
            if (e->spare_slabs[sm].n < b->slab.n) e->spare_slabs[sm] = std::move(b->slab);
        }
    }
    delete b;
}

int rg_batch_stats(rg_engine* e, rg_batch* b, uint64_t out[8]) {
    RG_TRY
    if (!e || !b || !out) throw ArgError("null argument");
    unsigned long long used = 0;
    if (b->ran) {
        RG_CUDA_CHECK(cudaStreamSynchronize(e->stream));
        RG_CUDA_CHECK(cudaMemcpy(&used, b->arena_next.p, 8, cudaMemcpyDeviceToHost));
    }
    out[0] = b->n_items;
    out[1] = b->postings;
    out[2] = b->algo_bytes;
    out[3] = used;
    out[4] = b->kernels_per_run;
    out[5] = b->h2d_bytes;
    out[6] = b->n_ids[kRouteOr] + b->n_ids[kRouteMs] + b->n_ids[kRouteLean] + b->n_ids[kRouteDpq];
    out[7] = b->n_ids[kRouteAnd] + b->n_ids[kRouteReqOpt];
    return RG_OK;
    RG_CATCH
}

// Prepare, run and fetch.  When the candidate arena overflows, the two halves of the batch run one after the other
// (queries are independent and refer to `clauses` by absolute index, so a half is just a sub-array of `queries`),
// recursively if need be.
static int search_batch(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                        uint32_t n_clauses, const rg_search_params* p, const rg_point_range* ranges, uint32_t n_ranges,
                        const rg_query* groups, uint32_t n_groups, rg_hit* out_hits, uint32_t* out_counts,
                        uint64_t* out_total_hits) {
    rg_batch* b = nullptr;
    int rc = batch_prepare(e, queries, n_queries, clauses, n_clauses, p, ranges, n_ranges, &b, groups, n_groups);
    if (rc != RG_OK) return rc;
    rc = rg_batch_run(e, b);
    if (rc == RG_OK) rc = rg_batch_fetch(e, b, out_hits, out_counts, out_total_hits);
    rg_batch_destroy(e, b);
    if (rc == RG_ENOMEM && n_queries > 1 && p && p->k) {
        const uint32_t h = n_queries / 2;
        rc = search_batch(e, queries, h, clauses, n_clauses, p, ranges, n_ranges, groups, n_groups, out_hits, out_counts,
                          out_total_hits);
        if (rc == RG_OK)
            rc = search_batch(e, queries + h, n_queries - h, clauses, n_clauses, p, ranges, n_ranges, groups, n_groups,
                              out_hits + (size_t)h * p->k, out_counts + h, out_total_hits + h);
    }
    return rc;
}

int rg_search_batch(rg_engine* e, const rg_query* queries, uint32_t n_queries,
                    const rg_clause* clauses, uint32_t n_clauses, const rg_search_params* p,
                    rg_hit* out_hits, uint32_t* out_counts, uint64_t* out_total_hits) {
    return search_batch(e, queries, n_queries, clauses, n_clauses, p, nullptr, 0, nullptr, 0, out_hits, out_counts,
                        out_total_hits);
}

int rg_search_batch_ranges(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                           uint32_t n_clauses, const rg_search_params* p, const rg_point_range* ranges,
                           uint32_t n_ranges, rg_hit* out_hits, uint32_t* out_counts, uint64_t* out_total_hits) {
    if (!readable(ranges, n_ranges)) return null_argument(nullptr);
    return search_batch(e, queries, n_queries, clauses, n_clauses, p, ranges, n_ranges, nullptr, 0, out_hits, out_counts,
                        out_total_hits);
}

int rg_search_batch_nested(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                           uint32_t n_clauses, const rg_search_params* p, const rg_point_range* ranges,
                           uint32_t n_ranges, const rg_query* groups, uint32_t n_groups, rg_hit* out_hits,
                           uint32_t* out_counts, uint64_t* out_total_hits) {
    if (!readable(ranges, n_ranges) || !readable(groups, n_groups)) return null_argument(nullptr);
    return search_batch(e, queries, n_queries, clauses, n_clauses, p, ranges, n_ranges, groups, n_groups, out_hits,
                        out_counts, out_total_hits);
}

// n counters of the batch's last run (zeros before it has run)
static void copy_counters(rg_engine* e, const rg_batch* b, const Span<unsigned long long>& src, uint64_t* out, size_t n) {
    memset(out, 0, n * sizeof(uint64_t));
    if (b->ran) {
        RG_CUDA_CHECK(cudaStreamSynchronize(e->stream));
        RG_CUDA_CHECK(cudaMemcpy(out, src.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    }
}

int rg_batch_range_stats(rg_engine* e, rg_batch* b, uint64_t out[3]) {
    RG_TRY
    if (!e || !b || !out) throw ArgError("null argument");
    copy_counters(e, b, b->range_stats, out, 3);
    return RG_OK;
    RG_CATCH
}

int rg_batch_group_stats(rg_engine* e, rg_batch* b, uint64_t out[3]) {
    RG_TRY
    if (!e || !b || !out) throw ArgError("null argument");
    copy_counters(e, b, b->group_stats, out, 3);
    return RG_OK;
    RG_CATCH
}

int rg_batch_debug(rg_engine* e, rg_batch* b, uint64_t out[16]) {
    RG_TRY
    if (!e || !b || !out) throw ArgError("null argument");
    copy_counters(e, b, b->dbg, out, 16);
    out[14] = b->n_ids[kRouteLean];
    return RG_OK;
    RG_CATCH
}

int rg_batch_columns(rg_engine* e, rg_batch* b, uint32_t* n_columns, uint64_t* bytes) {
    RG_TRY
    if (!e || !b || !n_columns || !bytes) throw ArgError("null argument");
    *n_columns = (uint32_t)b->cols.size();
    *bytes = b->col_floats * sizeof(float);
    return RG_OK;
    RG_CATCH
}

int rg_batch_leaf_records(rg_engine* e, rg_batch* b, void** dev_ptr, size_t* record_bytes) {
    RG_TRY
    if (!e || !b || !dev_ptr || !record_bytes) throw ArgError("null argument");
    if (b->mode != RG_MODE_SEARCH_PARALLEL) throw ArgError("leaf records exist only in RG_MODE_SEARCH_PARALLEL");
    *dev_ptr = b->leaf_records.p;
    *record_bytes = leaf_record_bytes(b->k);
    return RG_OK;
    RG_CATCH
}

// finish_parallel on the device into the engine's merge scratch; nothing is copied back and nothing waits
static void merge_on_device(rg_engine* e, const void* dev_records_all, uint32_t n_leaves, uint32_t n_queries, uint32_t k) {
    if (k == 0 || k > kDeepMaxK) throw ArgError("k out of range");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    // grow-only engine scratch: no cudaMalloc/cudaFree on the per-batch path
    const size_t nq = std::max<uint32_t>(1, n_queries);
    const size_t hits_b = (nq * k * sizeof(rg_hit) + 255) & ~(size_t)255;
    const size_t counts_b = (nq * 4 + 255) & ~(size_t)255;
    const size_t total_b = nq * 8;
    if (e->merge_scratch.n < hits_b + counts_b + total_b) e->merge_scratch.alloc(hits_b + counts_b + total_b);
    rg_hit* d_hits = reinterpret_cast<rg_hit*>(e->merge_scratch.p);
    uint32_t* d_counts = reinterpret_cast<uint32_t*>(e->merge_scratch.p + hits_b);
    unsigned long long* d_total = reinterpret_cast<unsigned long long*>(e->merge_scratch.p + hits_b + counts_b);
    RG_CUDA_CHECK(cudaMemsetAsync(d_hits, 0, nq * k * sizeof(rg_hit), st));
    launch_merge_leaf_records(st, static_cast<const uint8_t*>(dev_records_all), n_leaves, n_queries, k, d_hits, d_counts, d_total);
    RG_CUDA_CHECK(cudaGetLastError());
    e->launches++;
    e->merged_queries = n_queries;
    e->merged_k = k;
}

int rg_merge_leaf_records_device(rg_engine* e, const void* dev_records_all, uint32_t n_leaves, uint32_t n_queries, uint32_t k) {
    RG_TRY
    if (!e || !dev_records_all) throw ArgError("null argument");
    merge_on_device(e, dev_records_all, n_leaves, n_queries, k);
    return RG_OK;
    RG_CATCH
}

int rg_merge_fetch(rg_engine* e, rg_hit* out_hits, uint32_t* out_counts, uint64_t* out_total_hits) {
    RG_TRY
    if (!e || !out_hits || !out_counts || !out_total_hits) throw ArgError("null argument");
    if (!e->merged_k) throw ArgError("rg_merge_fetch before a merge");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    const size_t nq = std::max<uint32_t>(1, e->merged_queries), k = e->merged_k;
    const size_t hits_b = (nq * k * sizeof(rg_hit) + 255) & ~(size_t)255;
    const size_t counts_b = (nq * 4 + 255) & ~(size_t)255;
    RG_CUDA_CHECK(cudaMemcpyAsync(out_hits, e->merge_scratch.p, (size_t)e->merged_queries * k * sizeof(rg_hit), cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(out_counts, e->merge_scratch.p + hits_b, (size_t)e->merged_queries * 4, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(out_total_hits, e->merge_scratch.p + hits_b + counts_b, (size_t)e->merged_queries * 8, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    return RG_OK;
    RG_CATCH
}

int rg_merge_leaf_records(rg_engine* e, const void* dev_records_all, uint32_t n_leaves,
                          uint32_t n_queries, uint32_t k, rg_hit* out_hits, uint32_t* out_counts,
                          uint64_t* out_total_hits) {
    RG_TRY
    if (!e || !dev_records_all || !out_hits || !out_counts || !out_total_hits) throw ArgError("null argument");
    merge_on_device(e, dev_records_all, n_leaves, n_queries, k);
    return rg_merge_fetch(e, out_hits, out_counts, out_total_hits);
    RG_CATCH
}

static int batch_rescore(rg_engine* e, rg_batch* b, const rg_query* queries, uint32_t n_queries,
                         const rg_clause* clauses, uint32_t n_clauses, const rg_point_range* ranges, uint32_t n_ranges,
                         const rg_query* groups, uint32_t n_groups, const rg_rescore_params* p) {
    RG_TRY
    if (!e || !b || !p || (n_queries && !queries) || (n_clauses && !clauses)) throw ArgError("null argument");
    check_rescore_params(p);
    if (!b->ran) throw ArgError("rg_batch_rescore before rg_batch_run");
    if (b->generation != e->generation)
        throw ArgError("stale batch: a segment was uploaded or a norm cache changed after rg_batch_prepare");
    if (n_queries != b->n_queries) throw ArgError("rg_batch_rescore: n_queries differs from the batch's");
    if (b->k > 1024) throw Unsupported("rows of more than 1024 hits are not accelerated");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    RescorePlan rp;
    plan_rescore(e, queries, n_queries, clauses, n_clauses, ranges, n_ranges, groups, n_groups, rp);
    queue_rescore(e, rp, b->rescore_plan, p, n_queries, b->k, b->out_hits.p, b->out_counts.p, b->out_total.p);
    RG_CUDA_CHECK(cudaEventRecord(b->done, e->stream));  // rg_batch_fetch waits for the rescored rows
    b->synced = false;
    return RG_OK;
    RG_CATCH
}

static int rescore_hits(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                        uint32_t n_clauses, const rg_point_range* ranges, uint32_t n_ranges, const rg_query* groups,
                        uint32_t n_groups, const rg_rescore_params* p, uint32_t k, rg_hit* hits, const uint32_t* counts,
                        const uint64_t* total_hits) {
    RG_TRY
    if (!e || !p || (n_queries && (!queries || !hits || !counts || !total_hits)) || (n_clauses && !clauses))
        throw ArgError("null argument");
    check_rescore_params(p);
    if (k == 0) throw ArgError("k must be >= 1");
    if (k > 1024) throw Unsupported("rows of more than 1024 hits are not accelerated");
    if (e->segs.empty()) throw ArgError("no segment uploaded");
    for (uint32_t qi = 0; qi < n_queries; qi++) {
        if (counts[qi] > k) throw ArgError("a row's count exceeds k");
        for (uint32_t i = 0; i < counts[qi]; i++) {
            const int32_t d = hits[(size_t)qi * k + i].doc;
            bool in_leaf = false;
            for (const Segment& sg : e->segs) in_leaf = in_leaf || (d >= sg.doc_base && d - sg.doc_base < sg.max_doc);
            if (!in_leaf) throw ArgError("hit docid " + std::to_string(d) + " is in no leaf");
        }
    }
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    e->sync_tables();
    RescorePlan rp;
    plan_rescore(e, queries, n_queries, clauses, n_clauses, ranges, n_ranges, groups, n_groups, rp);
    if (n_queries == 0) return RG_OK;
    const size_t hits_b = ((size_t)n_queries * k * sizeof(rg_hit) + 255) & ~(size_t)255;
    const size_t counts_b = ((size_t)n_queries * 4 + 255) & ~(size_t)255;
    DevBuf<uint8_t> rows, plan;
    rows.alloc(hits_b + counts_b + (size_t)n_queries * 8);
    rg_hit* d_hits = reinterpret_cast<rg_hit*>(rows.p);
    uint32_t* d_counts = reinterpret_cast<uint32_t*>(rows.p + hits_b);
    unsigned long long* d_total = reinterpret_cast<unsigned long long*>(rows.p + hits_b + counts_b);
    cudaStream_t st = e->stream;
    RG_CUDA_CHECK(cudaMemcpyAsync(d_hits, hits, (size_t)n_queries * k * sizeof(rg_hit), cudaMemcpyHostToDevice, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(d_counts, counts, (size_t)n_queries * 4, cudaMemcpyHostToDevice, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(d_total, total_hits, (size_t)n_queries * 8, cudaMemcpyHostToDevice, st));
    queue_rescore(e, rp, plan, p, n_queries, k, d_hits, d_counts, d_total);
    RG_CUDA_CHECK(cudaMemcpyAsync(hits, d_hits, (size_t)n_queries * k * sizeof(rg_hit), cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    return RG_OK;
    RG_CATCH
}

int rg_batch_rescore(rg_engine* e, rg_batch* b, const rg_query* queries, uint32_t n_queries,
                     const rg_clause* clauses, uint32_t n_clauses, const rg_rescore_params* p) {
    return batch_rescore(e, b, queries, n_queries, clauses, n_clauses, nullptr, 0, nullptr, 0, p);
}

int rg_batch_rescore_nested(rg_engine* e, rg_batch* b, const rg_query* queries, uint32_t n_queries,
                            const rg_clause* clauses, uint32_t n_clauses, const rg_point_range* ranges,
                            uint32_t n_ranges, const rg_query* groups, uint32_t n_groups, const rg_rescore_params* p) {
    if (!readable(ranges, n_ranges) || !readable(groups, n_groups)) return null_argument(nullptr);
    return batch_rescore(e, b, queries, n_queries, clauses, n_clauses, ranges, n_ranges, groups, n_groups, p);
}

int rg_rescore_hits(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                    uint32_t n_clauses, const rg_rescore_params* p, uint32_t k, rg_hit* hits,
                    const uint32_t* counts, const uint64_t* total_hits) {
    return rescore_hits(e, queries, n_queries, clauses, n_clauses, nullptr, 0, nullptr, 0, p, k, hits, counts,
                        total_hits);
}

int rg_rescore_hits_nested(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                           uint32_t n_clauses, const rg_point_range* ranges, uint32_t n_ranges, const rg_query* groups,
                           uint32_t n_groups, const rg_rescore_params* p, uint32_t k, rg_hit* hits,
                           const uint32_t* counts, const uint64_t* total_hits) {
    if (!readable(ranges, n_ranges) || !readable(groups, n_groups)) return null_argument(nullptr);
    return rescore_hits(e, queries, n_queries, clauses, n_clauses, ranges, n_ranges, groups, n_groups, p, k, hits,
                        counts, total_hits);
}

// ncclAllGather, resolved at run time so that librucene_gpu.so carries no link-time NCCL dependency (a PyTorch
// process already holds its own libnccl; a Rust host links whichever it wants)
using nccl_all_gather_fn = int (*)(const void*, void*, size_t, int /*ncclDataType_t*/, void* /*ncclComm_t*/, cudaStream_t);
static nccl_all_gather_fn resolve_nccl_all_gather() {
    static nccl_all_gather_fn fn = [] {
        void* sym = dlsym(RTLD_DEFAULT, "ncclAllGather");
        if (!sym) {
            if (void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL)) sym = dlsym(h, "ncclAllGather");
        }
        return reinterpret_cast<nccl_all_gather_fn>(sym);
    }();
    return fn;
}

int rg_batch_run_sharded(rg_engine* e, rg_batch* b, void* nccl_comm, uint32_t n_ranks, rg_hit* out_hits,
                         uint32_t* out_counts, uint64_t* out_total_hits) {
    RG_TRY
    if (!e || !b || !nccl_comm || !out_hits || !out_counts || !out_total_hits) throw ArgError("null argument");
    if (b->mode != RG_MODE_SEARCH_PARALLEL) throw ArgError("rg_batch_run_sharded needs a RG_MODE_SEARCH_PARALLEL batch");
    if (n_ranks == 0 || (uint64_t)n_ranks * b->n_leaves > 65535) throw ArgError("bad rank count");
    const nccl_all_gather_fn all_gather = resolve_nccl_all_gather();
    if (!all_gather) throw Unsupported("libnccl is not available in this process (ncclAllGather not found)");
    int rc = rg_batch_run(e, b);
    if (rc != RG_OK) return rc;
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    const size_t local = (size_t)b->n_leaves * std::max<uint32_t>(1, b->n_queries) * leaf_record_bytes(b->k);
    if (e->gather_scratch.n < local * n_ranks) e->gather_scratch.alloc(local * n_ranks);
    const int nrc = all_gather(b->leaf_records.p, e->gather_scratch.p, local, 1 /* ncclUint8 */, nccl_comm, e->stream);
    if (nrc != 0) throw ArgError("ncclAllGather failed with ncclResult_t " + std::to_string(nrc));
    return rg_merge_leaf_records(e, e->gather_scratch.p, n_ranks * b->n_leaves, b->n_queries, b->k, out_hits, out_counts,
                                 out_total_hits);
    RG_CATCH
}

}  // extern "C"
