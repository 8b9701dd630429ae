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

struct rg_batch {
    uint32_t n_queries = 0, k = 0, mode = 0;
    float k1 = 1.2f;
    uint32_t n_items = 0, n_or = 0, n_ms = 0, n_and = 0, n_ro = 0, n_groups = 0, n_leaves = 0, max_or_terms = 1,
             max_ms_streams = 0;
    uint64_t generation = 0;  // engine->generation at prepare time
    // One device allocation per batch (cudaMalloc/cudaFree cost milliseconds each next to a
    // multi-GB index image; the engine keeps the last slab for the next batch).  Layout:
    // [plan arrays copied from the host][item_head: 0xff per run][everything zeroed per run].
    DevBuf<uint8_t> slab;
    Span<WorkItem> items;
    Span<ItemClause> clauses;
    Span<uint32_t> or_ids, and_ids;  // launch order (range-major) of the OR / AND work items
    Span<uint32_t> ms_ids;           // OR work items evaluated by k_eval_or_ms (bitmaps + non-essential clauses)
    Span<uint32_t> dpq_ids;          // disjunctions with >= 10 clauses in the leaf (k_eval_dpq), one per (query, leaf)
    uint32_t n_dpq = 0, max_dpq_terms = 0;
    bool uses_planes = false;        // some column / bitmap reference of this batch carries tf-norm planes
    Span<uint32_t> ro_ids;           // MUST+SHOULD (ReqOptScorer) work items: one per (query, leaf)
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
    // two batches may be in flight (prepare the next while one runs): the plan goes up on the engine's copy stream,
    // the run waits for `uploaded`, the fetch waits for `done` on the copy stream; timing events are the batch's own
    cudaEvent_t uploaded = nullptr, done = nullptr, ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool synced = false;  // the host has waited for `done`
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
    std::vector<uint32_t> or_ids, ms_ids, and_ids, ro_ids, dpq_ids;
    uint32_t max_dpq_terms = 0;
    std::vector<ColRef> col_refs;
    std::map<std::tuple<uint32_t, uint32_t, uint32_t>, uint32_t> bitmap_refs;  // (leaf, term, cache) -> col_refs entry {null, bits, hi}
    std::vector<std::shared_ptr<ColEntry>> cols, lists;
    uint32_t n_cols_built = 0, n_lists_built = 0, max_ms_streams = 0;
    uint64_t col_floats = 0, list_floats = 0;
    std::vector<uint32_t> or_rank, ms_rank, and_rank;  // range index of each id (launch-order key)
    std::vector<uint32_t> group_item_begin, group_out;
    uint64_t postings = 0, algo_bytes = 0;
    uint32_t max_or_terms = 1;
    bool or_has_not = false, or_has_msm = false, or_has_dmax = false, or_nonpos = false;
    // back to the empty plan, keeping the vectors' storage (a plan is tens of MB: fresh vectors would be page-faulted
    // in by every rg_batch_prepare)
    void reset() {
        items.clear(); clauses.clear(); or_ids.clear(); ms_ids.clear(); and_ids.clear(); ro_ids.clear(); dpq_ids.clear();
        col_refs.clear(); bitmap_refs.clear(); cols.clear(); lists.clear(); or_rank.clear(); ms_rank.clear(); and_rank.clear();
        group_item_begin.clear(); group_out.clear();
        max_dpq_terms = n_cols_built = n_lists_built = max_ms_streams = 0;
        col_floats = list_floats = postings = algo_bytes = 0;
        max_or_terms = 1;
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
};

// what a clause scores with: a FILTER clause is a required clause with NonScoringSimilarity, i.e. exactly 0f32
// (= BM25 with weight +0: 0 * (k1+1) * f / (f + norm) = +0 for any finite norm)
inline float clause_weight(const rg_clause& c) { return c.occur == RG_FILTER ? 0.0f : c.weight; }

// BooleanQuery::build + BooleanWeight::create_scorer wiring for the accelerated shapes.
QShape classify(const rg_query& q, const rg_clause* clauses, uint32_t n_clauses_total) {
    if ((uint64_t)q.clause_begin + q.n_clauses > n_clauses_total) throw ArgError("query clause range out of bounds");
    QShape s;
    if (q.flags & RG_Q_DISMAX) {
        // DisjunctionMaxQuery::build (search/query/disjunction_max_query.rs:51-68) over TermQuerys;
        // DisjunctionMaxScorer::new (disjunction_scorer.rs:118-139): SimpleQueue below 10 disjuncts
        if (q.n_clauses == 0) throw ArgError("DisjunctionMaxQuery: sub query should not be empty!");
        if (q.n_clauses > (uint32_t)kDpqMaxTerms) throw Unsupported("more than 32 disjuncts");
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
        if (!pure_should || n_all > (size_t)kDpqMaxTerms || msm > 1)
            throw Unsupported("more than 9 clauses (only pure SHOULD disjunctions of up to 32 clauses with min_should_match <= 1 go wider)");
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
        return s;
    }
    s.type = kTypeOr;
    s.clause_idx = shoulds;
    // min_should_match > 1 only ever filters a disjunction that is iterated with next(): the
    // top-level SHOULD side.  Beside a MUST it sits behind ReqOptScorer::score -> advance(), which
    // does not look at it (disjunction_scorer.rs:350-363), so those shapes ignore it above.
    s.msm = msm > 1 ? (uint32_t)msm : 0u;
    if (s.msm > 15u) throw Unsupported("min_should_match > 15");
    return s;
}

// Score columns: which (leaf, term, weight, norm cache, k1) clauses of the batch's disjunctions are read
// from a materialised f32 column (k_build_columns) instead of their block stream.  Only terms with a
// presence bitmap (df >= max_doc/64, chosen at upload) qualify.  Columns are persistent: a key that is
// already in the engine's cache is used as is; a new one is built when at least two clauses of the
// batch share it (RG_CFG_EAGER_COLUMNS: one), most valuable (uses x df) first, evicting least recently
// used columns no batch references while over the HBM budget.  RG_CFG_NO_COLUMNS turns the feature off.
constexpr uint32_t kMatchAllTerm = 0xffffffffu;  // ColKey term of a leaf's MatchAllDocsQuery column

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
                const float w = clause_weight(c);
                if (!scores_positive(seg, w, c.cache_id, k1)) return;  // a column cell of +0.0f means "no posting"
                uint32_t wbits;
                memcpy(&wbits, &w, 4);
                uses[ColKey(si, c.term_id, wbits, c.cache_id, k1bits)]++;
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
        ColRef ref{ent->col, ent->bits, nullptr, nullptr, 1.0f, 1.0f};
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
        const uint64_t len = ((uint64_t)seg.max_doc + 1024 + 3) & ~3ull;  // windows read past max_doc
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
        RG_CUDA_CHECK(cudaMemsetAsync(ent->col, 0, len * sizeof(float), st));
        ColumnJob job{};
        job.seg = std::get<0>(r.second);
        job.term_id = std::get<1>(r.second);
        const uint32_t wbits = std::get<2>(r.second);
        memcpy(&job.weight, &wbits, 4);
        job.cache_id = std::get<3>(r.second);
        job.dst = ent->col;
        job.unit_begin = n_units;
        n_units += th.n_blocks + (th.tail_n ? 1u : 0u);
        jobs.push_back(job);
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
                const float w = clause_weight(c);
                uint32_t wbits;
                memcpy(&wbits, &w, 4);
                const ColKey key(si, c.term_id, wbits, c.cache_id, k1bits);
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
        ColumnJob job{};
        job.seg = std::get<0>(pk.key);
        job.term_id = std::get<1>(pk.key);
        const uint32_t wbits = std::get<2>(pk.key);
        memcpy(&job.weight, &wbits, 4);
        job.cache_id = std::get<3>(pk.key);
        job.dst = ent->col;
        job.unit_begin = n_units;
        n_units += pk.units;
        jobs.push_back(job);
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

void plan_batch(rg_engine* e, const rg_query* queries, uint32_t n_queries, const rg_clause* clauses,
                uint32_t n_clauses, uint32_t mode, float k1, HostPlan& hp, PlanTimer& tm, PlanScratch& scratch) {
    const uint32_t n_caches = (uint32_t)(e->h_caches.size() / 256);
    const uint32_t n_segs = (uint32_t)e->segs.size();
    std::vector<QShape> shapes(n_queries);
    for (uint32_t qi = 0; qi < n_queries; qi++) {
        shapes[qi] = classify(queries[qi], clauses, n_clauses);
        for (uint32_t ci : shapes[qi].clause_idx)
            if (clauses[ci].cache_id >= n_caches) throw ArgError("clause refers to an unset norm cache");
        for (uint32_t ci : shapes[qi].opt_idx)
            if (clauses[ci].cache_id >= n_caches) throw ArgError("clause refers to an unset norm cache");
        // MUST_NOT clauses never score, but the kernels still form cache pointers from the id
        for (uint32_t ci : shapes[qi].not_idx)
            if (clauses[ci].cache_id >= n_caches) throw ArgError("clause refers to an unset norm cache");
    }
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
    tm.mark("classify");
    const std::map<ColKey, uint32_t> columns = choose_columns(e, shapes, clauses, k1, hp, tm);
    tm.mark("columns");
    const std::map<ColKey, uint32_t> lists = choose_lists(e, shapes, clauses, k1, columns, hp);
    tm.mark("lists");
    uint32_t k1bits;
    memcpy(&k1bits, &k1, 4);
    const bool no_ms = (e->cfg.flags & RG_CFG_MAXSCORE) == 0;
    // Queries are planned in parallel: contiguous chunks, one HostPlan each, concatenated in query order (item order
    // is collection order, so the result equals the serial plan).
    std::mutex refs_mutex;
    const uint32_t n_threads = n_queries >= 512 ? std::min<uint32_t>(16u, std::max(1u, std::thread::hardware_concurrency())) : 1u;
    auto plan_range = [&](uint32_t q_begin, uint32_t q_end, HostPlan& lp) {
    for (uint32_t qi = q_begin; qi < q_end; qi++) {
        const QShape& shape = shapes[qi];
        bool group_open = false;
        uint32_t chain_pos = 0;
        for (uint32_t si = 0; si < n_segs; si++) {
            const Segment& seg = e->segs[si];
            // resolve clauses against this leaf
            std::vector<uint32_t> present;
            bool dead = false;
            for (uint32_t ci : shape.clause_idx) {
                const uint32_t t = clauses[ci].term_id;
                const int32_t df = t < seg.host_terms.size() ? seg.host_terms[t].doc_freq : 0;
                if (df > 0) present.push_back(ci);
                else if (shape.type != kTypeOr) dead = true;  // create_scorer -> None (:201-206)
            }
            const bool new_group = mode == RG_MODE_SEARCH_PARALLEL || !group_open;
            if (dead || (present.empty() && !shape.match_all)) continue;
            if (shape.type == kTypeOr && shape.msm > present.size()) continue;  // nothing can reach msm here
            std::vector<uint32_t> nots;  // MUST_NOT clauses present in this leaf (:236-251)
            for (uint32_t ci : shape.not_idx) {
                const uint32_t t = clauses[ci].term_id;
                if (t < seg.host_terms.size() && seg.host_terms[t].doc_freq > 0) nots.push_back(ci);
            }
            std::vector<uint32_t> opts;  // SHOULD clauses present in this leaf (:217-234)
            for (uint32_t ci : shape.opt_idx) {
                const uint32_t t = clauses[ci].term_id;
                if (t < seg.host_terms.size() && seg.host_terms[t].doc_freq > 0) opts.push_back(ci);
            }
            // no SHOULD scorer in this leaf -> the MUST side alone, no ReqOptScorer (:259-266)
            // ten or more sub-scorers in this leaf: DisjunctionSumScorer / DisjunctionMaxScorer switch to the
            // DisiPriorityQueue (disjunction_scorer.rs:41-45,118-139), whose summation order only k_eval_dpq reproduces
            const bool leaf_dpq = shape.type == kTypeOr && !shape.match_all && present.size() >= 10;
            const int leaf_type = leaf_dpq ? (int)kTypeDpq
                                           : (shape.type == kTypeReqOpt && opts.empty() ? (int)kTypeAnd : shape.type);
            uint64_t cost = 0, bytes = 0, total_df = 0;
            if (shape.match_all) {
                cost = total_df = (uint64_t)seg.max_doc;  // AllDocsIterator: every docid of the leaf
            } else if (shape.type != kTypeOr) {
                // ConjunctionScorer::new: stable sort by cost() = doc_freq (:30)
                std::stable_sort(present.begin(), present.end(), [&](uint32_t a, uint32_t b) {
                    return seg.host_terms[clauses[a].term_id].doc_freq < seg.host_terms[clauses[b].term_id].doc_freq;
                });
                cost = (uint64_t)seg.host_terms[clauses[present[0]].term_id].doc_freq;
                const TermHost& lead = seg.host_terms[clauses[present[0]].term_id];
                bytes = lead.enc_bytes + cost;
                for (size_t i = 1; i < present.size(); i++) {  // upper bound: min(list, one block per lead doc)
                    const TermHost& th = seg.host_terms[clauses[present[i]].term_id];
                    const uint64_t per_block = th.n_blocks ? th.enc_bytes / th.n_blocks : th.enc_bytes;
                    bytes += std::min<uint64_t>(th.enc_bytes, cost * per_block);
                }
                for (uint32_t ci : opts) {
                    const TermHost& th = seg.host_terms[clauses[ci].term_id];
                    const uint64_t per_block = th.n_blocks ? th.enc_bytes / th.n_blocks : th.enc_bytes;
                    bytes += std::min<uint64_t>(th.enc_bytes, cost * per_block);
                }
                total_df = cost;
            } else {
                for (uint32_t ci : present) {
                    const TermHost& th = seg.host_terms[clauses[ci].term_id];
                    cost += (uint64_t)th.doc_freq;
                    bytes += th.enc_bytes + 12ull * th.n_blocks;  // + skip table / descriptors
                }
                bytes += cost;  // one norm byte per scored posting
                total_df = cost;
            }
            for (uint32_t ci : nots) bytes += seg.host_terms[clauses[ci].term_id].enc_bytes;
            lp.postings += total_df;
            lp.algo_bytes += bytes;
            const uint32_t clause_begin = (uint32_t)lp.clauses.size();
            // score column of a clause in this leaf (-1: none)
            auto col_of = [&](uint32_t ci) -> int64_t {
                if (columns.empty()) return -1;
                const rg_clause& c = clauses[ci];
                const float w = clause_weight(c);
                uint32_t wbits;
                memcpy(&wbits, &w, 4);
                const auto it = columns.find(ColKey(si, c.term_id, wbits, c.cache_id, k1bits));
                return it == columns.end() ? -1 : (int64_t)it->second;
            };
            auto df_of = [&](uint32_t ci) { return (uint64_t)seg.host_terms[clauses[ci].term_id].doc_freq; };
            bool use_ms = false;
            uint32_t n_streams = 0;
            bool item_pos = !shape.match_all;  // every clause score > 0: the plain-sum kernel variant applies
            for (uint32_t ci : present) item_pos = item_pos && scores_positive(seg, clause_weight(clauses[ci]), clauses[ci].cache_id, k1);
            if (shape.match_all) {
                // the leaf's match-all column (every docid present, score 0) + the MUST_NOT streams: k_eval_or<NOT>
                const auto it = columns.find(ColKey(si, kMatchAllTerm, 0u, 0u, 0u));
                if (it == columns.end()) throw Unsupported("no memory for the MatchAllDocsQuery column");
                lp.clauses.push_back(ItemClause{it->second, 0.0f, 0u, 4u | 16u | 64u});  // 64: every docid present
            } else if (leaf_dpq) {
                for (uint32_t ci : present) lp.clauses.push_back(ItemClause{clauses[ci].term_id, clause_weight(clauses[ci]), clauses[ci].cache_id, 0});
            } else if (shape.type == kTypeOr) {
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
                    const int64_t col = col_of(ci);
                    const float w = clause_weight(c);
                    // bit4: the score bound w*(k1+1) needs weight >= 0 and cache entries >= 0
                    const bool boundable = w >= 0.0f && w < INFINITY && k1 >= 0.0f &&
                                           c.cache_id < e->cache_nonneg.size() && e->cache_nonneg[c.cache_id];
                    // the exhaustive kernel scans a column docid by docid: that only pays for df >= max_doc/8
                    if (col >= 0 && (use_ms || df_of(ci) * e->or_col_den >= (uint64_t)seg.max_doc)) {
                        lp.clauses.push_back(ItemClause{(uint32_t)col, w, c.cache_id, 4u | (boundable ? 0u : 16u)});
                        continue;
                    }
                    n_streams++;
                    uint32_t flags = 0;
                    if (!use_ms && !lists.empty()) {  // a scored list of this clause: streamed instead of decoded
                        uint32_t wbits;
                        memcpy(&wbits, &w, 4);
                        const auto lt = lists.find(ColKey(si, c.term_id, wbits, c.cache_id, k1bits));
                        if (lt != lists.end()) flags = 128u | (lt->second << 16);
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
                        if (it->second < 65536u) flags = 32u | (boundable ? 0u : 16u) | (it->second << 16);
                    }
                    lp.clauses.push_back(ItemClause{c.term_id, w, c.cache_id, flags});
                }
            } else {
                // conjunction: the lead (cheapest) clause is a block stream; every other clause that has a score
                // column is probed by one gather per lead doc instead of skip search + block decode
                for (size_t i = 0; i < present.size(); i++) {
                    const rg_clause& c = clauses[present[i]];
                    const int64_t col = i == 0 ? -1 : col_of(present[i]);
                    if (col >= 0) lp.clauses.push_back(ItemClause{(uint32_t)col, clause_weight(c), c.cache_id, 4u});
                    else lp.clauses.push_back(ItemClause{c.term_id, clause_weight(c), c.cache_id, 0});
                }
            }
            for (uint32_t ci : nots) {
                const int64_t col = shape.type == kTypeOr ? -1 : col_of(ci);  // conjunctions: any column of the term will do
                if (col >= 0) lp.clauses.push_back(ItemClause{(uint32_t)col, 0.0f, clauses[ci].cache_id, 1u | 4u});
                else lp.clauses.push_back(ItemClause{clauses[ci].term_id, 0.0f, clauses[ci].cache_id, 1u});
            }
            for (uint32_t ci : opts) {
                const int64_t col = col_of(ci);
                if (col >= 0) lp.clauses.push_back(ItemClause{(uint32_t)col, clauses[ci].weight, clauses[ci].cache_id, 2u | 4u});
                else lp.clauses.push_back(ItemClause{clauses[ci].term_id, clauses[ci].weight, clauses[ci].cache_id, 2u});
            }
            const uint32_t n_item_terms = (uint32_t)(present.size() + (shape.match_all ? 1 : 0) + nots.size() + opts.size());
            // DisjunctionMaxWeight::create_scorer (disjunction_max_query.rs:135-155): one scorer in this
            // leaf is that scorer; otherwise the tie breaker rides in a meta clause after the item's
            const bool leaf_dismax = shape.dismax && present.size() > 1;
            if (leaf_dismax) lp.clauses.push_back(ItemClause{0u, shape.tie, 0u, 8u});
            // ranges of ~range_postings postings, at most max_ranges per (query, leaf): long lists get
            // longer ranges (a range is one warp's sequential job; there are thousands of warps)
            const uint64_t range_postings = leaf_type == (int)kTypeOr ? or_rp : and_rp;
            uint64_t R = (cost + range_postings - 1) / range_postings;
            R = std::min<uint64_t>(R, max_ranges);
            uint32_t rank_step = 1;  // launch-order key of range r = r * rank_step (its start on the leaf's grid)
            if (leaf_type == (int)kTypeOr && or_grid[si]) {
                R = or_grid[si];
                while (R > 1 && cost / R < (1u << 13)) {
                    R >>= 1;
                    rank_step <<= 1;
                }
            }
            R = std::max<uint64_t>(1, std::min<uint64_t>(R, (uint64_t)(seg.max_doc + kBlock - 1) / kBlock));
            if (leaf_type == (int)kTypeReqOpt || leaf_dpq) R = 1;  // sequential scorer state: one item per leaf
            if (new_group) {
                // SEARCH: one heap per query over all its leaves; SEARCH_PARALLEL: one per leaf
                lp.group_out.push_back(mode == RG_MODE_SEARCH_PARALLEL ? si * n_queries + qi : qi);
                group_open = true;
            }
            for (uint64_t r = 0; r < R; r++) {
                WorkItem it{};
                it.query = qi;
                it.seg = (uint16_t)si;
                it.type = (uint8_t)(leaf_type | (shape.type == kTypeOr ? shape.msm << 4 : 0u) | (leaf_dismax ? 4u : 0u));
                it.n_terms = (uint8_t)n_item_terms;
                it.lo = (int32_t)((uint64_t)seg.max_doc * r / R);
                it.hi = (int32_t)((uint64_t)seg.max_doc * (r + 1) / R);
                it.clause_begin = clause_begin;
                it.chain_pos = (r == 0 && new_group) ? 0u : chain_pos;
                chain_pos = it.chain_pos + 1;
                const uint32_t idx = (uint32_t)lp.items.size();
                lp.items.push_back(it);
                if (leaf_dpq) {
                    lp.dpq_ids.push_back(idx);
                    lp.max_dpq_terms = std::max<uint32_t>(lp.max_dpq_terms, n_item_terms);
                } else if (leaf_type == (int)kTypeReqOpt) {
                    lp.ro_ids.push_back(idx);
                } else if (leaf_type == (int)kTypeAnd) {
                    lp.and_ids.push_back(idx);
                    lp.and_rank.push_back((uint32_t)r);
                } else if (use_ms) {
                    lp.ms_ids.push_back(idx);
                    lp.ms_rank.push_back((uint32_t)r * rank_step);
                    lp.max_ms_streams = std::max<uint32_t>(lp.max_ms_streams, n_streams);
                } else {
                    lp.or_ids.push_back(idx);
                    lp.or_rank.push_back((uint32_t)r * rank_step);
                    lp.max_or_terms = std::max<uint32_t>(lp.max_or_terms, n_item_terms);
                    if (!nots.empty()) lp.or_has_not = true;
                    if (!item_pos) lp.or_nonpos = true;
                    if (shape.msm) lp.or_has_msm = true;
                    if (leaf_dismax) lp.or_has_dmax = true;
                }
            }
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
        struct Off { size_t items, clauses, or_ids, ms_ids, and_ids, ro_ids, dpq_ids, groups; };
        std::vector<Off> off(n_threads + 1, Off{0, 0, 0, 0, 0, 0, 0, 0});
        for (uint32_t t = 0; t < n_threads; t++) {
            const HostPlan& lp = parts[t];
            off[t + 1] = Off{off[t].items + lp.items.size(), off[t].clauses + lp.clauses.size(), off[t].or_ids + lp.or_ids.size(),
                             off[t].ms_ids + lp.ms_ids.size(), off[t].and_ids + lp.and_ids.size(), off[t].ro_ids + lp.ro_ids.size(),
                             off[t].dpq_ids + lp.dpq_ids.size(), off[t].groups + lp.group_out.size()};
            hp.postings += lp.postings;
            hp.algo_bytes += lp.algo_bytes;
            hp.max_or_terms = std::max(hp.max_or_terms, lp.max_or_terms);
            hp.max_ms_streams = std::max(hp.max_ms_streams, lp.max_ms_streams);
            hp.max_dpq_terms = std::max(hp.max_dpq_terms, lp.max_dpq_terms);
            hp.or_has_not = hp.or_has_not || lp.or_has_not;
            hp.or_nonpos = hp.or_nonpos || lp.or_nonpos;
            hp.or_has_msm = hp.or_has_msm || lp.or_has_msm;
            hp.or_has_dmax = hp.or_has_dmax || lp.or_has_dmax;
        }
        const Off& end = off[n_threads];
        hp.items.resize(end.items);
        hp.clauses.resize(end.clauses);
        hp.or_ids.resize(end.or_ids);
        hp.or_rank.resize(end.or_ids);
        hp.ms_ids.resize(end.ms_ids);
        hp.ms_rank.resize(end.ms_ids);
        hp.and_ids.resize(end.and_ids);
        hp.and_rank.resize(end.and_ids);
        hp.ro_ids.resize(end.ro_ids);
        hp.dpq_ids.resize(end.dpq_ids);
        hp.group_out.resize(end.groups);
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
                auto put_ids = [&](std::vector<uint32_t>& dst, size_t at, const std::vector<uint32_t>& src) {
                    for (size_t i = 0; i < src.size(); i++) dst[at + i] = src[i] + item_off;
                };
                put_ids(hp.or_ids, o.or_ids, lp.or_ids);
                put_ids(hp.ms_ids, o.ms_ids, lp.ms_ids);
                put_ids(hp.and_ids, o.and_ids, lp.and_ids);
                put_ids(hp.ro_ids, o.ro_ids, lp.ro_ids);
                put_ids(hp.dpq_ids, o.dpq_ids, lp.dpq_ids);
                std::copy(lp.or_rank.begin(), lp.or_rank.end(), hp.or_rank.begin() + o.or_ids);
                std::copy(lp.ms_rank.begin(), lp.ms_rank.end(), hp.ms_rank.begin() + o.ms_ids);
                std::copy(lp.and_rank.begin(), lp.and_rank.end(), hp.and_rank.begin() + o.and_ids);
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
    by_rank(hp.or_ids, hp.or_rank);
    by_rank(hp.ms_ids, hp.ms_rank);
    by_rank(hp.and_ids, hp.and_rank);
    // heap groups = contiguous item runs starting at chain-start items
    for (uint32_t i = 0; i < hp.items.size(); i++)
        if (hp.items[i].chain_pos == 0) hp.group_item_begin.push_back(i);
    hp.group_item_begin.push_back((uint32_t)hp.items.size());
    if (hp.group_item_begin.size() != hp.group_out.size() + 1) throw ArgError("internal: group bookkeeping mismatch");
    tm.mark("order");
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

}  // namespace

#define RG_TRY try {
#define RG_CATCH \
    }            \
    catch (...) { return translate_exception(); }

extern "C" {

int rg_batch_prepare(rg_engine* e, const rg_query* queries, uint32_t n_queries,
                     const rg_clause* clauses, uint32_t n_clauses, const rg_search_params* p,
                     rg_batch** out) {
    RG_TRY
    if (!e || !p || !out || (n_queries && !queries) || (n_clauses && !clauses)) throw ArgError("null argument");
    *out = nullptr;
    if (p->k == 0) throw ArgError("k must be >= 1");
    if (p->k > 1024) throw Unsupported("k > 1024 is not accelerated");
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
    plan_batch(e, queries, n_queries, clauses, n_clauses, p->mode, p->k1, hp, tm, scratch);
    std::unique_ptr<rg_batch> b(new rg_batch());
    b->generation = e->generation;
    b->cols = std::move(hp.cols);
    b->lists = std::move(hp.lists);
    b->n_cols_built = hp.n_cols_built;
    b->n_lists_built = hp.n_lists_built;
    b->list_floats = hp.list_floats;
    b->col_floats = hp.col_floats;
    b->n_ms = (uint32_t)hp.ms_ids.size();
    b->max_ms_streams = hp.max_ms_streams;
    for (const ColRef& r : hp.col_refs) b->uses_planes = b->uses_planes || r.hi1 != nullptr;
    b->n_dpq = (uint32_t)hp.dpq_ids.size();
    b->max_dpq_terms = hp.max_dpq_terms;
    b->n_queries = n_queries;
    b->k = p->k;
    b->mode = p->mode;
    b->k1 = p->k1;
    b->n_items = (uint32_t)hp.items.size();
    b->n_or = (uint32_t)hp.or_ids.size();
    b->n_and = (uint32_t)hp.and_ids.size();
    b->n_ro = (uint32_t)hp.ro_ids.size();
    b->n_groups = (uint32_t)hp.group_out.size();
    b->max_or_terms = hp.max_or_terms;
    b->or_has_not = hp.or_has_not;
    b->or_nonpos = hp.or_nonpos;
    b->or_has_msm = hp.or_has_msm;
    b->or_has_dmax = hp.or_has_dmax;
    b->n_leaves = (uint32_t)e->segs.size();
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
    carve(b->or_ids, hp.or_ids.size());
    carve(b->and_ids, hp.and_ids.size());
    carve(b->ms_ids, hp.ms_ids.size());
    carve(b->dpq_ids, hp.dpq_ids.size());
    carve(b->ro_ids, hp.ro_ids.size());
    carve(b->col_refs, hp.col_refs.size());
    carve(b->group_item_begin, hp.group_item_begin.size());
    carve(b->group_out, hp.group_out.size());
    // running top-k scores of every OR work item (theta inheritance along a heap chain); skipped when it would
    // not fit comfortably (huge batches with k near 1024): theta then falls back to the per-range bound
    b->topk_cap = (std::min<uint32_t>(p->k, 1024u) + 31u) & ~31u;
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
    rebase(b->items); rebase(b->clauses); rebase(b->or_ids); rebase(b->and_ids); rebase(b->ms_ids); rebase(b->dpq_ids); rebase(b->ro_ids); rebase(b->col_refs);
    rebase(b->group_item_begin); rebase(b->group_out); rebase(b->item_head); rebase(b->item_matches);
    rebase(b->item_theta); rebase(b->item_topk_n); rebase(b->item_topk); rebase(b->arena_next); rebase(b->dbg); rebase(b->out_hits); rebase(b->out_counts);
    rebase(b->out_total);
    if (p->mode == RG_MODE_SEARCH_PARALLEL) rebase(b->leaf_records);
    b->zero_begin = b->slab.p + zero_off;
    b->zero_bytes = off - zero_off;
    cudaStream_t cs = e->copy_stream;
    up(b->items, hp.items, cs);
    up(b->clauses, hp.clauses, cs);
    up(b->or_ids, hp.or_ids, cs);
    up(b->and_ids, hp.and_ids, cs);
    up(b->ms_ids, hp.ms_ids, cs);
    up(b->dpq_ids, hp.dpq_ids, cs);
    up(b->ro_ids, hp.ro_ids, cs);
    up(b->col_refs, hp.col_refs, cs);
    up(b->group_item_begin, hp.group_item_begin, cs);
    up(b->group_out, hp.group_out, cs);
    RG_CUDA_CHECK(cudaEventCreateWithFlags(&b->uploaded, cudaEventDisableTiming));
    RG_CUDA_CHECK(cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming));
    for (auto& x : b->ev) RG_CUDA_CHECK(cudaEventCreate(&x));
    RG_CUDA_CHECK(cudaEventRecord(b->uploaded, cs));
    b->h2d_bytes = (hp.items.size() * sizeof(WorkItem)) + hp.clauses.size() * sizeof(ItemClause) +
                   4 * (hp.or_ids.size() + hp.ms_ids.size() + hp.dpq_ids.size() + hp.and_ids.size() + hp.ro_ids.size() + hp.group_item_begin.size() + hp.group_out.size()) +
                   hp.col_refs.size() * sizeof(ColRef);
    b->kernels_per_run = (b->n_ms ? 1 : 0) + (b->n_dpq ? 1 : 0) + (b->n_or ? 1 : 0) + (b->n_and ? 1 : 0) + (b->n_ro ? 1 : 0) + (b->n_groups ? 1 : 0) +
                         (p->mode == RG_MODE_SEARCH_PARALLEL ? 1 : 0);
    tm.mark("alloc_copy_issue");
    RG_CUDA_CHECK(cudaStreamSynchronize(cs));  // the host vectors go out of scope (a running batch is not waited for)
    tm.mark("sync");
    *out = b.release();
    return RG_OK;
    RG_CATCH
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
    RG_CUDA_CHECK(cudaEventRecord(b->ev[2], st));
    ep.cols = b->col_refs.p;
    bool has_live = false, has_other = false;
    for (const Segment& sg : e->segs) {
        has_live = has_live || sg.live.p != nullptr;
        has_other = has_other || sg.has_other_enc;
    }
    launch_eval_or_ms(st, ep, b->ms_ids.p, b->n_ms, b->max_ms_streams, has_live, b->uses_planes);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_or(st, ep, b->or_ids.p, b->n_or, b->max_or_terms, has_live, b->or_has_not, b->or_has_msm, b->or_has_dmax,
                   !b->or_nonpos);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_dpq(st, ep, b->dpq_ids.p, b->n_dpq, b->max_dpq_terms, has_live);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and(st, ep, b->and_ids.p, b->n_and, false, has_other);
    RG_CUDA_CHECK(cudaGetLastError());
    launch_eval_and(st, ep, b->ro_ids.p, b->n_ro, true, has_other);
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
    if (e && b->ran && !b->synced) cudaEventSynchronize(b->done);
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
    out[6] = b->n_or + b->n_ms + b->n_dpq;
    out[7] = b->n_and + b->n_ro;
    return RG_OK;
    RG_CATCH
}

int rg_search_batch(rg_engine* e, const rg_query* queries, uint32_t n_queries,
                    const rg_clause* clauses, uint32_t n_clauses, const rg_search_params* p,
                    rg_hit* out_hits, uint32_t* out_counts, uint64_t* out_total_hits) {
    rg_batch* b = nullptr;
    int rc = rg_batch_prepare(e, queries, n_queries, clauses, n_clauses, p, &b);
    if (rc != RG_OK) return rc;
    rc = rg_batch_run(e, b);
    if (rc == RG_OK) rc = rg_batch_fetch(e, b, out_hits, out_counts, out_total_hits);
    rg_batch_destroy(e, b);
    if (rc == RG_ENOMEM && n_queries > 1 && p && p->k) {
        // the candidate arena overflowed: the two halves of the batch, one after the other (queries are independent and
        // refer to `clauses` by absolute index, so a half is just a sub-array of `queries`); recursively if need be
        const uint32_t h = n_queries / 2;
        rc = rg_search_batch(e, queries, h, clauses, n_clauses, p, out_hits, out_counts, out_total_hits);
        if (rc == RG_OK)
            rc = rg_search_batch(e, queries + h, n_queries - h, clauses, n_clauses, p, out_hits + (size_t)h * p->k, out_counts + h,
                                 out_total_hits + h);
    }
    return rc;
}

int rg_batch_debug(rg_engine* e, rg_batch* b, uint64_t out[16]) {
    RG_TRY
    if (!e || !b || !out) throw ArgError("null argument");
    memset(out, 0, 16 * sizeof(uint64_t));
    if (b->ran) {
        RG_CUDA_CHECK(cudaStreamSynchronize(e->stream));
        RG_CUDA_CHECK(cudaMemcpy(out, b->dbg.p, 16 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    }
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
    if (k == 0 || k > 1024) throw ArgError("k out of range");
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
