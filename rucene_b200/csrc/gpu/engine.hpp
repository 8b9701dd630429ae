// engine.hpp — host-side engine state and kernel launch prototypes (internal).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <deque>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace rg {

struct CudaError : std::runtime_error {
    cudaError_t code;
    CudaError(cudaError_t e, const char* expr, const char* file, int line)
        : std::runtime_error(std::string(cudaGetErrorString(e)) + " at " + file + ":" +
                             std::to_string(line) + " (" + expr + ")"),
          code(e) {}
};
struct ArgError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct Unsupported : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct OutOfArena : std::runtime_error {
    using std::runtime_error::runtime_error;
};

template <class T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p;
            n = o.n;
            o.p = nullptr;
            o.n = 0;
        }
        return *this;
    }
    ~DevBuf() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
    void alloc(size_t count) {
        release();
        if (count == 0) return;
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), count * sizeof(T));
        if (e != cudaSuccess) throw CudaError(e, "cudaMalloc", __FILE__, __LINE__);
        n = count;
    }
    size_t bytes() const { return n * sizeof(T); }
};

// A score column as the kernels see it: f32 BM25 contribution per leaf-local docid (+0.0f = no
// posting) + the term's presence bitmap (null when the term has none).
struct ColRef {
    const float* col;
    const uint32_t* bits;
    const uint32_t* hi1;  // plane "tf-norm factor above tau1" of the term for the clause's norm cache (null: none)
    const uint32_t* hi2;  // plane "... above tau2" (a subset of hi1)
    float tau1, tau2;
};

// BM25's tf-norm factor f/(f+norm) of most postings is far below 1 (f = 1 in an average-length doc gives 0.45; where
// norms say "long document" much less).  For every bitmap term two more bits per docid say "this posting's factor is
// above tau1" / "above tau2", tau1 <= tau2 being the term's 90th and 99th percentile of the factor for one norm cache
// and k1 (taken from a histogram over a sample of its blocks), so the per-document score bound of k_eval_or_ms can
// count tau1*ub, tau2*ub or ub.  One buffer per (segment, cache id, k1), built for all bitmap terms of the segment the
// first time a batch needs it.  ANY thresholds give correct results; the percentiles make the bound tight.
struct TfPlanes {
    DevBuf<uint32_t> bits;     // [2][n bitmap terms][bitmap_words], slot order of Segment::bitmaps
    std::vector<float> tau1, tau2;  // per slot
};

// Persistent score column (engine-owned, LRU): the contributions of one (leaf, term, weight, norm
// cache, k1) are the same f32 values for every query that carries the clause, in this batch and in
// later ones, so they are materialised once and kept while HBM allows.
using ColKey = std::tuple<uint32_t, uint32_t, uint32_t, uint32_t, uint32_t>;  // leaf, term, weight bits, cache, k1 bits
struct ColKeyHash {
    size_t operator()(const ColKey& k) const {
        uint64_t h = ((uint64_t)std::get<0>(k) << 32 | std::get<1>(k)) * 0x9e3779b97f4a7c15ull;
        h ^= ((uint64_t)std::get<2>(k) << 32 | std::get<3>(k)) * 0xc2b2ae3d27d4eb4full + (h >> 29);
        h ^= (uint64_t)std::get<4>(k) * 0x165667b19e3779f9ull + (h >> 31);
        return (size_t)(h ^ (h >> 32));
    }
};
struct ColEntry {
    ColKey key;
    float* col = nullptr;  // len floats: its own cudaMalloc (score column) or a piece of the engine's list arena
    bool in_arena = false;
    const uint32_t* bits = nullptr;
    uint64_t len = 0;
    uint64_t last_use = 0;
    ~ColEntry() {
        if (col && !in_arena) cudaFree(col);
    }
};

// host-side view of a term (for planning and byte accounting)
struct TermHost {
    int32_t doc_freq = 0;
    uint32_t n_blocks = 0;
    uint64_t enc_bytes = 0;  // encoded block bytes incl. header bytes + vint tail bytes
    uint32_t tail_n = 0;     // postings in the vint tail (1 for a singleton)
    int32_t tail_base = 0;   // last doc of the last full block
};

struct Segment {
    SegDev dev{};
    DevBuf<uint4> arena;
    DevBuf<int32_t> blk_last;
    DevBuf<BlockDesc> blk_desc;
    DevBuf<uint8_t> tails;
    DevBuf<TermDev> terms;
    DevBuf<uint8_t> norms;
    DevBuf<uint64_t> live;
    bool has_other_enc = false;  // some doc block is EF / BITSET encoded
    uint64_t n_blocks_total = 0;
    uint64_t block_enc_bytes = 0;  // sum over block pairs of (1 + payload) per part, as the codec wrote them
    // Presence bitmaps of the dense terms (df >= max_doc / kBitmapDen, largest first, within a byte
    // budget): bit d of a term's bitmap = "the term has a posting on docid d".  Built once at upload
    // (k_build_bitmaps); total_hits of a disjunction is then a popcount over ORed words and the
    // non-essential clauses of k_eval_or_ms never have to be decoded.  bitmap_words = words per term
    // (max_doc/32 rounded up + 64 zero words so a 1024-doc window may read past max_doc).
    DevBuf<uint32_t> bitmaps;
    uint64_t bitmap_words = 0;
    std::vector<int32_t> bitmap_slot;  // per term: index of its bitmap, -1 = none
    uint8_t norm_seen[256] = {0};      // norm byte values that occur in this leaf (all zero: the leaf has no norms)
    std::vector<uint8_t> cache_small;  // per norm cache: every entry a norm byte of this leaf selects is in [0, 1e10]
    std::vector<uint32_t> bitmap_terms;  // slot -> term id
    std::map<std::pair<uint32_t, uint32_t>, TfPlanes> tf_planes;  // (cache id, k1 bits) -> high tf-norm planes
    std::vector<TermHost> host_terms;
    // terms dictionary for exact lookups on the device (terms_dict.cu): sorted term bytes + engine-wide ids
    DevBuf<uint8_t> dict_bytes;
    DevBuf<uint64_t> dict_off;
    DevBuf<uint32_t> dict_ids;
    uint32_t dict_n = 0;
    bool has_dict = false;
    int32_t doc_base = 0, max_doc = 0;
    uint64_t device_bytes = 0;
};

// kernel launchers (decode_kernels.cu)
void launch_decode_staged(cudaStream_t st, const uint4* arena, const BlockDesc* desc,
                          uint32_t n_blocks, int32_t* out, int version, uint32_t sb_mask);
void launch_decode_segment(cudaStream_t st, const uint4* arena, const BlockDesc* desc, uint32_t first,
                           uint32_t n_blocks, int32_t* out, int version, uint32_t sb_mask);
void launch_decode_raw(cudaStream_t st, const uint8_t* stream, const uint64_t* offsets,
                       uint32_t n_blocks, int32_t* out, int version, uint32_t sb_mask);

// query kernels (query_kernels.cu)
struct EvalParams {
    const SegDev* segs;
    const WorkItem* items;
    const ItemClause* clauses;
    const float* caches;       // n_caches * 256
    const ColRef* cols;        // score columns referenced by this batch (see k_build_columns)
    uint32_t n_items;
    uint32_t k;
    float k1;
    // outputs / scratch
    rg_hit* cand_arena;        // slot array; slot 0.. ; run = header slot + entries
    uint32_t arena_slots;
    unsigned long long* arena_next;  // bump pointer (slots)
    uint32_t* item_head;       // first run header slot per item (0xffffffff none)
    uint32_t* item_matches;    // matches per item (total_hits contribution)
    uint32_t* item_theta;      // ordered-uint running k-th best, chained item -> item+1
    float* item_topk;          // [n_items][kcap] running top-k scores per item (see wtheta_inherit), may be null
    uint32_t* item_topk_n;     // entries published per item
    uint32_t* error_flag;      // bit0: arena exhausted
    unsigned long long* dbg;   // optional event counters of k_eval_or_ms (RG_CFG_STATS), else null
    unsigned long long* touched;  // bytes k_eval_and actually asked for: decoded blocks + tables + gathers (its roofline)
};
// one score column to materialise: the BM25 contributions of (leaf, term, weight, norm cache, k1);
// a bitmap job (weight unused) sets presence bits instead
struct ColumnJob {
    uint32_t seg, term_id, cache_id;
    float weight;         // idf * boost, as in the clause
    void* dst;            // float* column (leaf-local docid index) or uint32_t* bitmap
    uint32_t unit_begin;  // first work unit (block / tail) of this job in the launch
    uint32_t pad;
};
void launch_build_columns(cudaStream_t st, const SegDev* segs, const ColumnJob* jobs, uint32_t n_jobs,
                          uint32_t n_units, const float* caches, float k1);
// scored posting lists: job.dst = uint4[units * 64], unit = block or vint tail of the job's term
void launch_build_lists(cudaStream_t st, const SegDev* segs, const ColumnJob* jobs, uint32_t n_jobs, uint32_t n_units,
                        const float* caches, float k1);
void launch_build_bitmaps(cudaStream_t st, const SegDev* seg, const ColumnJob* jobs, uint32_t n_jobs,
                          uint32_t n_units);
// jobs carry cache_id.  hist != null: every 8th block of a job adds its postings' factors (rounded up, 256 bins) to
// hist[job][256].  Else: a posting sets its bit in job.dst when its factor exceeds job.weight (tau1) and in
// job.dst + plane_stride when it exceeds job.pad (the bits of tau2).
void launch_build_tf_planes(cudaStream_t st, const SegDev* segs, const ColumnJob* jobs, uint32_t n_jobs,
                            uint32_t n_units, const float* caches, float k1, uint32_t* hist, size_t plane_stride);
// recompute Segment::cache_small for every (leaf, norm cache) — after an upload and after rg_norm_cache_set
void refresh_cache_small(rg_engine* e);
void launch_eval_or(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n,
                    uint32_t max_terms, bool has_live, bool has_not, bool has_msm, bool has_dmax, bool all_pos);
// eval_dpq.cu: disjunctions with >= 10 clauses in a leaf (DisiPriorityQueue order), one warp per (query, leaf)
void launch_eval_dpq(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, uint32_t max_terms,
                     bool has_live);
// eval_or_ms.cu: pure-SHOULD sum disjunctions whose dense clauses all have a score column + bitmap
void launch_eval_or_ms(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n,
                       uint32_t max_streams, bool has_live, bool planes);
void launch_eval_and(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, bool req_opt,
                     bool has_other_enc);

struct ReplayParams {
    const rg_hit* cand_arena;
    const uint32_t* item_head;
    const uint32_t* item_matches;
    const uint32_t* group_item_begin;  // n_groups+1 : items of heap group g
    const uint32_t* group_query;       // query of group g
    uint32_t n_groups;
    uint32_t k;
    // outputs: sorted hits per group or leaf records
    rg_hit* out_hits;        // [n_groups * k] sorted (descending) — used when !leaf_records
    uint32_t* out_counts;
    unsigned long long* out_total;
    uint8_t* leaf_records;   // non-null: write {u32 n; u32 pad; u64 total; rg_hit heap[k]} per group
};
void launch_heap_replay(cudaStream_t st, const ReplayParams& p);
// finish_parallel over leaf records laid out [leaf][query]
void launch_merge_leaf_records(cudaStream_t st, const uint8_t* records, uint32_t n_leaves,
                               uint32_t n_queries, uint32_t k, rg_hit* out_hits,
                               uint32_t* out_counts, unsigned long long* out_total);

__host__ __device__ inline size_t leaf_record_bytes(uint32_t k) { return 16 + (size_t)k * sizeof(rg_hit); }

extern thread_local std::string g_last_error;
int translate_exception();  // maps the in-flight exception to an RG_E* code + g_last_error

}  // namespace rg

// the opaque handle of include/rucene_gpu.h
struct rg_engine {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;  // plan uploads and result fetches: they must not queue behind a running batch
    cudaStream_t stream = nullptr;
    rg_config cfg{};
    std::vector<rg::Segment> segs;
    rg::DevBuf<rg::SegDev> d_segs;
    bool segs_dirty = true;
    rg::DevBuf<float> d_caches;   // n_caches * 256
    std::vector<float> h_caches;
    bool caches_dirty = true;
    rg::DevBuf<rg_hit> cand_arena;
    // persistent score columns: map-resident entries count against col_budget_floats (1/3 of the free
    // HBM when first needed); batches hold shared_ptrs, so an evicted / invalidated column lives until
    // the last batch that references it is destroyed
    std::map<rg::ColKey, std::shared_ptr<rg::ColEntry>> col_cache;
    uint64_t col_floats = 0;            // floats held by map-resident entries
    uint64_t col_budget_floats = 0;     // 0 = not computed yet (reset by rg_segment_upload)
    uint64_t col_tick = 0, col_builds = 0, col_hits = 0;
    // persistent scored posting lists (same key, same budget and LRU clock as the columns)
    std::map<rg::ColKey, std::shared_ptr<rg::ColEntry>> list_cache;
    uint64_t list_floats = 0, list_builds = 0, list_hits = 0;
    rg::DevBuf<rg::ColumnJob> list_jobs[4];  // grow-only, round robin: the build kernel reads one in stream order
    cudaEvent_t list_jobs_done[4] = {nullptr, nullptr, nullptr, nullptr};  // ... and this says when it is done with it
    uint32_t list_jobs_next = 0;
    // The lists live in one arena allocated at first need (a cudaMalloc per batch costs more than building the lists):
    // a ring of slabs, one per rg_batch_prepare that built something; space is reclaimed oldest slab first, and only
    // when no batch still references one of its lists.
    struct ListSlab {
        uint64_t off, len;
        std::vector<std::shared_ptr<rg::ColEntry>> entries;
    };
    rg::DevBuf<float> list_arena;
    uint64_t list_head = 0;  // next free float of the ring
    std::deque<ListSlab> list_slabs;
    bool list_arena_tried = false;
    // the exhaustive disjunction kernel scans a score column docid by docid: that beats streaming the clause's postings
    // (scored list) for df >= max_doc / or_col_den; measured on C4 (one H100 at 400 W, 256 ranges per leaf):
    // 1/4 641 ms, 1/8 627, 1/16 669 per step
    uint64_t or_col_den = 8;
    bool range_postings_set = false;  // rg_config.range_postings was given (else the planner chooses per batch)
    uint64_t generation = 1;            // bumped by rg_segment_upload / rg_norm_cache_set (stale-batch check)
    std::vector<uint8_t> cache_nonneg;  // per norm cache: every entry >= 0 (MaxScore bound needs it)
    rg::DevBuf<uint8_t> merge_scratch;  // rg_merge_leaf_records outputs (grow-only)
    rg::DevBuf<uint8_t> gather_scratch; // rg_batch_run_sharded: all ranks' leaf records (grow-only)
    uint32_t merged_queries = 0, merged_k = 0;  // shape of the result sitting in merge_scratch
    std::shared_ptr<void> plan_scratch;  // host-side plan buffers kept between rg_batch_prepare calls (search.cu: PlanScratch)
    std::vector<rg::DevBuf<uint8_t>> spare_slabs;  // device slabs of destroyed batches (at most 3), reused by the next ones
    uint64_t launches = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
    float last_decode_ms = -1.f, last_eval_ms = -1.f, last_replay_ms = -1.f, last_run_ms = -1.f;
    void sync_tables();  // (re)upload SegDev array and norm caches when dirty
};

namespace rg {

}  // namespace rg
