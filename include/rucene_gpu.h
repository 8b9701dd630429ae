/*
 * rucene_gpu.h — C ABI of the H100 query-evaluation engine (librucene_gpu.so).
 *
 * The reference (zhihu/rucene) has no FFI for this path: the hot path sits behind Rust
 * traits.  Each entry point below names the reference interface it replaces; paths are
 * relative to src/core/ of zhihu/rucene.  A Rust shim implementing `IndexSearcher<C>` binds
 * exactly these symbols (see INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes, no exceptions across the boundary; every function
 * returns 0 on success or a negative RG_E* code, with a message in rg_last_error().
 * Handles are engine-owned; output buffers are caller-owned.  There is NO CPU fallback:
 * without a CUDA device every compute entry point fails with RG_ENODEVICE.
 */
#ifndef RUCENE_GPU_H
#define RUCENE_GPU_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define RG_OK 0
#define RG_EINVAL (-1)      /* bad argument / corrupt index bytes */
#define RG_ENODEVICE (-2)   /* no usable CUDA device */
#define RG_ECUDA (-3)       /* CUDA runtime error */
#define RG_EUNSUPPORTED (-4)/* plan shape outside the accelerated path: caller falls back to
                               DefaultIndexSearcher (searcher.rs:487-525) */
#define RG_ENOMEM (-5)      /* candidate arena exhausted: split the batch (rg_search_batch does so itself; the split
                               calls rg_batch_prepare/run/fetch report it to the caller) */

#define RG_NO_MORE_DOCS 0x7fffffff /* search/mod.rs:59 */

/* rg_config.flags.  Presence bitmaps: every term with df >= max_doc/64 (max_doc/1024 when the engine is created
 * with RG_CFG_MAXSCORE; largest first, within a byte budget) gets a bitmap over the leaf's docids at upload.  Score columns: the BM25 contributions of
 * such a term for one (weight, norm cache, k1) are materialised into a docid-indexed f32 column (the
 * same f32 values the per-query path computes) the first time two clauses of a batch share them, kept
 * across batches (LRU within 1/3 of the free HBM) and read from there. */
#define RG_CFG_NO_COLUMNS 1u    /* never materialise score columns */
#define RG_CFG_EAGER_COLUMNS 2u /* a column for every disjunction clause with df >= max_doc/64 (tests) */
#define RG_CFG_NO_BITMAPS 4u    /* no presence bitmaps at upload (and therefore no score columns) */
#define RG_CFG_MAXSCORE 8u      /* plain sum disjunctions that have a bitmap clause go to k_eval_or_ms (presence bitmaps for
                                   df >= max_doc/1024, bit-sliced per-document score bound) instead of the exhaustive
                                   k_eval_or.  On the benchmark index the two are equally fast on one GPU and the exhaustive
                                   kernel scales better to small leaves (DESIGN.md section 6); off by default */
#define RG_CFG_TFPLANES 32u     /* (with RG_CFG_MAXSCORE) build and use tf-norm planes: the per-document score bound of k_eval_or_ms then knows three
                                   levels of a posting's BM25 tf-norm factor instead of presence only.  Cuts the docs it has
                                   to score ~16x, but scanning three planes costs more than it saves on the benchmark index
                                   (DESIGN.md section 6); off by default */
#define RG_CFG_NO_LISTS 64u     /* never materialise scored posting lists: a disjunction clause (df >= 4096) that two clauses of a batch share
                                   is decoded and BM25-scored ONCE into (docid, f32 score) pairs, 1 KB per 128-posting block, kept
                                   across batches in the engine's list arena (a sixth of the free HBM, reclaimed oldest first); k_eval_or then streams the pairs
                                   instead of unpacking, prefix-summing, gathering norms and dividing per query */
#define RG_CFG_STATS 16u        /* count events inside k_eval_or_ms (rg_batch_debug); costs a few atomics per work item */

/* Environment variables read by the library (diagnostics / tuning sweeps; none is needed in production):
 * RG_PLAN_TIMING=1 prints where rg_batch_prepare's host time goes; RG_OR_COL_DEN=n reads a disjunction clause from its
 * score column when df >= max_doc/n (default 8); RG_MAX_RANGES=n caps the docid ranges per (query, leaf) (default 256);
 * RG_LIST_ARENA_KB=n sizes the scored-list arena (default: a sixth of the free HBM, at most 24 GiB). */

typedef struct rg_engine rg_engine;
typedef struct rg_batch rg_batch;
typedef struct rg_blockset rg_blockset;

typedef struct {
    int32_t device;            /* CUDA ordinal; -1 = current device */
    uint64_t cand_arena_bytes; /* candidate arena for exact top-k replay; 0 = default */
    uint32_t range_postings;   /* target postings per (query, docid-range) work item; 0 = the planner chooses per batch
                                  (32 K for conjunctions, 8 K..128 K for disjunctions depending on the batch's size) */
    uint32_t flags;            /* RG_CFG_* */
} rg_config;

/* Per-term, per-segment handle == BlockTermState
 * (codec/postings/blocktree/mod.rs:33-59; filled by lucene50_decode_term,
 * codec/postings/posting_reader.rs:264-306).  doc_freq==0: term absent in the segment
 * (Weight::create_scorer returns None, search/query/mod.rs:139). */
typedef struct {
    int32_t doc_freq;
    int32_t singleton_doc_id; /* docid when doc_freq==1, else -1 */
    int64_t total_term_freq;
    int64_t doc_start_fp;     /* into the .doc file */
    int64_t skip_offset;      /* relative to doc_start_fp; -1 when doc_freq<=128 */
} rg_term_state;

/* BooleanClause occur (search/query/boolean_query.rs:30-36: must/should/filter/must_not lists).
 * RG_FILTER: a required clause that does not score — its weight is built with needs_scores = false
 * (boolean_query.rs:108-110), i.e. NonScoringSimilarity, score 0f32 (searcher.rs:158-197); the clause's
 * `weight` is ignored.  A query whose only clause is a FILTER is the reference's
 * ConstantScoreQuery::with_boost(filter, 0) (boolean_query.rs:66-75): the term's docs with score 0. */
enum { RG_MUST = 0, RG_SHOULD = 1, RG_MUST_NOT = 2, RG_FILTER = 3 };

/* One TermQuery leaf of the plan, with what TermWeight carries after
 * BM25Similarity::compute_weight (search/similarity/bm25_similarity.rs:151-177):
 *   weight   = idf * boost                       (:363-366)
 *   cache_id = which 256-entry norm cache (:161-165) registered by rg_norm_cache_set. */
typedef struct {
    int32_t occur;
    uint32_t term_id;
    float weight;
    uint32_t cache_id;
} rg_clause;

/* flags */
#define RG_Q_BOOLEAN 1u /* built by BooleanQuery::build (boolean_query.rs:40-87); without it
                           the query is a bare TermQuery and n_clauses must be 1 */
#define RG_Q_DISMAX 2u  /* built by DisjunctionMaxQuery::build over TermQuerys
                           (search/query/disjunction_max_query.rs:51-68): the clauses are the disjuncts
                           (occur is ignored), min_should_match carries the BITS of the f32
                           tie_breaker_multiplier; score = max + (sum - max) * tie_breaker
                           (search/scorer/disjunction_scorer.rs:241-263) */
typedef struct {
    uint32_t clause_begin; /* index into the clause array */
    uint32_t n_clauses;
    int32_t min_should_match; /* as passed to BooleanQuery::build (RG_Q_DISMAX: f32 bits, see above) */
    uint32_t flags;
} rg_query;

/* ScoreDoc (search/sort_field/collapse_top_docs.rs:22-27), global docid = doc + doc_base
 * (search/collector/top_docs.rs:89). */
typedef struct {
    int32_t doc;
    float score;
} rg_hit;

#define RG_MODE_SEARCH 0          /* IndexSearcher::search, searcher.rs:487-525 */
#define RG_MODE_SEARCH_PARALLEL 1 /* search_parallel, searcher.rs:527-630: one TopDocs heap per
                                     leaf, merged in leaf order (top_docs.rs:157-172) */
typedef struct {
    uint32_t k;    /* TopDocsCollector::new(k), search/collector/top_docs.rs:107-113 */
    float k1;      /* BM25Similarity k1, bm25_similarity.rs:45 */
    uint32_t mode; /* RG_MODE_* */
    uint32_t reserved;
} rg_search_params;

/* ---------------------------------------------------------------- engine ---------- */
int rg_engine_create(const rg_config* cfg, rg_engine** out);
void rg_engine_destroy(rg_engine* e);
/* Message for the last failure on this thread (engine may be NULL). */
const char* rg_last_error(rg_engine* e);
/* Launch on this cudaStream_t (e.g. torch's current stream); NULL = the engine's own stream. */
int rg_engine_set_stream(rg_engine* e, void* cuda_stream);
/* Change rg_config.flags of a live engine (planning-time flags take effect with the next
 * rg_batch_prepare; RG_CFG_NO_BITMAPS only affects later uploads). */
int rg_engine_set_flags(rg_engine* e, uint32_t flags);
/* Persistent score columns: [0]=columns cached, [1]=their bytes in HBM, [2]=columns built so far,
 * [3]=cache hits so far. */
int rg_engine_column_stats(rg_engine* e, uint64_t out[4]);
/* Persistent scored posting lists (see RG_CFG_NO_LISTS), same four figures. */
int rg_engine_list_stats(rg_engine* e, uint64_t out[4]);
/* Number of this library's kernels launched so far (bench.py's gpu_launches). */
uint64_t rg_engine_launch_count(rg_engine* e);
/* Device-side timing of the last rg_batch_run / rg_blockset_decode, CUDA events on the launch
 * stream.  Returns milliseconds, <0 if nothing was timed. */
float rg_engine_last_kernel_ms(rg_engine* e, const char* which);

/* ---------------------------------------------------------------- index ---------- */
/* Replaces Lucene50PostingsReader::open + LeafReader::{postings,norm_values,live_docs}
 * (codec/postings/posting_reader.rs:85-158, index/reader/leaf_reader.rs:92-104).
 * doc_file: the whole `.doc` file (IndexHeader, ForUtil table, term regions, footer) of a
 * DocsAndFreqs field.  norms: max_doc bytes (Lucene53 norms, bytes_per_value==1) or NULL.
 * live_docs: FixedBitSet words (bit doc&63 of word doc>>6) or NULL for "all live".
 * terms[term_id]: the segment's BlockTermState per engine-wide term id (doc_freq 0 = absent).
 * Segments must be uploaded in leaf order with seg_ord 0,1,2...; doc_base as in
 * LeafReaderContext (leaf_reader.rs:195-202). Host buffers may be freed on return. */
int rg_segment_upload(rg_engine* e, uint32_t seg_ord, int32_t doc_base, int32_t max_doc,
                      const uint8_t* doc_file, size_t doc_len, const uint8_t* norms,
                      const uint64_t* live_docs, const rg_term_state* terms, uint32_t n_terms);
/* Terms dictionary of an uploaded segment, for exact lookups on the device: replaces the per-query
 * SegmentTermIterator::seek_exact (codec/postings/blocktree/blocktree_reader.rs:1364, term_iter_frame.rs:436) +
 * decode_term (posting_reader.rs:264-306) of TermQuery::create_weight / TermWeight::create_scorer.
 * bytes: the field's terms concatenated in dictionary order (sorted unsigned bytewise, unique — the order the
 * BlockTree iterates them); offsets[n_terms + 1]; term_ids[i] = engine-wide term id of entry i (its row in the
 * rg_term_state table of rg_segment_upload), NULL = i. */
int rg_terms_upload(rg_engine* e, uint32_t seg_ord, const uint8_t* bytes, const uint64_t* offsets,
                    const uint32_t* term_ids, uint32_t n_terms);
/* Resolve a batch of query terms (concatenated bytes + offsets[n + 1]) against every segment's dictionary with one
 * kernel.  out_term_ids[i] = the engine-wide id to put into rg_clause.term_id (0xffffffff: in no segment — such a
 * clause is simply absent everywhere); out_doc_freq (optional, [n_segments][n]) = its doc_freq per segment, which
 * is what term_statistics (searcher.rs:732-767) needs for the weight. */
int rg_terms_lookup(rg_engine* e, const uint8_t* bytes, const uint64_t* offsets, uint32_t n, uint32_t* out_term_ids,
                    int32_t* out_doc_freq);
/* BM25SimWeight.cache (bm25_similarity.rs:161-165), one per (field, k1, b, avgdl). */
int rg_norm_cache_set(rg_engine* e, uint32_t cache_id, const float cache[256]);
/* Bytes of device memory held by segment images. */
uint64_t rg_engine_index_bytes(rg_engine* e);

/* ---------------------------------------------------------------- search ---------- */
/* IndexSearcher::search for a batch of queries against all uploaded segments with a
 * TopDocsCollector::new(k) each (searcher.rs:487-525, collector/top_docs.rs).
 * out_hits[n_queries*k] (row i = TopDocs::score_docs() of query i, descending score, exactly
 * the reference's order incl. ties), out_counts[i] = hits in row i, out_total_hits[i] =
 * TopDocs::total_hits().  Host buffers; H2D/D2H happen inside. */
int rg_search_batch(rg_engine* e, const rg_query* queries, uint32_t n_queries,
                    const rg_clause* clauses, uint32_t n_clauses, const rg_search_params* p,
                    rg_hit* out_hits, uint32_t* out_counts, uint64_t* out_total_hits);

/* The same in three steps, so the evaluation can be timed with inputs resident in HBM — and so that batches can be
 * pipelined: calls are made from one thread at a time, but several batches may be in flight.  rg_batch_prepare
 * (host planning + plan upload on the engine's copy stream) does not wait for a batch that is running,
 * rg_batch_run queues the kernels on the engine stream behind the previous run, rg_batch_fetch waits for ITS
 * batch only.  The usual loop: run(i); prepare(i+1); fetch(i); destroy(i). */
int rg_batch_prepare(rg_engine* e, const rg_query* queries, uint32_t n_queries,
                     const rg_clause* clauses, uint32_t n_clauses, const rg_search_params* p,
                     rg_batch** out);
int rg_batch_run(rg_engine* e, rg_batch* b);   /* kernels only, asynchronous on the stream */
int rg_batch_fetch(rg_engine* e, rg_batch* b, rg_hit* out_hits, uint32_t* out_counts,
                   uint64_t* out_total_hits); /* synchronises */
void rg_batch_destroy(rg_engine* e, rg_batch* b);
/* Statistics of a prepared batch: [0]=work items, [1]=postings in scope (sum of df over scored
 * clauses), [2]=algorithmic bytes the evaluation must read (encoded blocks + tails + tables
 * touched + norms), [3]=candidates emitted by the last run, [4]=kernels per run. */
int rg_batch_stats(rg_engine* e, rg_batch* b, uint64_t out[8]);
/* RG_CFG_STATS event counters of the last run: [0]=work items of k_eval_or_ms, [1]=windows, [2]=windows that ran
 * the bit-sliced bound, [3]=windows before any theta, [4]=docids only counted (between windows), [5]=stream postings
 * visited, [6]=column gathers, [7]=block refills, [8]=candidates, [9]=32-doc steps scanned for candidates,
 * [10]=windows cut by a sparse stream's cache end, [11]=windows with a non-empty scoring set, [12]=docs scored.
 * Always counted (no flag needed): [15]=bytes the conjunction kernel (k_eval_and) asked for in the last run —
 * decoded block parts + 12 B of tables per block, 4 B per skip probe and column gather, 1 norm byte per scored
 * posting: the "touched blocks" figure of its roofline. */
int rg_batch_debug(rg_engine* e, rg_batch* b, uint64_t out[16]);
/* Score columns the planner chose for this batch (see RG_CFG_*): how many, and their bytes in HBM. */
int rg_batch_columns(rg_engine* e, rg_batch* b, uint32_t* n_columns, uint64_t* bytes);

/* Sharded mode (one segment per GPU).  After rg_batch_run with RG_MODE_SEARCH_PARALLEL the
 * per-query leaf record {uint32 n; uint32 pad; uint64 total_hits; rg_hit heap[k]} (heap-array
 * order == BinaryHeap::into_vec, top_docs.rs:203-213) lives on the device: */
int rg_batch_leaf_records(rg_engine* e, rg_batch* b, void** dev_ptr, size_t* record_bytes);
/* finish_parallel (top_docs.rs:157-172) on the device: records_all holds n_leaves consecutive
 * arrays of n_queries records (leaf order), e.g. the output of one all-gather. Host outputs. */
int rg_merge_leaf_records(rg_engine* e, const void* dev_records_all, uint32_t n_leaves,
                          uint32_t n_queries, uint32_t k, rg_hit* out_hits, uint32_t* out_counts,
                          uint64_t* out_total_hits);

/* The same merge without the copy back: the result stays in engine memory (asynchronous on the stream) until
 * rg_merge_fetch — a serving loop can launch the next batch before it reads this one's TopDocs. */
int rg_merge_leaf_records_device(rg_engine* e, const void* dev_records_all, uint32_t n_leaves,
                                 uint32_t n_queries, uint32_t k);
int rg_merge_fetch(rg_engine* e, rg_hit* out_hits, uint32_t* out_counts, uint64_t* out_total_hits);

/* The whole sharded step behind one call, for a host that holds an ncclComm_t (no Python / torch needed):
 * runs the prepared RG_MODE_SEARCH_PARALLEL batch, all-gathers every rank's leaf records with ncclAllGather on the
 * engine's stream and replays finish_parallel in leaf order (rank r holds leaves [r*L, (r+1)*L), L = segments
 * uploaded to each engine, the same on every rank).  nccl_comm: the caller's ncclComm_t, n_ranks its size.
 * libnccl is resolved at run time (symbols already in the process, else dlopen("libnccl.so.2")); without it the
 * call fails with RG_EUNSUPPORTED.  Host outputs as in rg_search_batch; every rank receives the merged result. */
int rg_batch_run_sharded(rg_engine* e, rg_batch* b, void* nccl_comm, uint32_t n_ranks, rg_hit* out_hits,
                         uint32_t* out_counts, uint64_t* out_total_hits);

/* ---------------------------------------------------------------- block codec ----- */
/* ForUtil::read_block over a raw block stream (codec/postings/for_util.rs:187-243;
 * SIMD128Packer::unpack util/packed/packed_simd.rs:126-252 when doc_version>0, else
 * BulkOperationPacked / BulkOperationPackedSingleBlock::decode_byte_to_int,
 * util/packed/packed_misc.rs:2655-2680, 2829-2841).  forutil_table: the 32 vints of the .doc
 * header ((format_id<<5)|(bpv-1), for_util.rs:128-139).  offsets[i]: byte offset of block i's
 * header byte.  out: n_blocks*128 int32.  Host buffers; copies happen inside. */
int rg_forutil_decode(rg_engine* e, const uint8_t* stream, size_t len, const uint64_t* offsets,
                      uint32_t n_blocks, int doc_version, const int32_t forutil_table[32],
                      int32_t* out);
/* The same over an uploaded segment: block pairs [first_block, first_block + n_blocks) of its index image
 * in file order, each decoded to 128 doc deltas + 128 freqs (BASELINE config 2, "realistic" blocks).
 * out (host, n_blocks*256 int32) may be NULL: the decode then only runs and is timed
 * (rg_engine_last_kernel_ms("decode")).  stats: [0]=encoded bytes read (pro rata of the segment's
 * 1+payload per part), [1]=bytes written, [2]=blocks decoded, [3]=blocks in the segment. */
int rg_segment_decode(rg_engine* e, uint32_t seg_ord, uint64_t first_block, uint64_t n_blocks, int32_t* out,
                      uint64_t stats[4]);
/* Staged variant: blocks are parsed once, their payload bytes copied unchanged into 16-byte
 * aligned slots in HBM; decode then runs with everything resident. */
int rg_blockset_stage(rg_engine* e, const uint8_t* stream, size_t len, const uint64_t* offsets,
                      uint32_t n_blocks, int doc_version, const int32_t forutil_table[32],
                      rg_blockset** out);
int rg_blockset_decode(rg_engine* e, rg_blockset* bs); /* async; output stays on the device */
int rg_blockset_fetch(rg_engine* e, rg_blockset* bs, int32_t* out); /* synchronises */
/* [0]=encoded bytes read per decode (sum of 1+16*b or 1+vint), [1]=bytes written (512/block) */
int rg_blockset_stats(rg_engine* e, rg_blockset* bs, uint64_t out[4]);
void rg_blockset_destroy(rg_engine* e, rg_blockset* bs);

#ifdef __cplusplus
}
#endif
#endif
