// common.cuh — shared device/host definitions of the H100 query-evaluation engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "rucene_gpu.h"

namespace rg {

constexpr int kBlock = 128;           // codec/postings/posting_format.rs BLOCK_SIZE
constexpr int kMaxTerms = 9;          // DisjunctionSumScorer SimpleQueue regime (< 10 children)
constexpr int kDpqMaxTerms = 32;      // widest disjunction the DisiPriorityQueue kernel takes (>= 10 clauses in a leaf)
constexpr int kNoMoreDocs = 0x7fffffff;
constexpr int kBitmapDen = 1024;      // RG_CFG_MAXSCORE: terms with df >= max_doc / 1024 get a presence bitmap at upload (within a budget)
constexpr int kColumnDen = 64;        // terms with df >= max_doc / 64 may also get a score column (per weight, on demand)
constexpr int kColBlk = 128;          // docids per entry of a score column's block-maximum table (ColRef::bmax)
constexpr int kDeepBuckets = 256;     // k > 1024: score buckets of a work item's theta histogram (eval_shared.cuh)
constexpr uint32_t kDeepMaxK = 16384; // deepest accelerated k: one replay heap of k * 8 bytes fits a CTA's shared memory

// ------------------------------------------------------------------ index image in HBM
// Every full 128-posting block pair of a term owns one 16-byte aligned slot in `arena`:
//   [doc part][freq part]; a part is the block's payload bytes exactly as the codec wrote them
//   (16*b bytes for SIMD128/COMPACT layouts), or one 16-byte cell holding the vint value when
//   the block is "all values equal" (code 0).  Header bytes live in BlockDesc.
struct BlockDesc {
    uint32_t off16;  // slot offset in 16-byte units
    uint32_t bits;   // [0:8) doc num_bits, [8:16) freq num_bits, [16:24) doc part size in 16B units
                     // [24:26) doc part EncodeType: 0 PF, 1 EF, 2 BITSET (unpack.cuh: decode_other_docs)
};

struct TermDev {
    uint32_t blk_begin;    // first entry in blk_last / blk_desc
    uint32_t n_blocks;     // full blocks (doc_freq / 128)
    uint32_t tail_off;     // byte offset of the vint tail in `tails`
    uint32_t tail_n;       // postings in the tail (doc_freq % 128), 1 for a singleton
    int32_t doc_freq;
    int32_t tail_base;     // last doc of the last full block (0 when none)
    int32_t singleton_doc; // docid when doc_freq == 1 else -1
    int32_t singleton_freq;
};

struct SegDev {
    const uint4* arena;
    const int32_t* blk_last;
    const BlockDesc* blk_desc;
    const uint8_t* tails;
    const TermDev* terms;
    const uint8_t* norms;     // may be null
    const uint64_t* live;     // may be null
    int32_t doc_base;
    int32_t max_doc;
    uint32_t n_terms;
    int32_t version;          // .doc version: 0 = Packed/PackedSingleBlock, 1 = SIMD128
    uint32_t sb_mask;         // version 0: bit (b-1) set => bpv b uses PackedSingleBlock
};

// ------------------------------------------------------------------ plan (device side)
enum : uint32_t { kTypeOr = 0, kTypeAnd = 1, kTypeReqOpt = 2, kTypeDpq = 3 };

// ItemClause::flags, written by the planner (search.cu) and read by the evaluation kernels
constexpr uint32_t kClauseNot = 1u << 0;       // MUST_NOT clause (ReqNotScorer: excludes, never scores)
constexpr uint32_t kClauseOpt = 1u << 1;       // SHOULD clause beside a MUST (ReqOptScorer's optional side)
constexpr uint32_t kClauseColumn = 1u << 2;    // score column: term_id indexes EvalParams::cols
constexpr uint32_t kClauseTie = 1u << 3;       // meta entry after a DisjunctionMaxScorer item's clauses: weight = tie breaker
constexpr uint32_t kClauseNoBound = 1u << 4;   // no usable score bound: weight < 0 / NaN or a norm cache with negative entries
constexpr uint32_t kClauseBitmap = 1u << 5;    // block stream of a term with a presence bitmap: the reference indexes
                                               // EvalParams::cols (.bits, tf-norm planes)
constexpr uint32_t kClauseAllDocs = 1u << 6;   // with kClauseColumn: every docid present, cells all 0 (MatchAllDocsQuery)
constexpr uint32_t kClauseList = 1u << 7;      // block stream read from a scored list: the reference indexes EvalParams::cols (.col)
constexpr uint32_t kClauseRange = 1u << 8;     // point range: term_id indexes RangeParams::ranges (k_eval_and_ranges / _nested)
constexpr uint32_t kClauseReqGroup = 1u << 9;  // member of a required pure-SHOULD group (k_eval_and_nested); a group's
constexpr uint32_t kClauseOptGroup = 1u << 10; // ... or of an optional one; members are contiguous, in member order
constexpr uint32_t kClauseGroupLast = 1u << 11;  // the last member of its group
constexpr uint32_t kClauseRefShift = 16;       // bits [16, 32): the EvalParams::cols reference of kClauseBitmap / kClauseList

// WorkItem::type: bits [0, 2) the kType* of the item, bit 2 a DisjunctionMaxScorer item (its tie breaker rides in a
// kClauseTie entry after the clauses), bits [4, 8) min_should_match when > 1 (kTypeOr only)
constexpr uint32_t kItemDismax = 1u << 2;
constexpr uint32_t kItemMsmShift = 4;

struct ItemClause {
    uint32_t term_id;
    float weight;      // idf * boost
    uint32_t cache_id;
    uint32_t flags;    // kClause* bits
};

struct WorkItem {
    uint32_t query;
    uint16_t seg;
    uint8_t type;      // kType* | kItemDismax | msm << kItemMsmShift
    uint8_t n_terms;
    int32_t lo, hi;          // docid range [lo, hi) inside the segment
    uint32_t clause_begin;   // into ItemClause[]
    uint32_t chain_pos;      // position inside its heap chain (0 = first: no theta to inherit)
};

// ------------------------------------------------------------------ 1-D point ranges
// Points of one (leaf, field): keys are the packed sortable bytes read as a big-endian unsigned integer (u32 for 4
// bytes, u64 for 8), which orders exactly as the byte strings compare.  CSR in docid order: the keys of doc d are
// keys[offsets[d], offsets[d + 1]), ascending.  One RangeBlock per 128 docids.
struct RangeBlock {
    uint64_t min, max;  // smallest / largest key in the block (meaningless when values == 0)
    uint32_t docs;      // docids of the block with at least one value
    uint32_t values;    // keys of the block
};
// one range clause in one leaf (an ItemClause with kClauseRange: term_id indexes RangeParams::ranges)
struct RangeRef {
    const uint32_t* offsets;
    const void* keys;  // uint32_t (wide == 0) or uint64_t (wide == 1)
    const RangeBlock* blocks;
    uint64_t lower, upper;  // inclusive
    uint32_t wide;
    uint32_t pad;
};

struct CandRun {  // header slot of a candidate run in the arena (same size as rg_hit)
    uint32_t next;   // slot index of the next run header, 0xffffffff = end
    uint32_t count;
};

// ------------------------------------------------------------------ small device helpers
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// order-preserving float <-> uint mapping (for atomicMax on scores of any sign)
__device__ __forceinline__ uint32_t float_to_ordered(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
constexpr uint32_t kOrderedNegInf = 0x007fffffu;  // float_to_ordered(-inf)

__device__ __forceinline__ uint4 ldg16(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void stg16_streaming(int4* p, int4 v) {
    asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
                 "r"(v.y), "r"(v.z), "r"(v.w));
}

// BM25SimScorer::compute_score (search/similarity/bm25_similarity.rs:203-212):
//   weight * (k1 + 1.0) * freq / (freq + norm), f32, left to right, no FMA, IEEE division.
__device__ __forceinline__ float bm25_score(float w_k1p1, float freq, float norm) {
    return __fdiv_rn(__fmul_rn(w_k1p1, freq), __fadd_rn(freq, norm));
}

}  // namespace rg

#define RG_CUDA_CHECK(expr)                                                        \
    do {                                                                           \
        cudaError_t _e = (expr);                                                   \
        if (_e != cudaSuccess) throw rg::CudaError(_e, #expr, __FILE__, __LINE__); \
    } while (0)
