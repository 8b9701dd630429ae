// eval_shared.cuh — device code shared by the query-evaluation kernels (query_kernels.cu, eval_or_ms.cu):
// candidate emission + theta tracking, skip-table search, vint tails, live docs, and the cached block
// stream of a clause (unpack -> docid scan -> norm gather -> BM25, once per block).
#pragma once
#include "engine.hpp"
#include "unpack.cuh"

namespace rg {

constexpr int kEvalThreads = 256;
constexpr int kEvalWarps = kEvalThreads / 32;
constexpr int kNewcMax = 512;           // candidate scores fed to the theta tracker per window
constexpr int kMaxK = 1024;             // theta tracking / replay heap capacity
constexpr uint32_t kNone = 0xffffffffu;
constexpr uint32_t kRunMin = 256;       // minimum candidate run length (slots)
constexpr uint32_t kRunFirst = 63;      // first run of a warp-sized work item (most items emit few)
constexpr uint32_t kSent = 0x7fc0dead;  // "no posting yet" marker in the accumulator window (a NaN)
constexpr uint32_t kExcl = 0x7fc0beef;  // doc matched a MUST_NOT clause (ReqNotScorer): not a hit

// ------------------------------------------------------------------------------------------
// candidate emission + theta tracking (shared by both evaluation kernels)
// ------------------------------------------------------------------------------------------
struct EmitShared {
    float topk[kMaxK];
    float newc[kNewcMax];
    uint32_t warp_c[kEvalWarps], warp_m[kEvalWarps];
    uint32_t newc_n;
    uint32_t topk_n;
    float theta_local;
    uint32_t theta_in;  // ordered-uint theta inherited from earlier ranges of the chain
    uint32_t run_slot, run_cap, run_cnt;
    uint32_t write_base;
    uint32_t matches;
    uint32_t overflow;
};

__device__ __forceinline__ void emit_init(EmitShared& es) {
    if (threadIdx.x == 0) {
        es.newc_n = 0;
        es.topk_n = 0;
        es.theta_local = -INFINITY;
        es.theta_in = 0;
        es.run_slot = kNone;
        es.run_cap = 0;
        es.run_cnt = 0;
        es.write_base = 0;
        es.matches = 0;
        es.overflow = 0;
    }
}

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// ------------------------------------------------------------------------------------------
// deep top-k (k > kMaxK): theta from a score histogram
// ------------------------------------------------------------------------------------------
// A batch with k > kMaxK keeps, per work item, kDeepBuckets u32 counts of its emitted candidate scores in the slot the
// running top-k uses otherwise (WarpShared's topk, EmitShared::topk), so shared memory does not grow with k.  Per query
// the planner picks a bucket map m = (base, shift) (EvalParams::deep_map):
//   key(s) = clamp((float_to_ordered(s) - base) >> shift, 0, B - 1),   edge(b) = ordered_to_float(base + (b << shift))
// for b >= 1; bucket 0 is the floor and its edge is -inf.  Since float_to_ordered is monotone, every score in bucket
// b >= 1 is >= edge(b), whatever range the map was sized for (a score above it clamps into bucket B - 1).
//
// theta = edge(b) for the largest b whose suffix count (buckets b..B-1) is >= k.  Why that is exact: the counts are of
// candidates this item (and, through deep_inherit, the earlier items of its heap chain) already emitted, each doc at
// most once along the chain, all of them earlier in collection order.  So at least k earlier-collected docs score
// >= edge(b), the heap root is >= edge(b) once the replay gets here, and a doc with score <= edge(b) cannot replace it
// (TopDocsCollector replaces the root only when root.score < score, top_docs.rs:67-76).  Counts only grow: a copy that
// races with a predecessor's increments undercounts and the bound stays valid, so the histogram needs no
// count-then-entries protocol, only volatile reads.  A NaN score is never counted.
__device__ __forceinline__ uint32_t deep_key(uint2 m, float s) {
    const uint32_t o = float_to_ordered(s);
    return o < m.x ? 0u : min((o - m.x) >> m.y, (uint32_t)(kDeepBuckets - 1));
}

__device__ __forceinline__ void deep_count(uint32_t* hist, uint2 m, float s) {
    if (s == s) atomicAdd(hist + deep_key(m, s), 1u);
}

// Warp-cooperative (lane l owns buckets [8l, 8l + 8)): theta of the histogram; mirrors it into
// EvalParams::item_topk[item] (stride kDeepBuckets), then publishes its total in item_topk_n[item] and theta in
// item_theta[item].
__device__ __forceinline__ float deep_publish(const uint32_t* hist, const EvalParams& p, uint32_t item_idx, uint2 m, int lane) {
    uint32_t* g = p.item_topk ? reinterpret_cast<uint32_t*>(p.item_topk) + (size_t)item_idx * kDeepBuckets : nullptr;
    uint32_t c[8], own = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        c[j] = hist[lane * 8 + j];
        own += c[j];
        if (g) g[lane * 8 + j] = c[j];
    }
    uint32_t suf = own;  // buckets of lanes >= this one
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, suf, o);
        if (lane + o < 32) suf += v;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, suf, 0);
    int best = -1;
    uint32_t s = suf - own;
#pragma unroll
    for (int j = 7; j >= 0; j--) {
        s += c[j];
        if (best < 0 && s >= p.k) best = lane * 8 + j;
    }
    best = __reduce_max_sync(0xffffffffu, best);
    const float theta = best >= 1 ? ordered_to_float(m.x + ((uint32_t)best << m.y)) : -INFINITY;
    if (lane == 0) {
        if (g && total) {  // buckets first, then the total a successor looks for
            __threadfence();
            *reinterpret_cast<volatile uint32_t*>(p.item_topk_n + item_idx) = total;
        }
        if (theta != -INFINITY) atomicMax(p.item_theta + item_idx, float_to_ordered(theta));
    }
    return theta;
}

// Warp-cooperative start of a deep work item: copy the nearest predecessor's published histogram into `hist` (zeros
// when there is none) and return its theta.
__device__ __forceinline__ float deep_inherit(uint32_t* hist, const EvalParams& p, uint32_t item_idx, uint32_t chain_pos,
                                           uint2 m, int lane) {
    const uint32_t* src = nullptr;
    if (p.item_topk && chain_pos) {
        const uint32_t cnt = (uint32_t)lane < chain_pos ? ld_volatile_u32(p.item_topk_n + item_idx - 1 - lane) : 0u;
        const uint32_t have = __ballot_sync(0xffffffffu, cnt > 0u);
        if (have) src = reinterpret_cast<const uint32_t*>(p.item_topk) + (size_t)(item_idx - (uint32_t)__ffs(have)) * kDeepBuckets;
        __threadfence();
    }
#pragma unroll
    for (int j = 0; j < 8; j++) hist[lane * 8 + j] = src ? ld_volatile_u32(src + lane * 8 + j) : 0u;
    __syncwarp();
    if (!src) return -INFINITY;
    return deep_publish(hist, p, item_idx, m, lane);
}

// warp 0: fold this window's candidate scores into the running top-k and publish theta
static __device__ void theta_update(EmitShared& es, uint32_t k, uint32_t* theta_out) {
    const int lane = lane_id();
    const uint32_t n_new = min(es.newc_n, (uint32_t)kNewcMax);
    uint32_t n = es.topk_n;
    float theta = es.theta_local;
    int argmin = 0;
    auto recompute = [&]() {
        float m = INFINITY;
        int mi = 0;
        for (uint32_t j = lane; j < k; j += 32) {
            float v = es.topk[j];
            if (v < m) {
                m = v;
                mi = (int)j;
            }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            float om = __shfl_xor_sync(0xffffffffu, m, o);
            int oi = __shfl_xor_sync(0xffffffffu, mi, o);
            if (om < m || (om == m && oi < mi)) {
                m = om;
                mi = oi;
            }
        }
        theta = m;
        argmin = mi;
    };
    if (k <= (uint32_t)kMaxK) {
        if (n == k && n_new) recompute();
        for (uint32_t i = 0; i < n_new; i++) {
            const float x = es.newc[i];
            if (n < k) {
                if (lane == 0) es.topk[n] = x;
                n++;
                __syncwarp();
                if (n == k) recompute();
            } else if (x > theta) {
                if (lane == 0) es.topk[argmin] = x;
                __syncwarp();
                recompute();
            }
        }
    }
    if (lane == 0) {
        es.topk_n = n;
        es.theta_local = (n == k && k <= (uint32_t)kMaxK) ? theta : -INFINITY;
        uint32_t ord = es.theta_in;
        if (es.theta_local != -INFINITY) ord = max(ord, float_to_ordered(es.theta_local));
        if (ord > kOrderedNegInf) atomicMax(theta_out, ord);
    }
}

// warp 0, deep batches: theta from the histogram in es.topk (when the window emitted something); publish theta
static __device__ void theta_update_deep(EmitShared& es, const EvalParams& p, uint32_t item_idx, uint2 m) {
    const int lane = lane_id();
    if (es.newc_n) {
        const float theta = deep_publish(reinterpret_cast<const uint32_t*>(es.topk), p, item_idx, m, lane);
        if (lane == 0) es.theta_local = theta;
    }
    if (lane == 0) {
        uint32_t ord = es.theta_in;
        if (es.theta_local != -INFINITY) ord = max(ord, float_to_ordered(es.theta_local));
        if (ord > kOrderedNegInf) atomicMax(p.item_theta + item_idx, ord);
    }
}

// One emission step.  Slot order = (warp, step, lane) ascending == docid order.  `present`
// marks matches; inherited_theta is thread 0's prefetched copy of the previous item's theta.
// DEEP (k > kMaxK): candidates are counted in the histogram of the query's bucket map `dmap` instead.
template <int STEPS, bool DEEP = false>
__device__ void emit_window(EmitShared& es, const EvalParams& p, uint32_t item_idx, int doc_base,
                            const bool (&present)[STEPS], const int (&doc)[STEPS],
                            const float (&score)[STEPS], uint32_t inherited_theta, uint2 dmap = uint2{0u, 0u}) {
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    float te = es.theta_local;
    if (es.theta_in > kOrderedNegInf) te = fmaxf(te, ordered_to_float(es.theta_in));
    const bool open = te == -INFINITY;
    uint32_t cmask[STEPS];
    uint32_t nm = 0, nc = 0;
#pragma unroll
    for (int s = 0; s < STEPS; s++) {
        const uint32_t pm = __ballot_sync(0xffffffffu, present[s]);
        cmask[s] = __ballot_sync(0xffffffffu, present[s] && (open || score[s] > te));
        nm += __popc(pm);
        nc += __popc(cmask[s]);
    }
    if (lane == 0) {
        es.warp_m[warp] = nm;
        es.warp_c[warp] = nc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t tc = 0, tm = 0;
        for (int w = 0; w < kEvalWarps; w++) {
            const uint32_t c = es.warp_c[w];
            es.warp_c[w] = tc;
            tc += c;
            tm += es.warp_m[w];
        }
        es.matches += tm;
        es.newc_n = 0;
        es.theta_in = max(es.theta_in, inherited_theta);
        if (tc > 0 && !es.overflow) {
            CandRun* hdr = reinterpret_cast<CandRun*>(p.cand_arena);
            if (es.run_slot == kNone || es.run_cnt + tc > es.run_cap) {
                const uint32_t cap = max(tc, kRunMin);
                const unsigned long long slot64 = atomicAdd(p.arena_next, (unsigned long long)cap + 1ull);
                const uint32_t slot = (uint32_t)slot64;
                if (slot64 + cap + 1ull > (unsigned long long)p.arena_slots) {
                    atomicOr(p.error_flag, 1u);
                    es.overflow = 1;
                } else {
                    if (es.run_slot == kNone) p.item_head[item_idx] = slot;
                    else hdr[es.run_slot] = CandRun{slot, es.run_cnt};
                    es.run_slot = slot;
                    es.run_cap = cap;
                    es.run_cnt = 0;
                }
            }
            if (!es.overflow) {
                es.write_base = es.run_slot + 1 + es.run_cnt;
                es.run_cnt += tc;
                hdr[es.run_slot] = CandRun{kNone, es.run_cnt};
            }
        }
    }
    __syncthreads();
    if (nc && !es.overflow) {
        uint32_t pos = es.write_base + es.warp_c[warp];
        const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
        for (int s = 0; s < STEPS; s++) {
            if ((cmask[s] >> lane) & 1u) {
                p.cand_arena[pos + __popc(cmask[s] & lt)] = rg_hit{doc[s] + doc_base, score[s]};
                const uint32_t i = atomicAdd(&es.newc_n, 1u);
                if (DEEP) deep_count(reinterpret_cast<uint32_t*>(es.topk), dmap, score[s]);
                else if (i < (uint32_t)kNewcMax) es.newc[i] = score[s];
            }
            pos += __popc(cmask[s]);
        }
    }
    __syncthreads();
    if (warp == 0) {
        if (DEEP) theta_update_deep(es, p, item_idx, dmap);
        else theta_update(es, p.k, p.item_theta + item_idx);
    }
}

// first index in [lo, hi) with a[i] >= key (hi if none)
__device__ __forceinline__ uint32_t lower_bound_i32(const int32_t* __restrict__ a, uint32_t lo,
                                                    uint32_t hi, int32_t key) {
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
// same, galloping forward from `hint` (<= answer)
__device__ __forceinline__ uint32_t lower_bound_gallop(const int32_t* __restrict__ a, uint32_t hint,
                                                       uint32_t n, int32_t key) {
    uint32_t lo = hint, step = 1, hi = hint;
    while (hi < n && __ldg(a + hi) < key) {
        lo = hi + 1;
        hi += step;
        step <<= 1;
    }
    return lower_bound_i32(a, lo, min(hi, n), key);
}

struct TermCtx {
    const int32_t* blk_last;   // this term's slice of the level-0 skip table
    const BlockDesc* blk_desc;
    const float* cache;
    uint32_t nb;               // full blocks
    uint32_t cur;              // first block not fully consumed
    uint32_t next_cur;
    uint32_t tail_n;           // postings in the (decoded) tail, 0 = no tail in scope
    uint32_t tail_pos;
    uint32_t tail_next;
    int32_t tail_base;
    float w1;                  // weight * (k1 + 1)
};

// Decode a term's vint tail (or singleton) into shared memory: absolute docids + freqs.
// codec/postings/posting_reader.rs:308-333 (read_vint_block), :545-547 (singleton).
static __device__ void decode_tail(const SegDev& seg, const TermDev& td, int32_t* docs, int32_t* freqs) {
    if (td.doc_freq == 1) {
        docs[0] = td.singleton_doc;
        freqs[0] = td.singleton_freq;
        return;
    }
    const uint8_t* p = seg.tails + td.tail_off;
    uint32_t pos = 0;
    int32_t acc = td.tail_base;
    for (uint32_t i = 0; i < td.tail_n; i++) {
        const uint32_t code = (uint32_t)read_vint(p, pos);
        acc += (int32_t)(code >> 1);
        docs[i] = acc;
        freqs[i] = (code & 1u) ? 1 : read_vint(p, pos);
    }
}

__device__ __forceinline__ bool is_live(const SegDev& seg, int doc) {
    if (!seg.live) return true;
    return (seg.live[doc >> 6] >> (doc & 63)) & 1ull;
}

// PointRangeIntersectVisitor::visit_by_packed_value over every value of doc d: lower <= key <= upper for any of
// them (keys ascending within a doc)
__device__ __forceinline__ bool range_hit(const RangeRef& r, int d) {
    const uint32_t o0 = __ldg(r.offsets + d), o1 = __ldg(r.offsets + d + 1);
    for (uint32_t j = o0; j < o1; j++) {
        const uint64_t key = r.wide ? __ldg(static_cast<const unsigned long long*>(r.keys) + j)
                                    : (uint64_t)__ldg(static_cast<const uint32_t*>(r.keys) + j);
        if (key > r.upper) return false;
        if (key >= r.lower) return true;
    }
    return false;
}

// ------------------------------------------------------------------------------------------
// k_eval_or  — one WARP per work item, no block-level synchronisation at all.
// ------------------------------------------------------------------------------------------
// A work item is a (query, segment, docid range) of ~32K postings.  Every clause is a *cached
// block stream*: its current 128-posting block lives decoded AND scored in shared memory
// (docids + BM25 scores), so each block is unpacked, prefix-summed and scored exactly once.
// The warp walks the range in windows of kWw docids that always start at a real posting:
//   for clause t = 0..T-1 (clause order): consume the stream's postings < window end, 32 per
//       step, "acc[d] = acc[d] + s" in the warp-private accumulator window — pair order ==
//       clause order == DisjunctionSumScorer::score_sum's f32 order; refill the stream (decode the
//       next block / the vint tail) whenever it runs dry;
//   scan the touched 32-doc steps in docid order -> total_hits, theta filter, candidates;
//   next window start = min over clauses of their next cached docid (exact).
constexpr int kOrWarps = 1;  // one warp per CTA: a CTA's slot is held until its slowest warp is done
constexpr int kOrThreads = kOrWarps * 32;
constexpr int kWw = 768;            // docids per window
constexpr int kNewcW = 64;

struct WTerm {
    const int32_t* blk_last;
    union {
        const BlockDesc* blk_desc;
        const uint32_t* col_bmax;  // score column (LEAN): ColRef::bmax, largest cell per kColBlk docids (null: none)
    };
    union {
        const float* cache;
        const uint32_t* col_bits;  // score column (LEAN): the term's presence bitmap (ColRef::bits)
    };
    uint32_t nb;        // full blocks; decode-free variant (LEAN): units of the scored list, full blocks + the tail if any
    uint32_t cur;       // next block to decode (nb = vint tail, nb+1 = exhausted); LEAN: the cursor's unit, nb = exhausted
    uint32_t n;         // valid entries in the stream cache
    uint32_t pos;       // next unconsumed entry (LEAN: within unit cur of the scored list)
    uint32_t term_id;
    float w1;           // weight * (k1 + 1)
    uint32_t is_not;    // MUST_NOT clause: its postings exclude docs (search/scorer/req_not_scorer.rs)
    uint32_t is_col;    // score column: blk_last is really a const float* indexed by docid (see k_build_columns)
    union {
        const uint4* pre;   // scored posting list (k_build_columns<4>): 1 KB per block = 128 docids + 128 f32 scores; null = decode
        unsigned long long* col_dbg;  // score column (LEAN): EvalParams::dbg (RG_CFG_STATS counters, else null)
    };
};

// One posting of a clause lands on window slot idx.  SHOULD clause: clause-order f32 add, first
// touch counts the match.  MUST_NOT clause (drained after every SHOULD clause of the window): a doc
// that is present becomes kExcl and its match is taken back.
// MSM (min_should_match > 1, disjunction_scorer.rs:317-329): a per-doc clause counter next to the
// sums; a doc becomes a match when its counter reaches msm.
// DMAX (DisjunctionMaxScorer, disjunction_scorer.rs:241-263): the running maximum of the clause scores
// next to their sum; the final score max + (sum - max) * tie_breaker is formed in the window epilogue.
struct MsmCtx {
    uint8_t* cnt;  // [kWw] clause counters of the window (MSM variants only)
    uint32_t msm;
    float* mx;     // [kWw] per-doc maximum clause score (DMAX variant only)
};
// POS (only with !NOT, !MSM, !DMAX): every clause score of the launch is > 0, so "no posting yet" is simply
// the sum +0.0f — the add needs no select; a doc matched iff its sum is non-zero, and the window epilogue counts
// the matches and finds the sums above theta in one pass over the finished window.
template <bool NOT, bool MSM, bool DMAX, bool POS = false>
__device__ __forceinline__ void accumulate_posting(uint32_t* acc, int idx, float s, bool is_not, bool live,
                                                   float te, uint32_t& hot, uint32_t& my_matches,
                                                   const MsmCtx& mc) {
    if (POS) {
        acc[idx] = __float_as_uint(__fadd_rn(__uint_as_float(acc[idx]), s));
        return;
    }
    const uint32_t old = acc[idx];
    if (!NOT || !is_not) {
        const float sum = __fadd_rn(old == kSent ? 0.0f : __uint_as_float(old), s);
        acc[idx] = __float_as_uint(sum);
        if (DMAX) mc.mx[idx] = old == kSent ? s : fmaxf(mc.mx[idx], s);
        if (MSM) {
            const uint32_t c = (uint32_t)mc.cnt[idx] + 1u;
            mc.cnt[idx] = (uint8_t)c;
            if (c == mc.msm && live) my_matches++;
        } else if (old == kSent && live) {
            my_matches++;
        }
        // DMAX: the final score is not the sum, so every touched step is scanned
        if (DMAX || sum > te) hot |= 1u << (idx >> 5);
    } else if (old != kSent && old != kExcl) {
        acc[idx] = kExcl;
        if (live && (!MSM || mc.cnt[idx] >= mc.msm)) my_matches--;
    }
}

struct alignas(16) WarpShared {  // followed by topk[kcap] floats, then cdocs[T][128], cscores[T][128]
    uint32_t acc[kWw];
    WTerm term[kMaxTerms];
    float newc[kNewcW];
};

// warp-level candidate emitter state (registers, uniform across lanes)
struct WEmit {
    float* topk;       // shared memory, kcap floats
    bool mirror;       // topk is mirrored into EvalParams::item_topk[item] and its count into item_topk_n[item]
                       // (formed from the params at each use: a pointer pair held across the window loop costs registers)
    uint32_t topk_n;
    float theta_local;
    uint32_t theta_in;
    uint32_t run_slot, run_cap, run_cnt;
    uint32_t matches;
    bool overflow;
};

__device__ __forceinline__ void wtheta_recompute(const WEmit& em, uint32_t k, int lane, float& theta, int& argmin) {
    float m = INFINITY;
    int mi = 0;
    for (uint32_t j = lane; j < k; j += 32) {
        const float v = em.topk[j];
        if (v < m) {
            m = v;
            mi = (int)j;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        if (om < m || (om == m && oi < mi)) {
            m = om;
            mi = oi;
        }
    }
    theta = m;
    argmin = mi;
}

__device__ __forceinline__ void wtheta_update(WEmit& em, const EvalParams& p, uint32_t item_idx, uint32_t kcap, int lane,
                                              const float* newc, uint32_t newc_n) {
    const uint32_t k = p.k;
    const uint32_t n_new = min(newc_n, (uint32_t)kNewcW);
    if (n_new == 0 || k > kcap) return;
    float* gtopk = em.mirror ? p.item_topk + (size_t)item_idx * kcap : nullptr;
    __syncwarp();
    float theta = em.theta_local;
    int argmin = 0;
    uint32_t n = em.topk_n;
    if (n == k) wtheta_recompute(em, k, lane, theta, argmin);
    for (uint32_t i = 0; i < n_new; i++) {
        const float x = newc[i];
        if (n < k) {
            if (lane == 0) {
                em.topk[n] = x;
                if (gtopk) gtopk[n] = x;
            }
            n++;
            __syncwarp();
            if (n == k) wtheta_recompute(em, k, lane, theta, argmin);
        } else if (x > theta) {
            if (lane == 0) {
                em.topk[argmin] = x;
                if (gtopk) gtopk[argmin] = x;
            }
            __syncwarp();
            wtheta_recompute(em, k, lane, theta, argmin);
        }
    }
    const bool grew = n != em.topk_n;
    em.topk_n = n;
    em.theta_local = n == k ? theta : -INFINITY;
    if (lane == 0) {
        if (em.mirror && grew) {  // entries first, then the count a successor reads
            __threadfence();
            *reinterpret_cast<volatile uint32_t*>(p.item_topk_n + item_idx) = n;
        }
        uint32_t ord = em.theta_in;
        if (em.theta_local != -INFINITY) ord = max(ord, float_to_ordered(em.theta_local));
        if (ord > kOrderedNegInf) atomicMax(p.item_theta + item_idx, ord);
    }
}

// Start of a work item: take over the running top-k of the heap chain.  Every item mirrors its top-k scores
// (of docs it has passed, plus what it inherited) into EvalParams::item_topk; a later range of the same chain
// copies the nearest predecessor's array — all of those docs come earlier in collection order, every doc lives
// in one slot of one array, so the k-th best of the copy is a lower bound of the heap root when this range
// starts — and keeps inserting its own candidates.  Without it theta would only be the best per-range k-th
// score, far below the root of a heap that has seen hundreds of ranges.
__device__ __forceinline__ void wtheta_inherit(WEmit& em, const EvalParams& p, uint32_t item_idx, uint32_t chain_pos,
                                               uint32_t kcap, int lane) {
    em.mirror = p.item_topk && p.k <= kcap;
    if (!em.mirror || chain_pos == 0) return;
    float* gtopk = p.item_topk + (size_t)item_idx * kcap;
    uint32_t cnt = 0;
    if ((uint32_t)lane < chain_pos) cnt = ld_volatile_u32(p.item_topk_n + item_idx - 1 - lane);
    const uint32_t have = __ballot_sync(0xffffffffu, cnt > 0u);
    if (!have) return;
    const int src_lane = __ffs(have) - 1;  // nearest predecessor that has published something
    const uint32_t n = min(__shfl_sync(0xffffffffu, cnt, src_lane), p.k);
    __threadfence();
    const float* src = p.item_topk + (size_t)(item_idx - 1 - (uint32_t)src_lane) * kcap;
    for (uint32_t j = lane; j < n; j += 32) {
        const float v = __uint_as_float(ld_volatile_u32(reinterpret_cast<const uint32_t*>(src + j)));
        em.topk[j] = v;
        gtopk[j] = v;
    }
    __syncwarp();
    em.topk_n = n;
    if (n == p.k) {
        float theta;
        int argmin;
        wtheta_recompute(em, p.k, lane, theta, argmin);
        em.theta_local = theta;
    }
    if (lane == 0) {
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(p.item_topk_n + item_idx) = n;
        if (em.theta_local != -INFINITY) atomicMax(p.item_theta + item_idx, float_to_ordered(em.theta_local));
    }
}

// the warp kernels' update after a window: only when it emitted something
__device__ __forceinline__ void wtheta_update_deep(WEmit& em, const EvalParams& p, uint32_t item_idx, uint2 m, int lane,
                                                   uint32_t emitted) {
    if (emitted == 0) return;
    __syncwarp();
    em.theta_local = deep_publish(reinterpret_cast<const uint32_t*>(em.topk), p, item_idx, m, lane);
}

// Refill clause t's stream cache with its next block (or vint tail): unpack, docid scan, norm
// gather, BM25 — once per block.  Entries outside [lo, hi) are trimmed.  Returns false when the
// list is exhausted.  Warp-cooperative; all lanes must call it.
// When called while clause t is being drained into the window [win0, win1) the new block's
// postings below win1 are accumulated straight from registers (no round trip through the cache).
template <bool LIVE, bool NOT, bool MSM, bool DMAX, bool POS = false>
__device__ __forceinline__ bool stream_refill(const SegDev& seg, const EvalParams& p, WTerm& tc, int32_t* cd,
                                           float* cs, int lo, int hi, int lane, int win0, int win1,
                                           uint32_t* acc, uint32_t& hot, uint32_t& my_matches, float te,
                                           const MsmCtx& mc) {
    for (;;) {
        const uint32_t b = tc.cur;
        if (b > tc.nb) return false;
        int4 docs, freqs;
        uint32_t n_in = kBlock;
        uint32_t next_off16 = 0;  // payload of the block after this one (0: none) — prefetched below
        bool interior = false;    // every posting of the block lies inside [lo, hi)
        bool all_direct = false;  // ... and inside the window being drained
        float sc[4];
        const uint4* pre = tc.pre;
        if (pre) {
            // the clause's postings were decoded and scored once for all batches (scored list): two 16-byte loads
            // per lane replace unpack + scan + norm gather + division; entries past the end hold kNoMoreDocs
            if (b < tc.nb) {
                const int base = b == 0 ? 0 : __ldg(tc.blk_last + b - 1);
                const int last = __ldg(tc.blk_last + b);
                interior = (b == 0 ? lo == 0 : base >= lo) && last < hi;
                all_direct = interior && last < win1;
            } else {
                n_in = seg.terms[tc.term_id].tail_n;
                if (n_in == 0) {
                    if (lane == 0) tc.cur = tc.nb + 1;
                    __syncwarp();
                    return false;
                }
            }
            const uint4* blk = pre + (size_t)b * 64;
            const uint4 dv = __ldg(blk + lane), sv = __ldg(blk + 32 + lane);
            docs = make_int4((int)dv.x, (int)dv.y, (int)dv.z, (int)dv.w);
            sc[0] = __uint_as_float(sv.x);
            sc[1] = __uint_as_float(sv.y);
            sc[2] = __uint_as_float(sv.z);
            sc[3] = __uint_as_float(sv.w);
            if (b < tc.nb && lane < 8) asm volatile("prefetch.global.L2 [%0];" ::"l"(blk + 64 + lane * 8));
        } else if (b < tc.nb) {
            const BlockDesc bd = tc.blk_desc[b];
            const int base = b == 0 ? 0 : __ldg(tc.blk_last + b - 1);
            const int last = __ldg(tc.blk_last + b);
            if (b + 1 < tc.nb) next_off16 = tc.blk_desc[b + 1].off16;  // same cache line as bd, almost always
            interior = (b == 0 ? lo == 0 : base >= lo) && last < hi;
            all_direct = interior && last < win1;
            const uint4* part = seg.arena + bd.off16;
            const int bdoc = (int)(bd.bits & 0xff), bfrq = (int)((bd.bits >> 8) & 0xff);
            int4 dl;
            const uint32_t enc = bd.bits >> 24;
            if (seg.version > 0 && bdoc > 0 && bfrq > 0) {  // the common case: both parts SIMD128-packed
                dl = unpack4_simd128(part, bdoc, lane);
                freqs = unpack4_simd128(part + ((bd.bits >> 16) & 0xff), bfrq, lane);
                docs = deltas_to_docs(dl, base);
            } else if (enc == 0) {
                dl = unpack4(part, bdoc, lane, seg.version, seg.sb_mask);
                freqs = unpack4(part + ((bd.bits >> 16) & 0xff), bfrq, lane, seg.version, seg.sb_mask);
                docs = deltas_to_docs(dl, base);
            } else {  // EF / BITSET doc part: docids, not deltas; the stream cache is free scratch here
                decode_other_docs(part, enc, b == 0 ? -1 : base, cd, lane);
                docs = reinterpret_cast<const int4*>(cd)[lane];
                freqs = unpack4(part + ((bd.bits >> 16) & 0xff), bfrq, lane, seg.version, seg.sb_mask);
                __syncwarp();
            }
        } else {  // vint tail / singleton (posting_reader.rs:308-333, :545-547): lane 0 decodes
            const TermDev td = seg.terms[tc.term_id];
            n_in = td.tail_n;
            if (n_in == 0) {
                if (lane == 0) tc.cur = tc.nb + 1;
                __syncwarp();
                return false;
            }
            if (lane == 0) {
                int32_t* fq = reinterpret_cast<int32_t*>(cs);
                decode_tail(seg, td, cd, fq);
            }
            __syncwarp();
            const int i0 = 4 * lane;
            const int32_t* fq = reinterpret_cast<const int32_t*>(cs);
            docs = make_int4(i0 < (int)n_in ? cd[i0] : kNoMoreDocs, i0 + 1 < (int)n_in ? cd[i0 + 1] : kNoMoreDocs,
                             i0 + 2 < (int)n_in ? cd[i0 + 2] : kNoMoreDocs, i0 + 3 < (int)n_in ? cd[i0 + 3] : kNoMoreDocs);
            freqs = make_int4(i0 < (int)n_in ? fq[i0] : 1, i0 + 1 < (int)n_in ? fq[i0 + 1] : 1,
                              i0 + 2 < (int)n_in ? fq[i0 + 2] : 1, i0 + 3 < (int)n_in ? fq[i0 + 3] : 1);
            __syncwarp();
        }
        const int d[4] = {docs.x, docs.y, docs.z, docs.w};
        uint32_t below = 0, inside = 0, direct = 0;
        const float w1 = tc.w1;
        const float* cache = tc.cache;
        const uint8_t* norms = seg.norms;
        const bool neg = NOT && tc.is_not != 0;
        // stage the gathers: 4 norm bytes, then 4 cache entries, then 4 divisions — branch-free, so the
        // loads of all four postings are in flight together (out-of-range lanes read a safe slot)
        bool ok[4];
        float nrm[4];
        if (interior) {
#pragma unroll
            for (int q = 0; q < 4; q++) ok[q] = true;
        } else {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                ok[q] = d[q] >= lo && d[q] < hi;
                below += d[q] < lo;
                inside += ok[q];
            }
        }
        if (!pre) {
            const int f[4] = {freqs.x, freqs.y, freqs.z, freqs.w};
            if (norms) {
                uint32_t nb8[4];
#pragma unroll
                for (int q = 0; q < 4; q++) nb8[q] = __ldg(norms + (ok[q] ? d[q] : lo));
#pragma unroll
                for (int q = 0; q < 4; q++) nrm[q] = __ldg(cache + nb8[q]);
            } else {
#pragma unroll
                for (int q = 0; q < 4; q++) nrm[q] = p.k1;
            }
#pragma unroll
            for (int q = 0; q < 4; q++) sc[q] = bm25_score(w1, (float)f[q], nrm[q]);
        }
        // pull the next block's payload towards L1 while this one is accumulated (dense clauses come
        // straight back for it).  Prefetching the norm bytes the next block will probably hit, or
        // carrying the next descriptor in shared memory, both measured slower.
        if (next_off16 && lane < 4) {
            const uint4* np = seg.arena + next_off16 + lane * 8;
            asm volatile("prefetch.global.L1 [%0];" ::"l"(np));
        }
        if (all_direct) {  // the common case for dense clauses: nothing to cache, no cursor arithmetic
#pragma unroll
            for (int q = 0; q < 4; q++)
                accumulate_posting<NOT, MSM, DMAX, POS>(acc, d[q] - win0, sc[q], neg, (LIVE && !POS) ? is_live(seg, d[q]) : true,
                                                   te, hot, my_matches, mc);
            __syncwarp();  // every lane has read tc.cur / tc.nb above
            if (lane == 0) {
                tc.pos = tc.n = 0;
                tc.cur = b + 1;
            }
            __syncwarp();
            continue;
        }
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (ok[q] && d[q] < win1) {  // still inside the window being drained: accumulate now
                accumulate_posting<NOT, MSM, DMAX, POS>(acc, d[q] - win0, sc[q], neg, (LIVE && !POS) ? is_live(seg, d[q]) : true,
                                                   te, hot, my_matches, mc);
                direct++;
            }
        }
        reinterpret_cast<int4*>(cd)[lane] = docs;
        reinterpret_cast<float4*>(cs)[lane] = make_float4(sc[0], sc[1], sc[2], sc[3]);
        if (interior) {
            inside = kBlock;
        } else {
            below = __reduce_add_sync(0xffffffffu, below);
            inside = __reduce_add_sync(0xffffffffu, inside);
        }
        direct = __reduce_add_sync(0xffffffffu, direct);
        const bool past_end = below + inside < n_in;  // some posting >= hi: nothing further in range
        below += direct;
        inside -= direct;
        __syncwarp();  // every lane has read tc.cur / tc.nb above
        if (lane == 0) {
            tc.pos = below;
            tc.n = below + inside;
            tc.cur = past_end ? tc.nb + 1 : b + 1;
        }
        __syncwarp();
        if (inside > 0) return true;
        if (past_end) return false;
        // whole block consumed (all below lo, or all accumulated directly): decode the next one
    }
}

}  // namespace rg
