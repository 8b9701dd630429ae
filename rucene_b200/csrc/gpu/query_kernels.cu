// query_kernels.cu — the fused query-evaluation kernels (sm_90a, integer/HBM-bound work).
//
//   k_build_columns: batch-level common subexpression — the BM25 contributions of a dense clause that
//                 several disjunctions of the batch share, computed once into a docid-indexed f32 column.
//   k_eval_or   : TermQuery / pure-SHOULD BooleanQuery (+ MUST_NOT, min_should_match) / DisjunctionMaxQuery.
//                 One WARP per (query, segment, docid range).  Every clause is a cached block stream: a
//                 posting block is unpacked (PF, or EF / BITSET by rank-select), prefix-summed (warp scan)
//                 and BM25-scored exactly once — straight into the window when it falls inside it, else
//                 into shared memory — or it is a score column read with 16-byte loads; clauses are
//                 drained in clause order into a warp-private window of 768 docids — the f32
//                 summation order of DisjunctionSumScorer::score_sum
//                 (search/scorer/disjunction_scorer.rs:211-225).  Matches are counted when a doc is
//                 first touched (total_hits); only docs whose sum can still beat the top-k heap root
//                 are scanned and appended, in docid order, to the query's candidate list.
//   k_eval_and  : pure-MUST BooleanQuery (+ MUST_NOT) (ConjunctionScorer, search/scorer/conjunction_scorer.rs)
//                 and MUST+SHOULD (ReqOptScorer: optional clauses + the sequential running-mean chain).
//                 The cheapest list leads (stable sort by cost, :30); 8 lead blocks per step are
//                 decoded, every lead doc locates its block in each other list via the level-0
//                 skip table (galloping binary search), that block is decoded once per warp into
//                 shared memory, membership is a 7-step binary search and the freq is extracted
//                 lazily by random access into the freq block.  Scores add in cost order
//                 (lead1 + lead2 + others, :87-95).
//   k_heap_replay: exact TopDocsCollector semantics (search/collector/top_docs.rs:67-95 over std
//                 BinaryHeap, util/external/binary_heap.rs:121-210) — one warp per heap replays
//                 add_doc over the candidate lists in collection order and pops the result.
//
// Exactness of the candidate lists (SURVEY.md Appendix B): a doc changes the heap iff fewer than
// k earlier docs score >= it.  Each CTA keeps theta = k-th best score of docs it has already
// passed (plus what earlier ranges of the same heap chain published), a lower bound of the heap
// root at that point; docs with score <= theta can never enter, everything else is emitted in
// docid order.  The replay over that superset is bit-identical to the reference, ties included.
#include <algorithm>

#include "eval_shared.cuh"

namespace rg {


// One score column over one accumulator window: four adjacent docids per lane, one 16-byte
// read-modify-write of the window per step (no MUST_NOT marker can be present yet: those clauses are
// drained last).  A column cell is the clause's BM25 contribution, +0.0f where the term has no posting
// (columns are only built for clauses whose every score is > 0).  Branch-free; only the first and the
// last window of a range (EDGE) clip by position.
// POS (every clause score of the launch > 0, plain sum): the window holds +0.0f for "no posting yet", so a
// column is just added — absent cells add +0.0f; matches are counted and the docs above theta found by the
// window epilogue.
template <bool LIVE, bool EDGE, bool POS>
__device__ __forceinline__ void column_window(uint32_t* acc, const float* __restrict__ col, bool every_doc,
                                              const SegDev& seg, int win0, int wlen, int first_in, float te, int lane,
                                              uint32_t& hot, uint32_t& my_matches) {
    if (POS && !EDGE && wlen == kWw) {
        // a whole window: three 16-byte column loads of the lane are in flight before the first is used (the column
        // comes from L2 / HBM; six at once would spill)
#pragma unroll
        for (int h = 0; h < kWw / 128; h += 3) {
            float4 v[3];
#pragma unroll
            for (int j = 0; j < 3; j++) v[j] = __ldg(reinterpret_cast<const float4*>(col + win0 + lane * 4 + (h + j) * 128));
#pragma unroll
            for (int j = 0; j < 3; j++) {
                float4* a = reinterpret_cast<float4*>(acc + lane * 4 + (h + j) * 128);
                const float4 o = *a;
                *a = make_float4(__fadd_rn(o.x, v[j].x), __fadd_rn(o.y, v[j].y), __fadd_rn(o.z, v[j].z), __fadd_rn(o.w, v[j].w));
            }
        }
        return;
    }
#pragma unroll 2
    for (int i = lane * 4; i < wlen; i += 128) {
        const int d0 = win0 + i;
        const float4 v = __ldg(reinterpret_cast<const float4*>(col + d0));
        float sv[4] = {v.x, v.y, v.z, v.w};
        const uint4 o4 = *reinterpret_cast<const uint4*>(acc + i);
        uint32_t o[4] = {o4.x, o4.y, o4.z, o4.w};
        bool any_hot = false;
        if (POS) {  // (the window epilogue finds the docs above theta)
#pragma unroll
            for (int q = 0; q < 4; q++) {
                if (EDGE) sv[q] = (i + q >= first_in && i + q < wlen) ? sv[q] : 0.0f;
                o[q] = __float_as_uint(__fadd_rn(__uint_as_float(o[q]), sv[q]));
            }
        } else {
            uint32_t live4 = 0xfu;
            if (LIVE && seg.live) live4 = (uint32_t)(seg.live[d0 >> 6] >> (d0 & 63)) & 0xfu;  // d0 % 4 == 0
#pragma unroll
            for (int q = 0; q < 4; q++) {
                bool present = every_doc || sv[q] != 0.0f;  // every_doc: the MatchAllDocsQuery column (all cells 0)
                if (EDGE) present = present && i + q >= first_in && i + q < wlen;
                const bool fresh = o[q] == kSent;
                const float sum = __fadd_rn(fresh ? 0.0f : __uint_as_float(o[q]), sv[q]);
                o[q] = present ? __float_as_uint(sum) : o[q];
                my_matches += (fresh && present && (!LIVE || ((live4 >> q) & 1u))) ? 1u : 0u;
                any_hot |= present && sum > te;
            }
        }
        *reinterpret_cast<uint4*>(acc + i) = make_uint4(o[0], o[1], o[2], o[3]);
        if (!POS) hot |= any_hot ? 1u << (i >> 5) : 0u;
    }
}

// Plain-sum variant, four finished sums of the window (docids win0 + 4 * (g * 32 + lane) ..): count the matches
// (a sum is non-zero iff some clause matched: every clause score is > 0) and keep the lane's running maximum.
// min.u32 through asm: the compiler would otherwise turn min(x, 1) into a compare + a select per element, chained.
__device__ __forceinline__ uint32_t min1(uint32_t x) {
    uint32_t r;
    asm("min.u32 %0, %1, 1;" : "=r"(r) : "r"(x));
    return r;
}
template <bool LIVE>
__device__ __forceinline__ void count_and_max(const uint4 o, int g, int lane, const uint64_t* __restrict__ live, int win0,
                                              uint32_t& matches, float& mx) {
    if (LIVE && live) {
        uint32_t m4 = (o.x != 0u ? 1u : 0u) | (o.y != 0u ? 2u : 0u) | (o.z != 0u ? 4u : 0u) | (o.w != 0u ? 8u : 0u);
        if (m4) {
            const int d0 = win0 + (g * 32 + lane) * 4;
            uint32_t l4 = 0;
#pragma unroll
            for (int q = 0; q < 4; q++) l4 |= ((live[(d0 + q) >> 6] >> ((d0 + q) & 63)) & 1ull) ? 1u << q : 0u;
            m4 &= l4;
        }
        matches += __popc(m4);
    } else {
        matches += (min1(o.x) + min1(o.y)) + (min1(o.z) + min1(o.w));
    }
    mx = fmaxf(fmaxf(mx, __uint_as_float(o.x)), fmaxf(fmaxf(__uint_as_float(o.y), __uint_as_float(o.z)), __uint_as_float(o.w)));
}

// A whole window in which only score columns have postings (plain-sum variant): their sums are formed in registers, in
// clause order from +0.0f exactly like the accumulator would, counted and compared with theta — the window in shared
// memory is neither read nor written.  Returns 0xffffffff when some doc beats theta (the caller then runs the general
// path to scan the window), else this lane's number of matches.  Not inlined: its 24 live float registers must not weigh on the
// register allocation of the stream loops.
template <bool LIVE>
__device__ __noinline__ uint32_t columns_only_window(const WTerm* term, uint32_t active, const uint64_t* __restrict__ live,
                                                     int win0, int hi, float te, int lane) {
    uint32_t c = 0;
    float mx = 0.0f;
    const int win1 = win0 + kWw;
#pragma unroll
    for (int h = 0; h < kWw / 128; h += 3) {
        float4 s3[3];
#pragma unroll
        for (int j = 0; j < 3; j++) s3[j] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        for (uint32_t m = active; m; m &= m - 1) {
            const float* col = reinterpret_cast<const float*>(term[__ffs(m) - 1].blk_last) + win0 + lane * 4;
            float4 v[3];
#pragma unroll
            for (int j = 0; j < 3; j++) v[j] = __ldg(reinterpret_cast<const float4*>(col + (h + j) * 128));
            if (h == 0 && lane < kWw / 32 && win1 + lane * 32 < hi)  // next window's slice towards L2
                asm volatile("prefetch.global.L2 [%0];" ::"l"(col - lane * 4 + kWw + lane * 32));
#pragma unroll
            for (int j = 0; j < 3; j++)
                s3[j] = make_float4(__fadd_rn(s3[j].x, v[j].x), __fadd_rn(s3[j].y, v[j].y), __fadd_rn(s3[j].z, v[j].z),
                                    __fadd_rn(s3[j].w, v[j].w));
        }
#pragma unroll
        for (int j = 0; j < 3; j++)
            count_and_max<LIVE>(make_uint4(__float_as_uint(s3[j].x), __float_as_uint(s3[j].y), __float_as_uint(s3[j].z),
                                           __float_as_uint(s3[j].w)),
                                h + j, lane, live, win0, c, mx);
    }
    return __any_sync(0xffffffffu, mx > te) ? 0xffffffffu : c;
}

template <bool LIVE, bool NOT, bool MSM, bool DMAX, bool POS>
__global__ void __launch_bounds__(kOrThreads, 24)
k_eval_or(EvalParams p, const uint32_t* __restrict__ item_ids, uint32_t n_ids, uint32_t warp_bytes,
          uint32_t kcap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const uint32_t wid = blockIdx.x * kOrWarps + warp;
    if (wid >= n_ids) return;
    unsigned char* base = smem_raw + (size_t)warp * warp_bytes;
    WarpShared& sh = *reinterpret_cast<WarpShared*>(base);
    float* topk = reinterpret_cast<float*>(base + sizeof(WarpShared));
    int32_t* cdocs = reinterpret_cast<int32_t*>(topk + kcap);
    const uint32_t item_idx = item_ids[wid];
    const WorkItem it = p.items[item_idx];
    const SegDev seg = p.segs[it.seg];
    const int T = it.n_terms;
    const int lo = it.lo, hi = it.hi;
    float* cscores = reinterpret_cast<float*>(cdocs + T * kBlock);

    for (int i = lane; i < kWw; i += 32) sh.acc[i] = POS ? 0u : kSent;
    MsmCtx mc;
    mc.cnt = reinterpret_cast<uint8_t*>(cscores + T * kBlock);  // MSM variants reserve kWw more bytes
    mc.msm = max(1u, (uint32_t)it.type >> 4);  // items without min_should_match in an MSM launch: 1
    mc.mx = reinterpret_cast<float*>(mc.cnt + kWw);  // DMAX variant reserves 4 * kWw more bytes
    // DisjunctionMaxScorer item: the tie breaker rides in a meta clause after the item's clauses
    const bool dmax_item = DMAX && (it.type & 4u) != 0;
    const float tie = dmax_item ? p.clauses[it.clause_begin + T].weight : 0.0f;
    if (MSM) {
        for (int i = lane; i < kWw / 4; i += 32) reinterpret_cast<uint32_t*>(mc.cnt)[i] = 0u;
    }
    if (lane < T && (p.clauses[it.clause_begin + lane].flags & 4u)) {
        // score column (a hot, dense clause whose BM25 contributions were materialised once for the
        // whole batch): no stream; the column is read window by window
        const ItemClause c = p.clauses[it.clause_begin + lane];
        WTerm& tc = sh.term[lane];
        tc.blk_last = reinterpret_cast<const int32_t*>(p.cols[c.term_id].col);
        tc.blk_desc = nullptr;
        tc.cache = nullptr;
        tc.nb = 0;
        tc.cur = 1;  // > nb: exhausted as a stream
        tc.n = 0;
        tc.pos = 0;
        tc.term_id = c.term_id;
        tc.w1 = 0.0f;
        tc.is_not = 0;
        tc.is_col = (c.flags & 64u) ? 2 : 1;  // 2: every docid present (MatchAllDocsQuery), cells all 0
        tc.pre = nullptr;
    } else if (lane < T) {
        const ItemClause c = p.clauses[it.clause_begin + lane];
        const TermDev td = seg.terms[c.term_id];
        WTerm& tc = sh.term[lane];
        tc.is_col = 0;
        tc.pre = (c.flags & 128u) ? reinterpret_cast<const uint4*>(p.cols[c.flags >> 16].col) : nullptr;
        tc.blk_last = seg.blk_last + td.blk_begin;
        tc.blk_desc = seg.blk_desc + td.blk_begin;
        tc.cache = p.caches + (size_t)c.cache_id * 256;
        tc.nb = td.n_blocks;
        tc.cur = lower_bound_i32(tc.blk_last, 0, td.n_blocks, lo);
        tc.n = 0;
        tc.pos = 0;
        tc.term_id = c.term_id;
        tc.w1 = __fmul_rn(c.weight, __fadd_rn(p.k1, 1.0f));
        tc.is_not = c.flags & 1u;
    }
    __syncwarp();
    const uint32_t col_mask = __ballot_sync(0xffffffffu, lane < T && sh.term[lane < T ? lane : 0].is_col != 0);
    uint32_t hot = 0, my_matches = 0;
    int nd = kNoMoreDocs;  // lane t: next cached docid of clause t (kNoMoreDocs = exhausted)
    for (int t = 0; t < T; t++) {
        if (stream_refill<LIVE, NOT, MSM, DMAX, POS>(seg, p, sh.term[t], cdocs + t * kBlock, cscores + t * kBlock, lo, hi,
                                                lane, 0, -2147483647 - 1, sh.acc, hot, my_matches, INFINITY, mc)) {
            const int first = cdocs[t * kBlock + sh.term[t].pos];
            if (lane == t) nd = first;
        }
    }
    // a column clause has a (potential) posting at every docid: windows become contiguous and
    // 4-aligned (16-byte column loads) from the start of the range
    if (lane < T && sh.term[lane].is_col && lo < hi) nd = lo & ~3;
    long long w0 = __reduce_min_sync(0xffffffffu, nd);

    WEmit em;
    em.topk = topk;
    em.topk_n = 0;
    em.theta_local = -INFINITY;
    em.theta_in = 0;
    em.run_slot = kNone;
    em.run_cap = 0;
    em.run_cnt = 0;
    em.matches = 0;
    em.overflow = false;
    wtheta_inherit(em, p, item_idx, it.chain_pos, kcap, lane);
    // theta look-back: the up-to-32 preceding items of this heap chain (each publishes
    // max(own, inherited)), re-read every 8 windows
    const bool lb_ok = (uint32_t)lane < it.chain_pos;
    const uint32_t* theta_lb = p.item_theta + item_idx - 1 - (lb_ok ? lane : 0);
    uint32_t win_no = 0;

    while (w0 < hi) {
        const int win0 = (int)w0;
        const int win1 = (int)min((long long)hi, w0 + kWw);
        uint32_t inherited = 0;
        if ((win_no++ & 7u) == 0 && it.chain_pos) {
            inherited = lb_ok ? ld_volatile_u32(theta_lb) : 0u;
            inherited = __reduce_max_sync(0xffffffffu, inherited);
        }
        hot = 0;
        if (inherited > em.theta_in) {
            // hand an inherited bound on at once: an item that finds no candidate of its own never reaches
            // wtheta_update, and its successors look back over 32 items only
            em.theta_in = inherited;
            if (lane == 0) atomicMax(p.item_theta + item_idx, inherited);
        }
        float te = em.theta_local;
        if (em.theta_in > kOrderedNegInf) te = fmaxf(te, ordered_to_float(em.theta_in));
        const bool open = !POS && te == -INFINITY;
        if (POS) te = fmaxf(te, 0.0f);  // every match scores > 0: "heap still open" needs no case of its own
        // ---- clauses with a posting in this window, in clause order: drain each stream up to the
        // window end (a sparse clause sits out most windows)
        uint32_t active = __ballot_sync(0xffffffffu, nd < win1);
        if (POS && active && (active & ~col_mask) == 0u && win1 - win0 == kWw && win0 >= lo) {
            // Only score columns have postings in this (whole) window: see columns_only_window.  Only if a doc beats
            // theta (rare) the general path below redoes the window to scan it.
            const uint32_t cnt = columns_only_window<LIVE>(sh.term, active, seg.live, win0, hi, te, lane);
            if (cnt != 0xffffffffu) {
                my_matches += cnt;
                if ((active >> lane) & 1u) nd = win1 < hi ? win1 : kNoMoreDocs;
                const int next_doc = __reduce_min_sync(0xffffffffu, nd);
                if (next_doc == kNoMoreDocs) break;
                w0 = next_doc;
                continue;
            }
        }
        while (active) {
            const int t = __ffs(active) - 1;
            active &= active - 1;
            WTerm& tc = sh.term[t];
            if (tc.is_col) {
                const float* col = reinterpret_cast<const float*>(tc.blk_last);
                const int wlen = win1 - win0;
                // the next window's slice of the column (kWw * 4 bytes = 24 lines) towards L1/L2 now:
                // columns are far larger than L2, and the loads below would otherwise serialise
                if (lane < kWw / 32 && win1 + lane * 32 < hi)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(col + win1 + lane * 32));
                const int first_in = lo - win0;  // > 0 only in the first window of a range
                const bool every_doc = tc.is_col == 2;
                if (MSM || DMAX) {  // per-doc clause counters / maxima: the scalar path
                    for (int i = lane * 4; i < wlen; i += 128) {
                        const int d0 = win0 + i;
                        const float4 v = __ldg(reinterpret_cast<const float4*>(col + d0));
                        const float sv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                        for (int q = 0; q < 4; q++) {
                            const int d = d0 + q;
                            if ((every_doc || sv[q] != 0.0f) && d >= lo && d < win1)
                                accumulate_posting<NOT, MSM, DMAX>(sh.acc, i + q, sv[q], false,
                                                                   LIVE ? is_live(seg, d) : true, te, hot, my_matches, mc);
                        }
                    }
                } else if (first_in > 0 || (wlen & 3)) {  // warp-uniform: first / last window of a range
                    column_window<LIVE, true, POS>(sh.acc, col, every_doc, seg, win0, wlen, first_in, te, lane, hot, my_matches);
                } else {
                    column_window<LIVE, false, POS>(sh.acc, col, every_doc, seg, win0, wlen, first_in, te, lane, hot, my_matches);
                }
                if (lane == t) nd = win1 < hi ? win1 : kNoMoreDocs;
                __syncwarp();
                continue;
            }
            const int32_t* cd = cdocs + t * kBlock;
            const float* cs = cscores + t * kBlock;
            uint32_t pos = tc.pos, n = tc.n;
            for (;;) {
                if (pos >= n) {
                    if (tc.cur > tc.nb) break;  // exhausted
                    __syncwarp();  // every lane has read tc.pos / tc.n / tc.cur before lane 0 rewrites them in there
                    if (!stream_refill<LIVE, NOT, MSM, DMAX, POS>(seg, p, tc, cdocs + t * kBlock, cscores + t * kBlock, lo, hi,
                                                             lane, win0, win1, sh.acc, hot, my_matches, te, mc)) {
                        pos = n = 0;
                        break;
                    }
                    pos = tc.pos;
                    n = tc.n;
                }
                const uint32_t i = pos + lane;
                const int d = i < n ? cd[i] : kNoMoreDocs;
                const float sv = i < n ? cs[i] : 0.0f;  // (loaded next to the docid, not behind the vote)
                const bool in_win = d < win1;
                const uint32_t c = __popc(__ballot_sync(0xffffffffu, in_win));  // sorted: a prefix
                if (in_win)
                    accumulate_posting<NOT, MSM, DMAX, POS>(sh.acc, d - win0, sv, NOT && tc.is_not != 0,
                                                            (LIVE && !POS) ? is_live(seg, d) : true, te, hot, my_matches, mc);
                pos += c;
                if (c < 32 && pos < n) break;  // next cached doc is beyond this window
            }
            // every lane stores the same cursor: each later reads back (at least) its own store (stream_refill, which
            // lets lane 0 write, synchronises on its own)
            tc.pos = pos;
            tc.n = n;
            const int nx = pos < n ? cd[pos] : kNoMoreDocs;
            if (lane == t) nd = nx;
            __syncwarp();  // the next clause's lanes read window slots other lanes have just written
        }
        const int next_doc = __reduce_min_sync(0xffffffffu, nd);
        if (POS) {
            // one pass over the finished window: a doc matched iff its sum is non-zero (every clause score is > 0), and
            // a 32-doc step is scanned for candidates iff one of its sums beats theta
            hot = 0;
            float mx = 0.0f;
#pragma unroll
            for (int g = 0; g < kWw / 128; g++)
                count_and_max<LIVE>(reinterpret_cast<const uint4*>(sh.acc)[g * 32 + lane], g, lane, seg.live, win0, my_matches, mx);
            if (__any_sync(0xffffffffu, mx > te)) {  // a few percent of the windows: which 32-doc steps hold such a sum
#pragma unroll
                for (int g = 0; g < kWw / 128; g++) {
                    const float4 o = reinterpret_cast<const float4*>(sh.acc)[g * 32 + lane];
                    hot |= fmaxf(fmaxf(o.x, o.y), fmaxf(o.z, o.w)) > te ? 1u << (g * 4 + (lane >> 3)) : 0u;
                }
            }
        }
        hot = __reduce_or_sync(0xffffffffu, hot);
        {
            uint32_t newc_n = 0;
            while (hot) {
                const int s = __ffs(hot) - 1;
                hot &= hot - 1;
                const int idx = s * 32 + lane;
                const uint32_t v = sh.acc[idx];
                float sc = __uint_as_float(v);
                if (DMAX && dmax_item) {  // score_max: max + (sum - max) * tie_breaker_multiplier
                    const float m = mc.mx[idx];
                    sc = __fadd_rn(m, __fmul_rn(__fsub_rn(sc, m), tie));
                }
                const bool cand = POS ? (sc > te && (LIVE ? is_live(seg, win0 + idx) : true))
                                      : (v != kSent && (!NOT || v != kExcl) && (open || sc > te) &&
                                         (!MSM || mc.cnt[idx] >= mc.msm) && (LIVE ? is_live(seg, win0 + idx) : true));
                const uint32_t cm = __ballot_sync(0xffffffffu, cand);
                if (!cm || em.overflow) continue;
                const uint32_t c = __popc(cm);
                CandRun* hdr = reinterpret_cast<CandRun*>(p.cand_arena);
                if (em.run_slot == kNone || em.run_cnt + c > em.run_cap) {
                    uint32_t slot = 0;
                    const uint32_t cap = em.run_slot == kNone ? kRunFirst : kRunMin;
                    if (lane == 0) {
                        const unsigned long long s64 = atomicAdd(p.arena_next, (unsigned long long)cap + 1ull);
                        slot = (s64 + cap + 1ull > (unsigned long long)p.arena_slots) ? kNone : (uint32_t)s64;
                        if (slot == kNone) atomicOr(p.error_flag, 1u);
                        else if (em.run_slot == kNone) p.item_head[item_idx] = slot;
                        else hdr[em.run_slot] = CandRun{slot, em.run_cnt};
                    }
                    slot = __shfl_sync(0xffffffffu, slot, 0);
                    if (slot == kNone) {
                        em.overflow = true;
                        continue;
                    }
                    em.run_slot = slot;
                    em.run_cap = cap;
                    em.run_cnt = 0;
                }
                if (cand) {
                    const uint32_t r = __popc(cm & ((1u << lane) - 1u));
                    p.cand_arena[em.run_slot + 1 + em.run_cnt + r] = rg_hit{win0 + idx + seg.doc_base, sc};
                    if (newc_n + r < (uint32_t)kNewcW) sh.newc[newc_n + r] = sc;
                }
                em.run_cnt += c;
                newc_n += c;
                if (lane == 0) hdr[em.run_slot] = CandRun{kNone, em.run_cnt};
            }
            __syncwarp();
#pragma unroll
            for (int g = 0; g < kWw / 128; g++) {
                const uint32_t z = POS ? 0u : kSent;
                reinterpret_cast<uint4*>(sh.acc)[g * 32 + lane] = make_uint4(z, z, z, z);
            }
            if (MSM) {
                for (int i = lane; i < kWw / 16; i += 32) reinterpret_cast<uint4*>(mc.cnt)[i] = make_uint4(0, 0, 0, 0);
            }
            wtheta_update(em, p.k, kcap, lane, sh.newc, newc_n, p.item_theta + item_idx);
            __syncwarp();
        }
        if (next_doc == kNoMoreDocs) break;
        w0 = next_doc;
    }
    my_matches = __reduce_add_sync(0xffffffffu, my_matches);
    if (lane == 0) p.item_matches[item_idx] = my_matches;
}

// ------------------------------------------------------------------------------------------
// k_eval_and
// ------------------------------------------------------------------------------------------
constexpr int kAndSlots = kEvalWarps * kBlock;  // 1024 lead docs per step
constexpr int kAndSteps = kBlock / 32;          // 4 slots per lane

struct AndShared {
    int32_t ldoc[kAndSlots];
    float lscore[kAndSlots];
    int32_t slab_docs[kEvalWarps][kBlock];
    int32_t slab_freqs[kEvalWarps][kBlock];
    TermCtx term[kMaxTerms];
    uint32_t term_id[kMaxTerms];
    uint32_t is_not[kMaxTerms];            // MUST_NOT clauses: a hit kills the lead doc, a miss keeps it
    uint32_t is_opt[kMaxTerms];            // SHOULD clauses next to a MUST (ReqOptScorer's optional side)
    const float* colp[kMaxTerms];          // non-lead clause read from its score column (one gather per lead doc)
    uint32_t hint[kEvalWarps][kMaxTerms];  // per-warp galloping hints into the skip tables
    // ReqOptScorer (search/scorer/req_opt_scorer.rs:19-65): optional-side sums per lead slot, the
    // per-step match masks in docid order, and the scorer's sequential state (thread 0 owns it)
    float oscore[kAndSlots];
    uint32_t mmask[kEvalWarps][kAndSteps];
    EmitShared emit;
};

// A (query, leaf) with MUST and SHOULD clauses.  required = the lead-list conjunction above;
// optional = DisjunctionSumScorer over the SHOULD clauses present in the leaf, summed in clause
// order from 0.0f.  score() keeps running (scores_sum, scores_num) over the REQUIRED scores of the
// docs whose optional side it looked at; after more than 100 of them a doc with
// 2*req < scores_sum/scores_num returns req alone and leaves the state untouched.  That state is a
// sequential f32 chain over the collected (live, not excluded) docs of the leaf, so such a work
// item always covers the whole leaf and one thread replays the chain per step, in docid order.
constexpr uint32_t kOptScoreThreshold = 100;

// OTHER: some leaf carries EF / BITSET doc blocks (their decoder is compiled out otherwise)
template <bool REQOPT, bool OTHER>
__global__ void __launch_bounds__(kEvalThreads, OTHER ? (REQOPT ? 4 : 5) : 0)  // the decoder call must not cost occupancy
k_eval_and(EvalParams p, const uint32_t* __restrict__ item_ids) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    AndShared& sh = *reinterpret_cast<AndShared*>(smem_raw);
    const uint32_t item_idx = item_ids[blockIdx.x];
    const WorkItem it = p.items[item_idx];
    const SegDev seg = p.segs[it.seg];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const int T = it.n_terms;
    const int lo = it.lo, hi = it.hi;

    emit_init(sh.emit);
    if ((int)threadIdx.x < T) {
        const ItemClause c = p.clauses[it.clause_begin + threadIdx.x];
        const bool is_col = (c.flags & 4u) != 0;  // term_id indexes p.cols then (never the lead clause)
        const TermDev td = is_col ? TermDev{} : seg.terms[c.term_id];
        TermCtx& tc = sh.term[threadIdx.x];
        sh.term_id[threadIdx.x] = c.term_id;
        sh.is_not[threadIdx.x] = c.flags & 1u;
        sh.is_opt[threadIdx.x] = (c.flags >> 1) & 1u;
        sh.colp[threadIdx.x] = is_col ? p.cols[c.term_id].col : nullptr;
        tc.blk_last = seg.blk_last + td.blk_begin;
        tc.blk_desc = seg.blk_desc + td.blk_begin;
        tc.cache = p.caches + (size_t)c.cache_id * 256;
        tc.nb = td.n_blocks;
        tc.cur = lower_bound_i32(tc.blk_last, 0, td.n_blocks, lo);
        tc.next_cur = 0;
        tc.tail_base = td.tail_base;
        tc.tail_n = td.tail_n;
        tc.tail_pos = 0;
        tc.tail_next = 0;
        tc.w1 = __fmul_rn(c.weight, __fadd_rn(p.k1, 1.0f));
    }
    const uint32_t* theta_prev = (it.chain_pos == 0) ? nullptr : p.item_theta + (item_idx - 1);
    __syncthreads();

    const TermCtx& lead = sh.term[0];
    const uint32_t lead_nb = lead.nb;
    const bool lead_has_tail = lead.tail_n > 0 && (lead_nb == 0 || hi - 1 > lead.tail_base);
    if (lane < kMaxTerms) sh.hint[warp][lane] = 0;
    __syncwarp();
    float ro_sum = 0.0f;    // ReqOptScorer::scores_sum / scores_num (thread 0)
    uint32_t ro_num = 0;
    uint32_t touched = 0;   // bytes this thread asked for (block parts are charged to lane 0 of the decoding warp)

    for (uint32_t b0 = lead.cur;; b0 += kEvalWarps) {
        // ---- 1. decode this step's lead blocks (one per warp; pseudo-block lead_nb = vint tail)
        if (b0 > lead_nb || (b0 == lead_nb && !lead_has_tail)) break;
        {
            const int first_prev = b0 == 0 ? -1 : __ldg(lead.blk_last + b0 - 1);
            if (first_prev >= hi - 1) break;
        }
        uint32_t inherited = 0;
        if (threadIdx.x == 0 && theta_prev) inherited = ld_volatile_u32(theta_prev);
        const uint32_t b = b0 + warp;
        int4 ld = make_int4(kNoMoreDocs, kNoMoreDocs, kNoMoreDocs, kNoMoreDocs);
        float4 ls = make_float4(0.f, 0.f, 0.f, 0.f);
        const float lw1 = lead.w1;
        if (b < lead_nb) {
            const int prev_last = b == 0 ? -1 : __ldg(lead.blk_last + b - 1);
            if (prev_last < hi - 1) {
                const BlockDesc bd = lead.blk_desc[b];
                const uint4* part = seg.arena + bd.off16;
                if (lane == 0) touched += 12u + 16u * (((bd.bits >> 16) & 0xffu) + max(1u, (bd.bits >> 8) & 0xffu));
                int4 dd;
                if (!OTHER || (bd.bits >> 24) == 0) {
                    const int4 dl = unpack4(part, (int)(bd.bits & 0xff), lane, seg.version, seg.sb_mask);
                    dd = deltas_to_docs(dl, b == 0 ? 0 : prev_last);
                } else {  // EF / BITSET doc part (this warp's ldoc slice is rewritten below)
                    decode_other_docs_call(part, bd.bits >> 24, b == 0 ? -1 : prev_last, sh.ldoc + warp * kBlock, lane);
                    dd = reinterpret_cast<const int4*>(sh.ldoc + warp * kBlock)[lane];
                    __syncwarp();
                }
                const int4 fr = unpack4(part + ((bd.bits >> 16) & 0xff), (int)((bd.bits >> 8) & 0xff), lane,
                                        seg.version, seg.sb_mask);
                const int docs[4] = {dd.x, dd.y, dd.z, dd.w};
                const int fq[4] = {fr.x, fr.y, fr.z, fr.w};
                int od[4];
                float os[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int d = docs[i];
                    const bool ok = d >= lo && d < hi;
                    od[i] = ok ? d : kNoMoreDocs;
                    float s = 0.f;
                    if (ok) {
                        const float nrm = seg.norms ? __ldg(lead.cache + __ldg(seg.norms + d)) : p.k1;
                        s = bm25_score(lw1, (float)fq[i], nrm);
                        touched += 1u;
                    }
                    os[i] = s;
                }
                ld = make_int4(od[0], od[1], od[2], od[3]);
                ls = make_float4(os[0], os[1], os[2], os[3]);
            }
            reinterpret_cast<int4*>(sh.ldoc + warp * kBlock)[lane] = ld;
            reinterpret_cast<float4*>(sh.lscore + warp * kBlock)[lane] = ls;
        } else {
            reinterpret_cast<int4*>(sh.ldoc + warp * kBlock)[lane] = ld;
            reinterpret_cast<float4*>(sh.lscore + warp * kBlock)[lane] = ls;
            __syncwarp();
            if (b == lead_nb && lead_has_tail) {
                if (lane == 0) {
                    decode_tail(seg, seg.terms[sh.term_id[0]], sh.slab_docs[warp], sh.slab_freqs[warp]);
                }
                __syncwarp();
                for (uint32_t j = lane; j < lead.tail_n; j += 32) {
                    const int d = sh.slab_docs[warp][j];
                    if (d >= lo && d < hi) {
                        const float nrm = seg.norms ? __ldg(lead.cache + __ldg(seg.norms + d)) : p.k1;
                        sh.ldoc[warp * kBlock + j] = d;
                        sh.lscore[warp * kBlock + j] = bm25_score(lw1, (float)sh.slab_freqs[warp][j], nrm);
                    }
                }
            }
        }
        if (REQOPT) {
#pragma unroll
            for (int r = 0; r < kAndSteps; r++) sh.oscore[warp * kBlock + r * 32 + lane] = __uint_as_float(kSent);
        }
        __syncwarp();
        // ---- 2. every other clause, in cost order; each warp works on its own 128 lead slots
        for (int t = 1; t < T; t++) {
            const TermCtx& tc = sh.term[t];
            const uint32_t nb = tc.nb;
            const float w1 = tc.w1;
            const bool neg = sh.is_not[t] != 0;
            const bool opt = REQOPT && sh.is_opt[t] != 0;
            if (const float* col = sh.colp[t]) {
                // the clause's BM25 contributions sit in a docid-indexed column (+0.0f = no posting): no skip
                // search, no block decode — the same f32 value the stream path would compute
#pragma unroll
                for (int r = 0; r < kAndSteps; r++) {
                    const int slot = warp * kBlock + r * 32 + lane;
                    const int d = sh.ldoc[slot];
                    if (d == kNoMoreDocs) continue;
                    const float v = __ldg(col + d);
                    touched += 4u;
                    if (v != 0.0f) {
                        if (neg) {
                            sh.ldoc[slot] = kNoMoreDocs;  // ReqNotScorer: excluded
                        } else if (opt) {
                            const float o = sh.oscore[slot];
                            sh.oscore[slot] = __fadd_rn(__float_as_uint(o) == kSent ? 0.0f : o, v);
                        } else {
                            sh.lscore[slot] = __fadd_rn(sh.lscore[slot], v);
                        }
                    } else if (!neg && !opt) {
                        sh.ldoc[slot] = kNoMoreDocs;
                    }
                }
                __syncwarp();
                continue;
            }
            for (int r = 0; r < kAndSteps; r++) {
                const int slot = warp * kBlock + r * 32 + lane;
                int d = sh.ldoc[slot];
                bool pending = d != kNoMoreDocs;
                uint32_t bi = 0;
                if (pending) {
                    touched += 8u;  // skip-table probe (galloping search)
                    bi = lower_bound_gallop(tc.blk_last, min(sh.hint[warp][t], nb), nb, d);
                    if (bi == nb && !(tc.tail_n > 0 && (nb == 0 || d > tc.tail_base))) {
                        pending = false;  // beyond the last posting of this clause
                        if (!neg && !opt) sh.ldoc[slot] = kNoMoreDocs;
                    }
                }
                uint32_t pend_mask = __ballot_sync(0xffffffffu, pending);
                __syncwarp();
                if (pend_mask) {
                    const int last_lane = 31 - __clz(pend_mask);
                    const uint32_t hb = __shfl_sync(0xffffffffu, bi, last_lane);
                    if (lane == 0) sh.hint[warp][t] = hb;
                }
                __syncwarp();
                while (pend_mask) {
                    const int leader = __ffs(pend_mask) - 1;
                    const uint32_t cb = __shfl_sync(0xffffffffu, bi, leader);
                    const bool full_block = cb < nb;
                    BlockDesc bd{};
                    if (full_block) {
                        bd = tc.blk_desc[cb];
                        if (lane == 0) touched += 12u + 16u * ((bd.bits >> 16) & 0xffu);
                        const int base = cb == 0 ? 0 : __ldg(tc.blk_last + cb - 1);
                        const uint4* part = seg.arena + bd.off16;
                        if (!OTHER || (bd.bits >> 24) == 0) {
                            const int4 dl = unpack4(part, (int)(bd.bits & 0xff), lane, seg.version, seg.sb_mask);
                            const int4 dd = deltas_to_docs(dl, base);
                            reinterpret_cast<int4*>(sh.slab_docs[warp])[lane] = dd;
                        } else {
                            decode_other_docs_call(part, bd.bits >> 24, cb == 0 ? -1 : base, sh.slab_docs[warp], lane);
                        }
                    } else if (lane == 0) {
                        decode_tail(seg, seg.terms[sh.term_id[t]], sh.slab_docs[warp], sh.slab_freqs[warp]);
                    }
                    __syncwarp();
                    const int n_in = cb < nb ? kBlock : (int)tc.tail_n;
                    const bool mine = pending && bi == cb;
                    if (mine) {
                        int l = 0, h = n_in;
                        while (l < h) {
                            const int m = (l + h) >> 1;
                            if (sh.slab_docs[warp][m] < d) l = m + 1;
                            else h = m;
                        }
                        if (l < n_in && sh.slab_docs[warp][l] == d && neg) {
                            sh.ldoc[slot] = kNoMoreDocs;  // ReqNotScorer: excluded
                        } else if (l < n_in && sh.slab_docs[warp][l] == d) {
                            int f;
                            if (full_block) {
                                f = extract1(seg.arena + bd.off16 + ((bd.bits >> 16) & 0xff),
                                             (int)((bd.bits >> 8) & 0xff), l, seg.version, seg.sb_mask);
                            } else {
                                f = sh.slab_freqs[warp][l];
                            }
                            const float nrm = seg.norms ? __ldg(tc.cache + __ldg(seg.norms + d)) : p.k1;
                            const float sc = bm25_score(w1, (float)f, nrm);
                            touched += 9u;  // freq word(s) + norm byte
                            if (opt) {  // DisjunctionSumScorer::score_sum: clause order, from 0.0f
                                const float o = sh.oscore[slot];
                                sh.oscore[slot] = __fadd_rn(__float_as_uint(o) == kSent ? 0.0f : o, sc);
                            } else {
                                sh.lscore[slot] = __fadd_rn(sh.lscore[slot], sc);
                            }
                        } else if (!neg && !opt) {
                            sh.ldoc[slot] = kNoMoreDocs;
                        }
                        pending = false;
                    }
                    __syncwarp();
                    pend_mask = __ballot_sync(0xffffffffu, pending);
                }
            }
            __syncwarp();
        }
        // ---- 2b. ReqOptScorer::score over this step's collected docs, in docid order
        if (REQOPT) {
#pragma unroll
            for (int r = 0; r < kAndSteps; r++) {
                const int d = sh.ldoc[warp * kBlock + r * 32 + lane];
                const uint32_t m = __ballot_sync(0xffffffffu, d != kNoMoreDocs && is_live(seg, d));
                if (lane == 0) sh.mmask[warp][r] = m;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                for (int w = 0; w < kEvalWarps; w++) {
                    for (int r = 0; r < kAndSteps; r++) {
                        uint32_t m = sh.mmask[w][r];
                        while (m) {
                            const int slot = w * kBlock + r * 32 + __ffs(m) - 1;
                            m &= m - 1;
                            const float req = sh.lscore[slot];
                            if (ro_num > kOptScoreThreshold &&
                                __fmul_rn(2.0f, req) < __fdiv_rn(ro_sum, __uint2float_rn(ro_num)))
                                continue;  // required score only; state untouched (:46-49)
                            ro_sum = __fadd_rn(ro_sum, req);
                            ro_num++;
                            const float o = sh.oscore[slot];
                            if (__float_as_uint(o) != kSent) sh.lscore[slot] = __fadd_rn(req, o);
                        }
                    }
                }
            }
            __syncthreads();
        }
        // ---- 3. surviving lead docs are the matches of this step, in docid order
        bool present[kAndSteps];
        int doc[kAndSteps];
        float score[kAndSteps];
#pragma unroll
        for (int s = 0; s < kAndSteps; s++) {
            const int slot = warp * kBlock + s * 32 + lane;
            doc[s] = sh.ldoc[slot];
            score[s] = sh.lscore[slot];
            present[s] = doc[s] != kNoMoreDocs && is_live(seg, doc[s]);
        }
        emit_window<kAndSteps>(sh.emit, p, item_idx, seg.doc_base, present, doc, score, inherited);
        __syncthreads();
    }
    __syncthreads();
    if (threadIdx.x == 0) p.item_matches[item_idx] = sh.emit.matches;
    touched = __reduce_add_sync(0xffffffffu, touched);
    if (lane == 0 && touched) atomicAdd(p.touched, (unsigned long long)touched);
}

// ------------------------------------------------------------------------------------------
// exact TopDocsCollector heap (one lane drives it; the warp pre-filters)
// ------------------------------------------------------------------------------------------
struct Heap {
    rg_hit* data;  // shared memory, capacity k
    uint32_t n;
    uint32_t k;
    // reversed PartialOrd on score only (sort_field/collapse_top_docs.rs:54-60):
    //   a <= b  <=>  a.score >= b.score
    __device__ static bool le(const rg_hit& a, const rg_hit& b) { return a.score >= b.score; }
    __device__ static bool ge(const rg_hit& a, const rg_hit& b) { return a.score <= b.score; }
    __device__ void sift_up(uint32_t start, uint32_t pos) {
        const rg_hit e = data[pos];
        while (pos > start) {
            const uint32_t parent = (pos - 1) / 2;
            if (le(e, data[parent])) break;
            data[pos] = data[parent];
            pos = parent;
        }
        data[pos] = e;
    }
    __device__ void sift_down_range(uint32_t pos, uint32_t end) {
        const rg_hit e = data[pos];
        uint32_t child = 2 * pos + 1;
        while (child < end) {
            const uint32_t right = child + 1;
            if (right < end && le(data[child], data[right])) child = right;
            if (ge(e, data[child])) break;
            data[pos] = data[child];
            pos = child;
            child = 2 * pos + 1;
        }
        data[pos] = e;
    }
    __device__ void sift_down_to_bottom(uint32_t pos) {
        const uint32_t end = n, start = pos;
        const rg_hit e = data[pos];
        uint32_t child = 2 * pos + 1;
        while (child < end) {
            const uint32_t right = child + 1;
            if (right < end && le(data[child], data[right])) child = right;
            data[pos] = data[child];
            pos = child;
            child = 2 * pos + 1;
        }
        data[pos] = e;
        sift_up(start, pos);
    }
    __device__ void add_doc(const rg_hit& h) {  // top_docs.rs:67-76
        if (n < k) {
            data[n] = h;
            n++;
            sift_up(0, n - 1);
        } else if (n > 0 && data[0].score < h.score) {
            data[0] = h;
            sift_down_range(0, n);
        }
    }
    __device__ rg_hit pop() {
        rg_hit item = data[n - 1];
        n--;
        if (n > 0) {
            const rg_hit top = data[0];
            data[0] = item;
            item = top;
            sift_down_to_bottom(0);
        }
        return item;
    }
};

constexpr int kReplayWarps = 4;

// warp-cooperative: feed `cnt` candidates starting at `src` (global memory) through add_doc
__device__ void replay_run(Heap& hp, const rg_hit* __restrict__ src, uint32_t cnt) {
    const int lane = lane_id();
    for (uint32_t base = 0; base < cnt; base += 32) {
        const uint32_t i = base + lane;
        const bool has = i < cnt;
        rg_hit c = has ? src[i] : rg_hit{0, 0.f};
        uint32_t pending = __ballot_sync(0xffffffffu, has);
        while (pending) {
            const uint32_t n = hp.n;
            const float root = n ? hp.data[0].score : 0.f;
            const bool ok = has && ((pending >> lane) & 1u) && (n < hp.k || root < c.score);
            const uint32_t acc = __ballot_sync(0xffffffffu, ok);
            if (!acc) break;
            const int l = __ffs(acc) - 1;
            rg_hit pick;
            pick.doc = __shfl_sync(0xffffffffu, c.doc, l);
            pick.score = __shfl_sync(0xffffffffu, c.score, l);
            if (lane == 0) hp.add_doc(pick);
            __syncwarp();
            hp.n = __shfl_sync(0xffffffffu, hp.n, 0);
            pending &= ~((2u << l) - 1u);
        }
    }
}

// top_docs(): pop min(total_hits, len) times and reverse (top_docs.rs:55-65)
__device__ void finish_sorted(Heap& hp, unsigned long long total, rg_hit* out, uint32_t* out_count,
                              unsigned long long* out_total) {
    if (lane_id() == 0) {
        const uint32_t n = (uint32_t)min((unsigned long long)hp.n, total);
        for (uint32_t i = 0; i < n; i++) out[n - 1 - i] = hp.pop();
        *out_count = n;
        *out_total = total;
    }
}

__global__ void __launch_bounds__(kReplayWarps * 32)
k_heap_replay(ReplayParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const uint32_t g = blockIdx.x * kReplayWarps + warp;
    if (g >= p.n_groups) return;
    Heap hp;
    hp.data = reinterpret_cast<rg_hit*>(smem_raw) + (size_t)warp * p.k;
    hp.n = 0;
    hp.k = p.k;
    unsigned long long total = 0;
    const CandRun* hdr = reinterpret_cast<const CandRun*>(p.cand_arena);
    for (uint32_t item = p.group_item_begin[g]; item < p.group_item_begin[g + 1]; item++) {
        total += p.item_matches[item];
        uint32_t run = p.item_head[item];
        while (run != kNone) {
            const CandRun h = hdr[run];
            replay_run(hp, p.cand_arena + run + 1, h.count);
            run = h.next;
        }
    }
    __syncwarp();
    const uint32_t q = p.group_query[g];
    if (p.leaf_records) {
        // LeafTopDocs { docs: heap.into_vec(), total_hits } (top_docs.rs:203-213)
        uint8_t* rec = p.leaf_records + (size_t)q * leaf_record_bytes(p.k);
        if (lane == 0) {
            reinterpret_cast<uint32_t*>(rec)[0] = hp.n;
            reinterpret_cast<uint32_t*>(rec)[1] = 0;
            reinterpret_cast<unsigned long long*>(rec)[1] = total;
        }
        rg_hit* dst = reinterpret_cast<rg_hit*>(rec + 16);
        for (uint32_t i = lane; i < hp.n; i += 32) dst[i] = hp.data[i];
    } else {
        finish_sorted(hp, total, p.out_hits + (size_t)q * p.k, p.out_counts + q, p.out_total + q);
    }
}

// finish_parallel (top_docs.rs:157-172): leaves in leaf order, each leaf's docs in heap-array
// order through add_doc; total_hits summed.
__global__ void __launch_bounds__(kReplayWarps * 32)
k_merge_leaf_records(const uint8_t* __restrict__ records, uint32_t n_leaves, uint32_t n_queries,
                     uint32_t k, rg_hit* out_hits, uint32_t* out_counts, unsigned long long* out_total) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * kReplayWarps + warp;
    if (q >= n_queries) return;
    Heap hp;
    hp.data = reinterpret_cast<rg_hit*>(smem_raw) + (size_t)warp * k;
    hp.n = 0;
    hp.k = k;
    unsigned long long total = 0;
    const size_t rb = leaf_record_bytes(k);
    for (uint32_t leaf = 0; leaf < n_leaves; leaf++) {
        const uint8_t* rec = records + ((size_t)leaf * n_queries + q) * rb;
        const uint32_t n = reinterpret_cast<const uint32_t*>(rec)[0];
        total += reinterpret_cast<const unsigned long long*>(rec)[1];
        replay_run(hp, reinterpret_cast<const rg_hit*>(rec + 16), min(n, k));
    }
    __syncwarp();
    finish_sorted(hp, total, out_hits + (size_t)q * k, out_counts + q, out_total + q);
}

// ------------------------------------------------------------------------------------------
// k_build_columns — batch-level common subexpression: the BM25 contributions of a hot, dense
// (term, weight, norm cache) are the same f32 values for every query of the batch that carries
// the clause, so they are decoded / gathered / divided ONCE into a docid-indexed f32 column
// (+0.0f = no posting; only clauses whose every score is > 0 get one) that k_eval_or then reads with 16-byte loads.  One warp per
// 128-posting block (or vint tail) of a job's term.
// ------------------------------------------------------------------------------------------
constexpr int kColWarps = 4;
// BITMAP = true: the same walk over a term's blocks, but every posting sets its presence bit in the term's
// bitmap (built once per segment at upload; weight / norms are not touched).
// MODE 4: scored posting list — per block 128 docids + 128 BM25 scores (1 KB), what stream_refill would compute.
// MODE 0: score column, 1: presence bitmap, 2: tf-norm planes (bit set when f/(f+norm), rounded up, exceeds the job's
// tau1 / tau2), 3: histogram of that factor over a sample of the job's blocks
template <int MODE>
__global__ void __launch_bounds__(kColWarps * 32)
k_build_columns(const SegDev* __restrict__ segs, const ColumnJob* __restrict__ jobs, uint32_t n_jobs,
                uint32_t n_units, const float* __restrict__ caches, float k1, uint32_t* __restrict__ hist,
                size_t plane_stride) {
    constexpr bool BITMAP = MODE == 1;
    __shared__ __align__(16) int32_t s_docs[kColWarps][kBlock];
    __shared__ __align__(16) int32_t s_freqs[kColWarps][kBlock];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const uint32_t unit = blockIdx.x * kColWarps + warp;
    if (unit >= n_units) return;
    uint32_t jl = 0, jh = n_jobs;  // last job with unit_begin <= unit
    while (jl + 1 < jh) {
        const uint32_t m = (jl + jh) >> 1;
        if (jobs[m].unit_begin <= unit) jl = m;
        else jh = m;
    }
    const ColumnJob job = jobs[jl];
    const SegDev seg = segs[job.seg];
    const TermDev td = seg.terms[job.term_id];
    const uint32_t b = unit - job.unit_begin;
    if (MODE == 3 && (b & 7u) != 0u && b < td.n_blocks) return;  // a sample: every 8th block (and the tail)
    int4 docs, freqs = make_int4(1, 1, 1, 1);
    if (b < td.n_blocks) {
        const BlockDesc bd = seg.blk_desc[td.blk_begin + b];
        const int base = b == 0 ? 0 : __ldg(seg.blk_last + td.blk_begin + b - 1);
        const uint4* part = seg.arena + bd.off16;
        const uint32_t enc = bd.bits >> 24;
        if (enc == 0) {
            docs = deltas_to_docs(unpack4(part, (int)(bd.bits & 0xff), lane, seg.version, seg.sb_mask), base);
        } else {
            decode_other_docs(part, enc, b == 0 ? -1 : base, s_docs[warp], lane);
            docs = reinterpret_cast<const int4*>(s_docs[warp])[lane];
        }
        if (!BITMAP)
            freqs = unpack4(part + ((bd.bits >> 16) & 0xff), (int)((bd.bits >> 8) & 0xff), lane, seg.version, seg.sb_mask);
    } else {
        const int n_in = (int)td.tail_n;
        if (lane == 0) decode_tail(seg, td, s_docs[warp], s_freqs[warp]);
        __syncwarp();
        const int i0 = 4 * lane;
        docs = make_int4(i0 < n_in ? s_docs[warp][i0] : -1, i0 + 1 < n_in ? s_docs[warp][i0 + 1] : -1,
                         i0 + 2 < n_in ? s_docs[warp][i0 + 2] : -1, i0 + 3 < n_in ? s_docs[warp][i0 + 3] : -1);
        freqs = make_int4(i0 < n_in ? s_freqs[warp][i0] : 1, i0 + 1 < n_in ? s_freqs[warp][i0 + 1] : 1,
                          i0 + 2 < n_in ? s_freqs[warp][i0 + 2] : 1, i0 + 3 < n_in ? s_freqs[warp][i0 + 3] : 1);
    }
    const int d[4] = {docs.x, docs.y, docs.z, docs.w};
    const int f[4] = {freqs.x, freqs.y, freqs.z, freqs.w};
    if (BITMAP) {
        uint32_t* bits = static_cast<uint32_t*>(job.dst);
#pragma unroll
        for (int q = 0; q < 4; q++)
            if (d[q] >= 0 && d[q] < seg.max_doc) atomicOr(bits + (d[q] >> 5), 1u << (d[q] & 31));
        return;
    }
    const float* cache = caches + (size_t)job.cache_id * 256;
    if (MODE == 2 || MODE == 3) {
        uint32_t* bits = static_cast<uint32_t*>(job.dst);
        const float tau1 = job.weight, tau2 = __uint_as_float(job.pad);
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (d[q] < 0 || d[q] >= seg.max_doc) continue;
            const float nrm = seg.norms ? __ldg(cache + __ldg(seg.norms + d[q])) : k1;
            const float fq = (float)f[q];
            const float t = __fdiv_ru(fq, __fadd_rd(fq, nrm));  // >= the true factor
            if (MODE == 3) {
                const int bin = t > 0.0f ? min(255, (int)ceilf(t * 256.0f) - 1) : 0;  // bin i <=> factor <= (i+1)/256; NaN -> 0..255 clamp
                atomicAdd(hist + (size_t)jl * 256 + (t <= 1.0f ? bin : 255), 1u);
            } else {
                if (!(t <= tau1)) atomicOr(bits + (d[q] >> 5), 1u << (d[q] & 31));  // NaN counts as high
                if (!(t <= tau2)) atomicOr(bits + plane_stride + (d[q] >> 5), 1u << (d[q] & 31));
            }
        }
        return;
    }
    float* col = static_cast<float*>(job.dst);
    const float w1 = __fmul_rn(job.weight, __fadd_rn(k1, 1.0f));  // as k_eval_or computes it
    if (MODE == 4) {  // scored list: the block's 128 docids, then its 128 scores (entries past the end: kNoMoreDocs, 0)
        uint32_t dv[4], sv[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const bool ok = d[q] >= 0 && d[q] < seg.max_doc;
            const float nrm = seg.norms ? __ldg(cache + __ldg(seg.norms + (ok ? d[q] : 0))) : k1;
            dv[q] = ok ? (uint32_t)d[q] : (uint32_t)kNoMoreDocs;
            sv[q] = ok ? __float_as_uint(bm25_score(w1, (float)f[q], nrm)) : 0u;
        }
        uint4* blk = static_cast<uint4*>(job.dst) + (size_t)b * 64;
        blk[lane] = make_uint4(dv[0], dv[1], dv[2], dv[3]);
        blk[32 + lane] = make_uint4(sv[0], sv[1], sv[2], sv[3]);
        return;
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        if (d[q] < 0 || d[q] >= seg.max_doc) continue;
        const float nrm = seg.norms ? __ldg(cache + __ldg(seg.norms + d[q])) : k1;
        col[d[q]] = bm25_score(w1, (float)f[q], nrm);
    }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
void launch_build_columns(cudaStream_t st, const SegDev* segs, const ColumnJob* jobs, uint32_t n_jobs,
                          uint32_t n_units, const float* caches, float k1) {
    if (!n_jobs || !n_units) return;
    k_build_columns<0><<<(n_units + kColWarps - 1) / kColWarps, kColWarps * 32, 0, st>>>(segs, jobs, n_jobs, n_units,
                                                                                         caches, k1, nullptr, 0);
}
void launch_build_lists(cudaStream_t st, const SegDev* segs, const ColumnJob* jobs, uint32_t n_jobs, uint32_t n_units,
                        const float* caches, float k1) {
    if (!n_jobs || !n_units) return;
    k_build_columns<4><<<(n_units + kColWarps - 1) / kColWarps, kColWarps * 32, 0, st>>>(segs, jobs, n_jobs, n_units,
                                                                                         caches, k1, nullptr, 0);
}
// seg: device pointer to ONE SegDev (jobs carry seg = 0)
void launch_build_bitmaps(cudaStream_t st, const SegDev* seg, const ColumnJob* jobs, uint32_t n_jobs,
                          uint32_t n_units) {
    if (!n_jobs || !n_units) return;
    k_build_columns<1><<<(n_units + kColWarps - 1) / kColWarps, kColWarps * 32, 0, st>>>(seg, jobs, n_jobs, n_units,
                                                                                         nullptr, 0.f, nullptr, 0);
}
void launch_build_tf_planes(cudaStream_t st, const SegDev* segs, const ColumnJob* jobs, uint32_t n_jobs,
                            uint32_t n_units, const float* caches, float k1, uint32_t* hist, size_t plane_stride) {
    if (!n_jobs || !n_units) return;
    const uint32_t ctas = (n_units + kColWarps - 1) / kColWarps;
    if (hist) k_build_columns<3><<<ctas, kColWarps * 32, 0, st>>>(segs, jobs, n_jobs, n_units, caches, k1, hist, 0);
    else k_build_columns<2><<<ctas, kColWarps * 32, 0, st>>>(segs, jobs, n_jobs, n_units, caches, k1, nullptr, plane_stride);
}
template <bool LIVE, bool NOT, bool MSM, bool DMAX, bool POS = false>
static void launch_eval_or_t(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, size_t wb,
                             uint32_t kcap) {
    const size_t smem = wb * kOrWarps;
    // per launch, not cached: the attribute is per device and engines may live on several
    cudaFuncSetAttribute(k_eval_or<LIVE, NOT, MSM, DMAX, POS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const uint32_t ctas = (n + kOrWarps - 1) / kOrWarps;
    k_eval_or<LIVE, NOT, MSM, DMAX, POS><<<ctas, kOrThreads, smem, st>>>(p, item_ids, n, (uint32_t)wb, kcap);
}
// has_live: some leaf has deleted docs; has_not: some item of the launch carries a MUST_NOT clause;
// all_pos: every clause score of every item of the launch is > 0 (the planner checked weights and norm caches)
void launch_eval_or(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n,
                    uint32_t max_terms, bool has_live, bool has_not, bool has_msm, bool has_dmax, bool all_pos) {
    if (!n) return;
    const uint32_t kcap = (std::min<uint32_t>(p.k, kMaxK) + 31u) & ~31u;
    size_t wb = sizeof(WarpShared) + (size_t)kcap * sizeof(float) + (size_t)max_terms * kBlock * 8;
    wb = (wb + 15) & ~size_t(15);
    if (has_dmax) {  // a DisjunctionMaxQuery in the batch: per-doc counters + per-doc maxima
        wb += kWw + kWw * sizeof(float);
        wb = (wb + 15) & ~size_t(15);
        launch_eval_or_t<true, true, true, true>(st, p, item_ids, n, wb, kcap);
    } else if (has_msm) {  // min_should_match > 1 somewhere in the batch: the general sum variant
        wb += kWw;  // per-doc clause counters
        wb = (wb + 15) & ~size_t(15);
        launch_eval_or_t<true, true, true, false>(st, p, item_ids, n, wb, kcap);
    } else if (has_live && has_not) launch_eval_or_t<true, true, false, false>(st, p, item_ids, n, wb, kcap);
    else if (has_not) launch_eval_or_t<false, true, false, false>(st, p, item_ids, n, wb, kcap);
    else if (has_live && all_pos) launch_eval_or_t<true, false, false, false, true>(st, p, item_ids, n, wb, kcap);
    else if (all_pos) launch_eval_or_t<false, false, false, false, true>(st, p, item_ids, n, wb, kcap);
    else if (has_live) launch_eval_or_t<true, false, false, false>(st, p, item_ids, n, wb, kcap);
    else launch_eval_or_t<false, false, false, false>(st, p, item_ids, n, wb, kcap);
}
template <bool REQOPT, bool OTHER>
static void launch_eval_and_t(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n) {
    cudaFuncSetAttribute(k_eval_and<REQOPT, OTHER>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)sizeof(AndShared));
    k_eval_and<REQOPT, OTHER><<<n, kEvalThreads, sizeof(AndShared), st>>>(p, item_ids);
}
void launch_eval_and(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, bool req_opt,
                     bool has_other_enc) {
    if (!n) return;
    if (req_opt && has_other_enc) launch_eval_and_t<true, true>(st, p, item_ids, n);
    else if (req_opt) launch_eval_and_t<true, false>(st, p, item_ids, n);
    else if (has_other_enc) launch_eval_and_t<false, true>(st, p, item_ids, n);
    else launch_eval_and_t<false, false>(st, p, item_ids, n);
}
void launch_heap_replay(cudaStream_t st, const ReplayParams& p) {
    if (!p.n_groups) return;
    const size_t smem = (size_t)kReplayWarps * p.k * sizeof(rg_hit);
    // per launch, not cached: the attribute is per device and engines may live on several
    cudaFuncSetAttribute(k_heap_replay, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_heap_replay<<<(p.n_groups + kReplayWarps - 1) / kReplayWarps, kReplayWarps * 32, smem, st>>>(p);
}
void launch_merge_leaf_records(cudaStream_t st, const uint8_t* records, uint32_t n_leaves,
                               uint32_t n_queries, uint32_t k, rg_hit* out_hits,
                               uint32_t* out_counts, unsigned long long* out_total) {
    if (!n_queries) return;
    const size_t smem = (size_t)kReplayWarps * k * sizeof(rg_hit);
    // per launch, not cached: the attribute is per device and engines may live on several
    cudaFuncSetAttribute(k_merge_leaf_records, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_merge_leaf_records<<<(n_queries + kReplayWarps - 1) / kReplayWarps, kReplayWarps * 32, smem, st>>>(
        records, n_leaves, n_queries, k, out_hits, out_counts, out_total);
}

}  // namespace rg
