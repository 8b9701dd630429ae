// eval_dpq.cu — k_eval_dpq: disjunctions with 10 or more clauses in a leaf.
//
// From ten sub-scorers on, DisjunctionSumScorer / DisjunctionMaxScorer keep them in a DisiPriorityQueue instead of
// the SimpleQueue (search/scorer/disjunction_scorer.rs:41-45,118-139): a binary min-heap on the sub-scorers' current
// docids (util/disi.rs:135-336).  score_sum / score_max add the scores of the sub-scorers that sit on the top docid
// in the order of top_list() (:190-231), a walk over the heap ARRAY — and the array's layout is a function of the
// whole history of next() calls.  The f32 sum therefore cannot be reproduced by any docid-parallel evaluation:
// this kernel replays the queue literally.  One warp per (query, leaf); every clause is a cached block stream
// (decoded / scored 128 postings at a time by the whole warp, eval_shared.cuh), lane 0 runs up_heap / down_heap /
// top_list exactly as the reference does and hands the (doc, score) pairs it produces, 32 at a time, to the
// warp-wide candidate filter (theta) + emitter the other disjunction kernels use.  It is a sequential algorithm by
// definition — tens of nanoseconds per posting — and exists for completeness, not speed; batches hide it.
#include "eval_shared.cuh"

namespace rg {

constexpr int kDpqWarps = 2;
constexpr int kDpqOut = 32;

struct alignas(16) DpqWarpShared {  // followed by topk[kcap], then cdocs[T][128], cscores[T][128]
    WTerm term[kDpqMaxTerms];
    int32_t cur[kDpqMaxTerms];       // current docid of sub-scorer t (-1 before the first next())
    uint8_t heap[kDpqMaxTerms];      // DisiPriorityQueue::heap (indices of sub-scorers)
    uint8_t list[kDpqMaxTerms];      // top_list(), head first
    rg_hit out[kDpqOut];             // produced docs waiting for the emitter
    float newc[kNewcW];
};

struct DpqState {   // lane 0
    uint32_t size;     // heap size = number of sub-scorers
    int32_t doc;       // docid the running next() started from
    bool in_next;      // interrupted inside next() by a refill
    uint32_t nout;
};

__device__ __forceinline__ void dpq_update_top(DpqWarpShared& sh, uint32_t size) {  // down_heap(size), disi.rs:311-336
    uint32_t i = 0;
    const uint8_t node = sh.heap[0];
    const int32_t node_doc = sh.cur[node];
    uint32_t j = 1;
    if (j < size) {
        uint32_t k = j + 1;
        if (k < size && sh.cur[sh.heap[k]] < sh.cur[sh.heap[j]]) j = k;
        if (sh.cur[sh.heap[j]] < node_doc) {
            for (;;) {
                sh.heap[i] = sh.heap[j];
                i = j;
                j = ((i + 1) << 1) - 1;
                k = j + 1;
                if (k < size && sh.cur[sh.heap[k]] < sh.cur[sh.heap[j]]) j = k;
                if (j >= size || sh.cur[sh.heap[j]] >= node_doc) break;
            }
            sh.heap[i] = node;
        }
    }
}

// top_list (disi.rs:190-231) without recursion: the reference prepends a node when it is visited, visits the left
// subtree, then the right one.  Returns the list length; sh.list[0] is the head (first score added).
__device__ __forceinline__ uint32_t dpq_top_list(DpqWarpShared& sh, uint32_t size) {
    // collected in visiting order into the tail of sh.list, i.e. written back to front = prepending
    uint32_t n = 0;
    const int32_t doc = sh.cur[sh.heap[0]];
    auto prepend = [&](uint8_t w) {
        n++;
        sh.list[kDpqMaxTerms - n] = w;
    };
    prepend(sh.heap[0]);
    if (size >= 3) {
        // explicit stack of heap positions still to visit (depth <= log2(32) + 1 pairs)
        uint8_t stack[12];
        int sp = 0;
        stack[sp++] = 2;
        stack[sp++] = 1;
        while (sp) {
            const uint32_t i = stack[--sp];
            const uint8_t w = sh.heap[i];
            if (sh.cur[w] != doc) continue;
            prepend(w);
            const uint32_t left = ((i + 1) << 1) - 1, right = left + 1;
            if (right < size) {
                stack[sp++] = (uint8_t)right;  // visited after the left subtree
                stack[sp++] = (uint8_t)left;
            } else if (left < size && sh.cur[sh.heap[left]] == doc) {
                prepend(sh.heap[left]);
            }
        }
    } else if (size == 2 && sh.cur[sh.heap[1]] == doc) {
        prepend(sh.heap[1]);
    }
    for (uint32_t i = 0; i < n; i++) sh.list[i] = sh.list[kDpqMaxTerms - n + i];
    return n;
}

// DEEP: k > kMaxK — theta from a score histogram in the topk slot (kcap = kDeepBuckets, see deep_publish)
template <bool LIVE, bool DEEP = false>
__global__ void __launch_bounds__(kDpqWarps * 32)
k_eval_dpq(EvalParams p, const uint32_t* __restrict__ item_ids, uint32_t n_ids, uint32_t warp_bytes, uint32_t kcap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const uint32_t wid = blockIdx.x * kDpqWarps + warp;
    if (wid >= n_ids) return;
    unsigned char* sbase = smem_raw + (size_t)warp * warp_bytes;
    DpqWarpShared& sh = *reinterpret_cast<DpqWarpShared*>(sbase);
    float* topk = reinterpret_cast<float*>(sbase + sizeof(DpqWarpShared));
    int32_t* cdocs = reinterpret_cast<int32_t*>(topk + kcap);
    const uint32_t item_idx = item_ids[wid];
    const WorkItem it = p.items[item_idx];
    const SegDev seg = p.segs[it.seg];
    const int T = it.n_terms;
    float* cscores = reinterpret_cast<float*>(cdocs + T * kBlock);
    const bool dmax_item = (it.type & kItemDismax) != 0;
    const float tie = dmax_item ? p.clauses[it.clause_begin + T].weight : 0.0f;
    const int lo = 0, hi = seg.max_doc;

    if (lane < T) {
        const ItemClause c = p.clauses[it.clause_begin + lane];
        const TermDev td = seg.terms[c.term_id];
        WTerm& tc = sh.term[lane];
        tc.is_col = 0;
        tc.pre = nullptr;
        tc.blk_last = seg.blk_last + td.blk_begin;
        tc.blk_desc = seg.blk_desc + td.blk_begin;
        tc.cache = p.caches + (size_t)c.cache_id * 256;
        tc.nb = td.n_blocks;
        tc.cur = 0;
        tc.n = 0;
        tc.pos = 0;
        tc.term_id = c.term_id;
        tc.w1 = __fmul_rn(c.weight, __fadd_rn(p.k1, 1.0f));
        tc.is_not = 0;
        sh.cur[lane] = -1;            // every sub-scorer starts before its first doc
        sh.heap[lane] = (uint8_t)lane;  // DisiPriorityQueue::new: pushes in child order; all docids equal -> no swap
    }
    __syncwarp();
    MsmCtx mc_unused{nullptr, 1u, nullptr};
    uint32_t hot_unused = 0, mm_unused = 0;
    // first block of every clause; pos = -1 relative to the first cached entry is modelled by cur[t] = -1 and a
    // cursor that points AT the first entry (the first next() consumes it without advancing)
    for (int t = 0; t < T; t++) {
        stream_refill<false, false, false, false>(seg, p, sh.term[t], cdocs + t * kBlock, cscores + t * kBlock, lo, hi, lane, 0,
                                                  -2147483647 - 1, reinterpret_cast<uint32_t*>(cdocs), hot_unused, mm_unused,
                                                  INFINITY, mc_unused);
    }

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
    const uint2 dmap = DEEP ? p.deep_map[it.query] : uint2{0u, 0u};
    if (DEEP) em.theta_local = deep_inherit(reinterpret_cast<uint32_t*>(topk), p, item_idx, it.chain_pos, dmap, lane);
    else wtheta_inherit(em, p, item_idx, it.chain_pos, kcap, lane);
    const bool lb_ok = (uint32_t)lane < it.chain_pos;
    const uint32_t* theta_lb = p.item_theta + item_idx - 1 - (lb_ok ? lane : 0);

    DpqState st{(uint32_t)T, -1, false, 0u};
    uint32_t matches = 0;  // lane 0
    uint32_t first_pending = 0xffffffffu;  // lane 0: bit t set = clause t has not consumed its first cached entry yet
    enum : uint32_t { kDone = 0, kRefill = 1, kFlush = 2 };
    for (;;) {
        uint32_t cmd = kDone;
        if (lane == 0) {
            for (;;) {
                // ---- next(): SubScorers::approximate_next, DPQ arm (disjunction_scorer.rs:334-347)
                if (!st.in_next) st.doc = sh.cur[sh.heap[0]];
                bool need_refill = false;
                uint32_t rt = 0;
                for (;;) {
                    if (!st.in_next) {
                        const uint32_t t = sh.heap[0];
                        WTerm& tc = sh.term[t];
                        if ((first_pending >> t) & 1u) first_pending &= ~(1u << t);  // the cursor already sits on the first entry
                        else tc.pos++;
                        if (tc.pos < tc.n) {
                            sh.cur[t] = cdocs[t * kBlock + tc.pos];
                        } else if (tc.cur <= tc.nb) {  // cached block used up: the warp decodes the next one
                            need_refill = true;
                            rt = t;
                            st.in_next = true;
                            break;
                        } else {
                            sh.cur[t] = kNoMoreDocs;
                        }
                    }
                    st.in_next = false;  // (after a refill the caller has set cur[t])
                    dpq_update_top(sh, st.size);
                    if (sh.cur[sh.heap[0]] != st.doc) break;
                }
                if (need_refill) {
                    cmd = kRefill | (rt << 2);
                    break;
                }
                const int32_t d = sh.cur[sh.heap[0]];
                if (d == kNoMoreDocs) {
                    cmd = kDone;
                    break;
                }
                // ---- score(): score_sum / score_max over top_list() (disjunction_scorer.rs:226-240,264-286)
                const uint32_t n = dpq_top_list(sh, st.size);
                float sum = 0.0f, mx = -INFINITY;
                for (uint32_t i = 0; i < n; i++) {
                    const uint32_t t = sh.list[i];
                    const float s = cscores[t * kBlock + sh.term[t].pos];
                    sum = __fadd_rn(sum, s);
                    if (s > mx) mx = s;
                }
                const float score = dmax_item ? __fadd_rn(mx, __fmul_rn(__fsub_rn(sum, mx), tie)) : sum;
                if (!LIVE || is_live(seg, d)) {  // BulkScorer: only live docs are collected
                    matches++;
                    sh.out[st.nout++] = rg_hit{d, score};
                    if (st.nout == kDpqOut) {
                        cmd = kFlush;
                        break;
                    }
                }
            }
        }
        cmd = __shfl_sync(0xffffffffu, cmd, 0);
        if ((cmd & 3u) == kRefill) {
            const int t = (int)(cmd >> 2);
            const bool ok = stream_refill<false, false, false, false>(seg, p, sh.term[t], cdocs + t * kBlock, cscores + t * kBlock,
                                                                      lo, hi, lane, 0, -2147483647 - 1,
                                                                      reinterpret_cast<uint32_t*>(cdocs), hot_unused, mm_unused,
                                                                      INFINITY, mc_unused);
            if (lane == 0) sh.cur[t] = ok ? cdocs[t * kBlock + sh.term[t].pos] : kNoMoreDocs;
            __syncwarp();
            continue;
        }
        // ---- hand the produced docs to the collector side: theta filter, candidate run, running top-k
        const uint32_t nout = __shfl_sync(0xffffffffu, st.nout, 0);
        __syncwarp();
        if (nout) {
            uint32_t inherited = 0;
            if (it.chain_pos) {
                inherited = lb_ok ? ld_volatile_u32(theta_lb) : 0u;
                inherited = __reduce_max_sync(0xffffffffu, inherited);
            }
            if (inherited > em.theta_in) {
                em.theta_in = inherited;
                if (lane == 0) atomicMax(p.item_theta + item_idx, inherited);
            }
            float te = em.theta_local;
            if (em.theta_in > kOrderedNegInf) te = fmaxf(te, ordered_to_float(em.theta_in));
            const bool open = te == -INFINITY;
            const rg_hit h = (uint32_t)lane < nout ? sh.out[lane] : rg_hit{0, 0.f};
            const bool cand = (uint32_t)lane < nout && (open || h.score > te);
            const uint32_t cm = __ballot_sync(0xffffffffu, cand);
            uint32_t newc_n = 0;
            if (cm && !em.overflow) {
                const uint32_t cn = __popc(cm);
                CandRun* hdr = reinterpret_cast<CandRun*>(p.cand_arena);
                if (em.run_slot == kNone || em.run_cnt + cn > em.run_cap) {
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
                    } else {
                        em.run_slot = slot;
                        em.run_cap = cap;
                        em.run_cnt = 0;
                    }
                }
                if (!em.overflow) {
                    if (cand) {
                        const uint32_t r = __popc(cm & ((1u << lane) - 1u));
                        p.cand_arena[em.run_slot + 1 + em.run_cnt + r] = rg_hit{h.doc + seg.doc_base, h.score};
                        if (DEEP) deep_count(reinterpret_cast<uint32_t*>(topk), dmap, h.score);
                        else sh.newc[r] = h.score;
                    }
                    em.run_cnt += cn;
                    newc_n = cn;
                    if (lane == 0) hdr[em.run_slot] = CandRun{kNone, em.run_cnt};
                }
            }
            __syncwarp();
            if (DEEP) wtheta_update_deep(em, p, item_idx, dmap, lane, newc_n);
            else wtheta_update(em, p, item_idx, kcap, lane, sh.newc, newc_n);
            __syncwarp();
            if (lane == 0) st.nout = 0;
        }
        if ((cmd & 3u) == kDone) break;
    }
    if (lane == 0) p.item_matches[item_idx] = matches;
}

template <bool LIVE, bool DEEP = false>
static void launch_eval_dpq_t(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, size_t wb,
                              uint32_t kcap) {
    const size_t smem = wb * kDpqWarps;
    cudaFuncSetAttribute(k_eval_dpq<LIVE, DEEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_eval_dpq<LIVE, DEEP><<<(n + kDpqWarps - 1) / kDpqWarps, kDpqWarps * 32, smem, st>>>(p, item_ids, n, (uint32_t)wb, kcap);
}

void launch_eval_dpq(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, uint32_t max_terms,
                     bool has_live) {
    if (!n) return;
    const bool deep = p.k > (uint32_t)kMaxK;
    const uint32_t kcap = deep ? (uint32_t)kDeepBuckets : (std::min<uint32_t>(p.k, kMaxK) + 31u) & ~31u;
    size_t wb = sizeof(DpqWarpShared) + (size_t)kcap * sizeof(float) + (size_t)max_terms * kBlock * 8;
    wb = (wb + 15) & ~size_t(15);
    if (deep && has_live) launch_eval_dpq_t<true, true>(st, p, item_ids, n, wb, kcap);
    else if (deep) launch_eval_dpq_t<false, true>(st, p, item_ids, n, wb, kcap);
    else if (has_live) launch_eval_dpq_t<true>(st, p, item_ids, n, wb, kcap);
    else launch_eval_dpq_t<false>(st, p, item_ids, n, wb, kcap);
}

}  // namespace rg
