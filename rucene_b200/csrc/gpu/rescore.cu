// rescore.cu — QueryRescorer::rescore (search/scorer/rescorer.rs:130-607) over a batch's TopDocs rows in HBM.
//
// k_rescore: one warp per query.  The first min(count, window_size) hits of the row are sorted by docid
// (query_rescore :301-307), cut into leaf runs, and every clause of the rescoring query's per-leaf scorer tree
// (RescoreLeaf, planned by search.cu from the same per-(query, leaf) resolution as the first pass) walks forward
// over the ascending targets of its run: gallop through the skip table to the block that holds the target,
// decode that block once, and look up every later target that falls in it (iterative_rescore :236-296, the
// scorer's advance() per target).  The clause results are folded in the reference scorer's f32 order, combined
// with the first-pass score (combine_score :349-367), the window is sorted by (score desc, docid asc)
// (ScoreDocHit's Ord, sort_field/collapse_top_docs.rs:180-201) and written back; every hit after the window is
// scaled by query_weight (combine_docs :375-417).
//
// k_rescore<true> is the same walk for rescoring queries with pure-SHOULD groups (kClauseReqGroup / kClauseOptGroup,
// members contiguous and in member order, kClauseGroupLast on the last) and point ranges (kClauseRange: term_id
// indexes RescoreParams::ranges per (leaf, range)).  A group's members add into a per-target DisjunctionSumScorer sum
// (from 0.0f); after its last member the sum folds into the group's side as one value.  A required range counts as one
// required clause that adds +0.0f; a MUST_NOT range excludes.  k_rescore<false> compiles none of that code.
#include "eval_shared.cuh"

namespace rg {

namespace {

constexpr uint32_t kRsReqAny = 1u;   // some scoring clause of the required side has the target
constexpr uint32_t kRsOptAny = 2u;   // some optional (ReqOptScorer) clause has it
constexpr uint32_t kRsExcl = 4u;     // some MUST_NOT clause has it (ReqNotScorer)
constexpr uint32_t kRsCountSh = 8u;  // bits [8, 16): required clauses that have it (conjunctions)
constexpr uint32_t kRsGroupAny = 1u << 16;  // some member of the group being walked has it (k_rescore<true>)
constexpr uint32_t kRsMatched = 0x80000000u;  // the leaf's scorer matched the target
constexpr uint32_t kRsOptThreshold = 100;     // ReqOptScorer: scores_num above which low scores skip the optional side

// ordered key of a combined score for "score descending": -0.0 and +0.0 are equal (partial_cmp)
__device__ __forceinline__ uint32_t desc_key(float s) {
    if (s == 0.0f) s = 0.0f;
    return ~float_to_ordered(s);
}

// warp bitonic sort of n (a power of two >= 32) 64-bit keys in shared memory, ascending
__device__ void warp_sort(unsigned long long* a, uint32_t n, int lane) {
    for (uint32_t size = 2; size <= n; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = lane; t < n / 2; t += 32) {
                const uint32_t i = 2 * t - (t & (stride - 1));
                const uint32_t j = i + stride;
                const bool up = (i & size) == 0;
                const unsigned long long x = a[i], y = a[j];
                if ((x > y) == up) {
                    a[i] = y;
                    a[j] = x;
                }
            }
            __syncwarp();
        }
    }
}

// RescoreMode::combine (rescorer.rs:96-115), f32
__device__ __forceinline__ float combine(uint32_t mode, float a, float b) {
    switch (mode) {
        case RG_RESCORE_AVG: return __fdiv_rn(__fadd_rn(a, b), 2.0f);
        case RG_RESCORE_MAX: return fmaxf(a, b);
        case RG_RESCORE_MIN: return fminf(a, b);
        case RG_RESCORE_TOTAL: return __fadd_rn(a, b);
        default: return __fmul_rn(a, b);
    }
}

// One clause over the targets keys[b, e) (ascending global docids in the high words) of one leaf: the
// scorer's advance(target) for each, as a forward walk.  Updates acc / acc2 / st of the targets it finds.  NESTED: a
// group member adds into the target's group sum (the ncap floats after bfreqs) and flags it kRsGroupAny.
template <bool NESTED>
__device__ void probe_clause(const RescoreParams& p, const SegDev& seg, const ItemClause c, uint32_t ci,
                             uint32_t kind, const unsigned long long* keys, uint32_t b, uint32_t e, float* acc,
                             float* acc2, uint32_t* st, int32_t* bdocs, int32_t* bfreqs, int lane) {
    const TermDev td = seg.terms[c.term_id];
    const int32_t* bl = seg.blk_last + td.blk_begin;
    const BlockDesc* bdesc = seg.blk_desc + td.blk_begin;
    const uint32_t nb = td.n_blocks;
    const float w1 = __fmul_rn(c.weight, __fadd_rn(p.k1, 1.0f));
    const float* cache = p.caches + (size_t)c.cache_id * 256;
    const uint32_t role = c.flags & (kClauseNot | kClauseOpt);  // 0 required / scoring, kClauseNot, kClauseOpt
    const int base = seg.doc_base;
    uint32_t pos = b, hint = 0;
    while (pos < e) {
        const int d = (int)(keys[pos] >> 32) - base;
        const uint32_t bi = lower_bound_gallop(bl, hint, nb, d);
        const bool tail = bi == nb;
        if (tail && !(td.tail_n > 0 && (nb == 0 || d > td.tail_base))) break;  // past the last posting
        int n_in;
        int last;
        if (!tail) {
            const BlockDesc bd = bdesc[bi];
            const int prev = bi == 0 ? 0 : __ldg(bl + bi - 1);
            const uint4* part = seg.arena + bd.off16;
            if ((bd.bits >> 24) == 0) {
                const int4 dl = unpack4(part, (int)(bd.bits & 0xff), lane, seg.version, seg.sb_mask);
                reinterpret_cast<int4*>(bdocs)[lane] = deltas_to_docs(dl, prev);
            } else {  // EF / BITSET doc part
                decode_other_docs(part, bd.bits >> 24, bi == 0 ? -1 : prev, bdocs, lane);
            }
            reinterpret_cast<int4*>(bfreqs)[lane] =
                unpack4(part + ((bd.bits >> 16) & 0xff), (int)((bd.bits >> 8) & 0xff), lane, seg.version, seg.sb_mask);
            n_in = kBlock;
            last = __ldg(bl + bi);
        } else {
            if (lane == 0) decode_tail(seg, td, bdocs, bfreqs);
            n_in = (int)td.tail_n;
        }
        __syncwarp();
        if (tail) last = bdocs[n_in - 1];
        // every target that falls in this block, 32 at a time (targets ascend, so the ones in it are a prefix)
        while (pos < e) {
            const uint32_t j = pos + lane;
            const int dj = j < e ? (int)(keys[j] >> 32) - base : kNoMoreDocs;
            const bool in = dj <= last;
            const uint32_t m = __ballot_sync(0xffffffffu, in);
            if (in) {
                int l = 0, h = n_in;
                while (l < h) {
                    const int mid = (l + h) >> 1;
                    if (bdocs[mid] < dj) l = mid + 1;
                    else h = mid;
                }
                if (l < n_in && bdocs[l] == dj) {
                    const float nrm = seg.norms ? __ldg(cache + __ldg(seg.norms + dj)) : p.k1;
                    const float s = bm25_score(w1, (float)bfreqs[l], nrm);
                    if (NESTED && (c.flags & (kClauseReqGroup | kClauseOptGroup))) {
                        float* gsum = reinterpret_cast<float*>(bfreqs + kBlock);
                        gsum[j] = __fadd_rn(gsum[j], s);  // DisjunctionSumScorer from 0.0f, member order
                        st[j] |= kRsGroupAny;
                    } else if (role == kClauseNot) {
                        st[j] |= kRsExcl;
                    } else if (role == kClauseOpt) {
                        acc2[j] = __fadd_rn(acc2[j], s);  // DisjunctionSumScorer from 0.0f, clause order
                        st[j] |= kRsOptAny;
                    } else if (kind == kRsTerm) {
                        acc[j] = s;
                        st[j] |= kRsReqAny;
                    } else if (kind == kRsConj) {  // ConjunctionScorer: lead1 + lead2 + others, cost order
                        acc[j] = ci == 0 ? s : __fadd_rn(acc[j], s);
                        st[j] += 1u << kRsCountSh;
                    } else {  // DisjunctionSumScorer / DisjunctionMaxScorer (sum from 0.0f, max from -inf)
                        acc[j] = __fadd_rn(acc[j], s);
                        if (kind == kRsMax) acc2[j] = fmaxf(acc2[j], s);
                        st[j] |= kRsReqAny;
                    }
                }
            }
            const uint32_t taken = __popc(m);
            pos += taken;
            __syncwarp();
            if (taken < 32) break;
        }
        if (tail) break;
        hint = bi + 1;
    }
    __syncwarp();
}

// PointRangeWeight's scorer over the targets keys[b, e) of one leaf (k_rescore<true>): a target's RangeBlock rules
// out a block wholly outside the range, takes a doc with a value in a block wholly inside it, and sends the rest to
// the doc's keys.  A required range counts as one required clause and adds +0.0f at position ci (a -0.0f sum becomes
// +0.0f, as in the reference); a MUST_NOT range excludes.
__device__ void probe_range(const RangeRef& rr, const SegDev& seg, uint32_t ci, bool excl,
                            const unsigned long long* keys, uint32_t b, uint32_t e, float* acc, uint32_t* st, int lane) {
    for (uint32_t j = b + lane; j < e; j += 32) {
        const int d = (int)(keys[j] >> 32) - seg.doc_base;
        const RangeBlock bk = rr.blocks[d / kBlock];
        if (bk.values == 0 || bk.max < rr.lower || bk.min > rr.upper) continue;
        const bool hit = bk.min >= rr.lower && bk.max <= rr.upper ? __ldg(rr.offsets + d + 1) > __ldg(rr.offsets + d)
                                                                  : range_hit(rr, d);
        if (!hit) continue;
        if (excl) {
            st[j] |= kRsExcl;
        } else {
            acc[j] = ci == 0 ? 0.0f : __fadd_rn(acc[j], 0.0f);
            st[j] += 1u << kRsCountSh;
        }
    }
    __syncwarp();
}

}  // namespace

// named outside the anonymous namespace so that its symbols (profiler traces) are stable across builds.  NESTED: the
// plan has group or range clauses; only nested or range rescoring launches k_rescore<true>
template <bool NESTED>
__global__ void __launch_bounds__(32) k_rescore(RescoreParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t q = blockIdx.x;
    const int lane = lane_id();
    const uint32_t ncap = p.ncap;
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);  // (docid, row index), sorted
    unsigned long long* order = keys + ncap;                                      // (score desc, position)
    float* acc = reinterpret_cast<float*>(order + ncap);
    float* acc2 = acc + ncap;
    uint32_t* st = reinterpret_cast<uint32_t*>(acc2 + ncap);
    int32_t* bdocs = reinterpret_cast<int32_t*>(st + ncap);
    int32_t* bfreqs = bdocs + kBlock;
    float* gsum = reinterpret_cast<float*>(bfreqs + kBlock);  // NESTED: the group sum of each target

    const uint32_t cnt = min(p.counts[q], p.k);
    if (p.totals[q] == 0 || cnt == 0) return;  // nothing changes, not even the tail (rescorer.rs:130-140)
    rg_hit* row = p.hits + (size_t)q * p.k;
    const uint32_t n = min(cnt, p.window);
    for (uint32_t i = n + lane; i < cnt; i += 32) row[i].score = __fmul_rn(row[i].score, p.query_weight);
    if (n == 0) return;

    // ---- the window, stable-sorted by docid (the row index breaks ties between equal docids)
    for (uint32_t i = lane; i < ncap; i += 32)
        keys[i] = i < n ? ((unsigned long long)(uint32_t)row[i].doc << 32 | i) : ~0ull;
    __syncwarp();
    warp_sort(keys, ncap, lane);
    for (uint32_t i = lane; i < n; i += 32) {
        acc[i] = 0.0f;
        acc2[i] = 0.0f;
        st[i] = 0u;
        if (NESTED) gsum[i] = 0.0f;
    }
    __syncwarp();

    // ---- leaf runs: one scorer per leaf, built for the leaf's first target (iterative_rescore :244-260)
    uint32_t b = 0;
    for (uint32_t si = 0; si < p.n_segs && b < n; si++) {
        const SegDev seg = p.segs[si];
        // first target at or above the end of this leaf (keys are sorted on their high word)
        const unsigned long long end_key = (unsigned long long)(uint32_t)(seg.doc_base + seg.max_doc) << 32;
        uint32_t lo = b, hi = n;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (keys[mid] < end_key) lo = mid + 1;
            else hi = mid;
        }
        const uint32_t e = lo;
        // targets below this leaf's doc_base belong to no leaf: they match nothing
        const unsigned long long begin_key = (unsigned long long)(uint32_t)seg.doc_base << 32;
        while (b < e && keys[b] < begin_key) b++;
        if (b == e) continue;
        const RescoreLeaf L = p.leaves[(size_t)q * p.n_segs + si];
        if (L.kind != kRsNone) {
            if (L.kind == kRsMax)
                for (uint32_t i = b + lane; i < e; i += 32) acc2[i] = -INFINITY;
            __syncwarp();
            const uint32_t n_cl = (uint32_t)L.n_req + L.n_opt + L.n_not;
            // NESTED: n_req counts group members one by one; a conjunction needs each required term, range and group
            // once.  g0: the first clause of the group being walked (the group is the first summand when it is 0)
            uint32_t need = L.n_req, g0 = 0;
            if (!NESTED) {
                for (uint32_t ci = 0; ci < n_cl; ci++)
                    probe_clause<false>(p, seg, p.clauses[L.clause_begin + ci], ci, L.kind, keys, b, e, acc, acc2, st,
                                        bdocs, bfreqs, lane);
            } else {
                need = 0;
            }
            for (uint32_t ci = 0; NESTED && ci < n_cl; ci++) {
                const ItemClause c = p.clauses[L.clause_begin + ci];
                if (NESTED && (c.flags & kClauseRange)) {
                    probe_range(p.ranges[c.term_id], seg, ci, (c.flags & kClauseNot) != 0, keys, b, e, acc, st, lane);
                    need += (c.flags & kClauseNot) ? 0u : 1u;
                    g0 = ci + 1;
                    continue;
                }
                probe_clause<true>(p, seg, c, ci, L.kind, keys, b, e, acc, acc2, st, bdocs, bfreqs, lane);
                const uint32_t side = c.flags & (kClauseReqGroup | kClauseOptGroup);
                if (!side) {
                    need += (c.flags & (kClauseNot | kClauseOpt)) ? 0u : 1u;
                    g0 = ci + 1;
                    continue;
                }
                if (!(c.flags & kClauseGroupLast)) continue;
                // the group's DisjunctionSumScorer landed on the targets some member has: a required group is one
                // summand of the conjunction (cost order), an optional one one summand of the optional side (clause
                // order); then its sums start again from 0.0f
                for (uint32_t i = b + lane; i < e; i += 32) {
                    const uint32_t s = st[i];
                    if (s & kRsGroupAny) {
                        const float v = gsum[i];
                        if (side == kClauseReqGroup) {
                            acc[i] = g0 == 0 ? v : __fadd_rn(acc[i], v);
                            st[i] = (s & ~kRsGroupAny) + (1u << kRsCountSh);
                        } else {
                            acc2[i] = __fadd_rn(acc2[i], v);
                            st[i] = (s & ~kRsGroupAny) | kRsOptAny;
                        }
                        gsum[i] = 0.0f;
                    }
                }
                __syncwarp();
                need += side == kClauseReqGroup ? 1u : 0u;
                g0 = ci + 1;
            }
            // the per-target scorer result: matched flag in st bit 31, score in acc
            for (uint32_t i = b + lane; i < e; i += 32) {
                const uint32_t s = st[i];
                bool m;
                float v = acc[i];
                if (L.kind == kRsAll) {
                    m = true;
                    v = 0.0f;
                } else if (L.kind == kRsConj) {
                    m = (s >> kRsCountSh) == need;
                } else {
                    m = (s & kRsReqAny) != 0;
                    if (L.kind == kRsMax) v = __fadd_rn(acc2[i], __fmul_rn(__fsub_rn(v, acc2[i]), L.tie));
                }
                m = m && !(s & kRsExcl);
                acc[i] = v;
                st[i] = s | (m ? kRsMatched : 0u);
            }
            __syncwarp();
            if (L.kind == kRsConj && L.n_opt > 0 && lane == 0) {
                // ReqOptScorer::score (req_opt_scorer.rs:19-65), in docid order over the matched targets
                float sum = 0.0f;
                uint32_t num = 0;
                for (uint32_t i = b; i < e; i++) {
                    if (!(st[i] & kRsMatched)) continue;
                    const float req = acc[i];
                    if (num > kRsOptThreshold && __fmul_rn(2.0f, req) < __fdiv_rn(sum, __uint2float_rn(num)))
                        continue;  // the required score alone, state untouched
                    sum = __fadd_rn(sum, req);
                    num++;
                    if (st[i] & kRsOptAny) acc[i] = __fadd_rn(req, acc2[i]);
                }
            }
            __syncwarp();
        }
        b = e;
    }

    // ---- combine_score, then the window in ScoreDocHit order (score desc, docid asc; stable)
    for (uint32_t i = lane; i < ncap; i += 32) {
        if (i < n) {
            const unsigned long long k = keys[i];
            const float last = __fmul_rn(row[(uint32_t)k].score, p.query_weight);
            const float v = (st[i] & kRsMatched) ? combine(p.mode, last, __fmul_rn(acc[i], p.rescore_weight)) : last;
            acc[i] = v;
            order[i] = (unsigned long long)desc_key(v) << 32 | i;
        } else {
            order[i] = ~0ull;
        }
    }
    __syncwarp();
    warp_sort(order, ncap, lane);
    for (uint32_t j = lane; j < n; j += 32) {
        const uint32_t i = (uint32_t)order[j];
        row[j] = rg_hit{(int32_t)(keys[i] >> 32), acc[i]};
    }
}


size_t rescore_smem_bytes(uint32_t ncap, bool nested) {
    return (size_t)ncap * (8 + 8 + 4 + 4 + 4 + (nested ? 4 : 0)) + 2 * kBlock * sizeof(int32_t);
}

void launch_rescore(cudaStream_t st, const RescoreParams& p, bool nested) {
    if (p.n_queries == 0) return;
    // at most 33.8 KB (ncap 1024, nested): no opt-in above 48 KB needed
    const size_t smem = rescore_smem_bytes(p.ncap, nested);
    if (nested) k_rescore<true><<<p.n_queries, 32, smem, st>>>(p);
    else k_rescore<false><<<p.n_queries, 32, smem, st>>>(p);
}

}  // namespace rg
