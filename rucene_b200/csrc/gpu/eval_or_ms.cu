// eval_or_ms.cu — k_eval_or_ms: pure-SHOULD sum disjunctions (DisjunctionSumScorer, TermScorer) over
// presence bitmaps, score columns and a bit-sliced per-document score bound.  sm_90a, integer/HBM work.
//
// What the reference computes (search/scorer/disjunction_scorer.rs:187-244, bulk_scorer.rs:89-122,
// collector/top_docs.rs:67-95) is, per (query, leaf): total_hits = |union of the clauses' live docs| and the
// TopDocsCollector heap fed with every union doc in docid order, score = clause-order f32 sum.  A doc changes
// the heap only if root.score < score.  With theta = a proven lower bound of the heap root at that point
// (eval_shared.cuh) the evaluation splits into
//   * counting   — needs presence only.  Every term with df >= max_doc/1024 carries a presence bitmap built at
//                  upload, so such a clause costs one 32-bit word per 32 docids: popc(OR of the words);
//   * candidates — only docs whose score can exceed theta.  A clause's contribution is bounded by
//                  ub = nextafter(weight*(k1+1)) (BM25's tf-norm factor is < 1 for norm >= 0).  The bounds are
//                  quantised to q = ceil(ub * 63 / theta) and summed PER DOCUMENT for 32 docids at a time with a
//                  bit-sliced adder over the clauses' bitmap words (6 planes + a sticky carry): a doc whose carry
//                  stays clear has sum(ub of its clauses) <= theta, scores <= theta <= root and can never be
//                  collected into the heap.  The docs with a carry, plus every doc of a clause without a bitmap
//                  (sparse block streams), form the window's set E and get their exact score: clauses are visited
//                  in clause order and add into a per-window accumulator — sparse streams by scatter, score columns
//                  by gathering col[d], block streams that have a bitmap by seeking to the window and scattering
//                  the postings that fall on E.
// Most postings of a long disjunction are therefore never decoded or scored, only counted, and the result is
// still bit-identical to the reference, ties included, because the heap replay sees every doc that could enter.
//
// Work item = (query, leaf, docid range), one WARP each.  The warp walks windows of up to 1024 docids (lane l owns
// presence word l).  While some combination of bitmap clauses can still beat theta the windows are contiguous
// (each costs the word loads + the adder unless E is non-empty); once no combination can, windows exist only at
// the postings of the sparse streams and everything between them is counted in bulk from the bitmaps.  A window
// ends where a sparse stream's cached block ends, so all its sparse postings are in shared memory when E is formed.
#include "eval_shared.cuh"

namespace rg {

// One warp per CTA: work items differ wildly in length (a range where nothing can beat theta is a bulk popcount,
// one that must score is thousands of windows), and a CTA keeps its slot until its slowest warp is done.
constexpr int kMsWarps = 1;
constexpr int kMsThreads = kMsWarps * 32;
constexpr int kMsW = 1024;     // docids per window = 32 lanes x one 32-bit presence word
constexpr int kMsSlots = 64;   // docs of a window that get an exact score (a fuller window is cut short)
constexpr int kMsPlanes = 6;   // bit-sliced bound: theta <-> 2^6 - 1
constexpr uint32_t kMsSat = 1u << kMsPlanes;

enum : int { kKindNone = 0, kKindCol = 1, kKindBStream = 2, kKindSparse = 3 };

struct alignas(16) MsWarpShared {  // followed by topk[kcap] floats, then cdocs[S][128], cscores[S][128]
    float acc[kMsSlots];           // one accumulator per doc of E, in docid order (slot = rank of the doc's bit in E)
    uint32_t ubits[32];            // presence words of the sparse streams in this window
    uint32_t ebits[32];            // E: the docs of this window that get an exact score
    uint32_t epre[32];             // number of E bits in the words before word w
    uint32_t cw[kMaxTerms][32];    // this window's presence words of the bitmap clauses (lane-owned, masked)
    WTerm term[kMaxTerms];         // block-stream clauses (same cursor as k_eval_or)
    const float* col[kMaxTerms];   // score column (leaf-local docid -> BM25 contribution), column clauses
    const uint32_t* bits[kMaxTerms];  // presence bitmap, column clauses and block streams of dense-enough terms
    const uint32_t* hi1[kMaxTerms];   // "tf-norm factor above tau1" plane of the same clauses (null: none)
    const uint32_t* hi2[kMaxTerms];   // "... above tau2" (subset of hi1)
    float newc[kNewcW];
};

// docs of [a, b) present in any bitmap clause (and live): bulk popcount; per-lane partial sum
template <bool LIVE>
__device__ __forceinline__ uint32_t ms_count_range(const MsWarpShared& sh, uint32_t bmask, const SegDev& seg,
                                                   int a, int b, int lane) {
    uint32_t cnt = 0;
    const int w_end = (b + 31) >> 5;
    for (int w = (a >> 5) + lane; w < w_end; w += 32) {
        const int d0 = w << 5;
        uint32_t m = 0xffffffffu;
        if (d0 < a) m &= ~((1u << (a - d0)) - 1u);
        if (d0 + 32 > b) m &= (1u << (b - d0)) - 1u;
        uint32_t u = 0;
        for (uint32_t cm = bmask; cm; cm &= cm - 1) u |= __ldg(sh.bits[__ffs(cm) - 1] + w);
        u &= m;
        if (LIVE && seg.live) u &= reinterpret_cast<const uint32_t*>(seg.live)[w];
        cnt += __popc(u);
    }
    return cnt;
}

// S += q on the docs of mask m (bit-sliced, kMsPlanes planes); a carry out of the top plane is sticky in `over`
__device__ __forceinline__ void ms_add(uint32_t (&S)[kMsPlanes], uint32_t& over, uint32_t m, uint32_t q) {
    uint32_t carry = 0u;
#pragma unroll
    for (int i = 0; i < kMsPlanes; i++) {
        if ((q >> i) & 1u) {  // warp-uniform
            const uint32_t x = S[i] ^ m;
            const uint32_t c2 = (S[i] & m) | (x & carry);
            S[i] = x ^ carry;
            carry = c2;
        } else {
            const uint32_t c2 = S[i] & carry;
            S[i] ^= carry;
            carry = c2;
        }
    }
    over |= carry;
}

// PLANES: the batch uses tf-norm planes (RG_CFG_TFPLANES): three-level bound, two more words per clause and window
// DEEP: k > kMaxK — theta from a score histogram in the topk slot (kcap = kDeepBuckets, see deep_publish)
template <bool LIVE, bool PLANES, bool DEEP = false>
__global__ void __launch_bounds__(kMsThreads, 24)
k_eval_or_ms(EvalParams p, const uint32_t* __restrict__ item_ids, uint32_t n_ids, uint32_t warp_bytes,
             uint32_t kcap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const uint32_t wid = blockIdx.x * kMsWarps + warp;
    if (wid >= n_ids) return;
    unsigned char* sbase = smem_raw + (size_t)warp * warp_bytes;
    MsWarpShared& sh = *reinterpret_cast<MsWarpShared*>(sbase);
    float* topk = reinterpret_cast<float*>(sbase + sizeof(MsWarpShared));
    int32_t* cdocs = reinterpret_cast<int32_t*>(topk + kcap);
    const uint32_t item_idx = item_ids[wid];
    const WorkItem it = p.items[item_idx];
    const SegDev seg = p.segs[it.seg];
    const int T = it.n_terms;
    const int lo = it.lo, hi = it.hi;
    const uint2 dmap = DEEP ? p.deep_map[it.query] : uint2{0u, 0u};

    // ---- clauses: lane t < T owns clause t
    int kind = kKindNone;
    float ub = 0.0f;  // score bound of a bitmap clause (INF: no usable bound)
    float tau1 = 1.0f, tau2 = 1.0f;  // thresholds of the clause's tf-norm planes
    ItemClause c{};
    if (lane < T) {
        c = p.clauses[it.clause_begin + lane];
        kind = (c.flags & kClauseColumn) ? kKindCol : (c.flags & kClauseBitmap) ? kKindBStream : kKindSparse;
    }
    const uint32_t col_mask = __ballot_sync(0xffffffffu, kind == kKindCol);
    const uint32_t bstream_mask = __ballot_sync(0xffffffffu, kind == kKindBStream);
    const uint32_t sparse_mask = __ballot_sync(0xffffffffu, kind == kKindSparse);
    const uint32_t stream_mask = bstream_mask | sparse_mask;
    const uint32_t bmask = col_mask | bstream_mask;  // clauses with a presence bitmap
    float* cscores = reinterpret_cast<float*>(cdocs + __popc(stream_mask) * kBlock);
    const int my_slot = __popc(stream_mask & ((1u << lane) - 1u));  // stream cache slot of clause `lane`
    if (kind == kKindCol) {
        const ColRef r = p.cols[c.term_id];
        sh.col[lane] = r.col;
        sh.bits[lane] = r.bits;
        sh.hi1[lane] = r.hi1;
        sh.hi2[lane] = r.hi2;
        tau1 = r.tau1;
        tau2 = r.tau2;
    } else if (kind != kKindNone) {
        const TermDev td = seg.terms[c.term_id];
        WTerm& tc = sh.term[lane];
        tc.is_col = 0;
        tc.pre = nullptr;
        tc.blk_last = seg.blk_last + td.blk_begin;
        tc.blk_desc = seg.blk_desc + td.blk_begin;
        tc.cache = p.caches + (size_t)c.cache_id * 256;
        tc.nb = td.n_blocks;
        tc.cur = lower_bound_i32(tc.blk_last, 0, td.n_blocks, lo);
        tc.n = 0;
        tc.pos = 0;
        tc.term_id = c.term_id;
        tc.w1 = __fmul_rn(c.weight, __fadd_rn(p.k1, 1.0f));
        tc.is_not = 0;
        sh.col[lane] = nullptr;
        sh.bits[lane] = nullptr;
        sh.hi1[lane] = sh.hi2[lane] = nullptr;
        if (kind == kKindBStream) {
            const ColRef r = p.cols[c.flags >> kClauseRefShift];
            sh.bits[lane] = r.bits;
            sh.hi1[lane] = r.hi1;
            sh.hi2[lane] = r.hi2;
            tau1 = r.tau1;
            tau2 = r.tau2;
        }
    }
    // bounds of a posting by its tf-norm planes: neither bit -> factor <= tau1, only hi1 -> <= tau2, hi2 -> <= 1
    float ub0 = 0.0f, ub1 = 0.0f;
    if ((bmask >> lane) & 1u) {
        const float w1 = __fmul_rn(c.weight, __fadd_rn(p.k1, 1.0f));
        // score = rn(rn(w1*f) / rn(f + norm)) with f >= 1, norm >= 0  =>  score <= nextafter(w1); with a tf-norm factor
        // (rounded up at build time) <= tau:  score <= w1 * tau * (1 + 4 * 2^-24)
        ub = (c.flags & kClauseNoBound) || !(w1 >= 0.0f) || !(w1 < INFINITY) ? INFINITY : __uint_as_float(__float_as_uint(w1) + 1u);
        const bool planes = PLANES && sh.hi1[lane] != nullptr && ub < INFINITY;
        ub0 = planes ? fminf(ub, __fmul_ru(__fmul_ru(w1, tau1), 1.000001f)) : ub;
        ub1 = planes ? fminf(ub, __fmul_ru(__fmul_ru(w1, tau2), 1.000001f)) : ub;
    }
    const uint32_t hmask = !PLANES ? 0u
                                   : __ballot_sync(0xffffffffu, ((bmask >> lane) & 1u) && sh.hi1[lane] != nullptr && ub < INFINITY);
    sh.acc[lane] = 0.0f;
    sh.acc[lane + 32] = 0.0f;
    __syncwarp();

    MsmCtx mc_unused{nullptr, 1u, nullptr};
    uint32_t hot_unused = 0, mm_unused = 0;
    int nd = kNoMoreDocs;  // sparse stream lane t: next cached docid of clause t (kNoMoreDocs = exhausted)
    for (uint32_t m = sparse_mask; m; m &= m - 1) {  // (streams that have a bitmap are decoded on demand)
        const int t = __ffs(m) - 1;
        const int slot = __popc(stream_mask & ((1u << t) - 1u));
        if (stream_refill<false, false, false, false>(seg, p, sh.term[t], cdocs + slot * kBlock, cscores + slot * kBlock, lo,
                                                      hi, lane, 0, -2147483647 - 1, sh.ubits,
                                                      hot_unused, mm_unused, INFINITY, mc_unused)) {
            const int first = cdocs[slot * kBlock + sh.term[t].pos];
            if (lane == t) nd = first;
        }
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
    if (DEEP) em.theta_local = deep_inherit(reinterpret_cast<uint32_t*>(topk), p, item_idx, it.chain_pos, dmap, lane);
    else wtheta_inherit(em, p, item_idx, it.chain_pos, kcap, lane);
    const bool lb_ok = (uint32_t)lane < it.chain_pos;
    const uint32_t* theta_lb = p.item_theta + item_idx - 1 - (lb_ok ? lane : 0);
    uint32_t win_no = 0;
    uint32_t my_matches = 0;
    int pos = lo;  // every docid < pos is counted and, where needed, scored
    // quantised bounds, valid for theta == q_te
    float q_te = NAN;
    uint32_t q = 0;          // lane t: q of clause t (kMsSat: any doc of the clause must be scored)
    uint32_t q0 = 0, q1 = 0; // ... of its postings with neither / only the first tf-norm plane bit (== q without planes)
    bool prune = false;      // a usable theta exists: docs without a carry are dropped
    bool need_scan = bmask != 0;  // some combination of bitmap clauses can still beat theta
    // RG_CFG_STATS event counters (warp-uniform unless noted)
    uint32_t st_win = 0, st_scan = 0, st_open = 0, st_gap = 0, st_post = 0, st_gather = 0 /* per lane */, st_refill = 0,
             st_cand = 0, st_steps = 0, st_cut = 0, st_scored = 0, st_edocs = 0 /* per lane */;

    for (;;) {
        uint32_t inherited = 0;
        if ((win_no++ & 7u) == 0 && it.chain_pos) {
            inherited = lb_ok ? ld_volatile_u32(theta_lb) : 0u;
            inherited = __reduce_max_sync(0xffffffffu, inherited);
        }
        if (inherited > em.theta_in) {
            // hand an inherited bound on at once: an item that finds no candidate of its own never reaches
            // wtheta_update, and its successors look back over 32 items only
            em.theta_in = inherited;
            if (lane == 0) atomicMax(p.item_theta + item_idx, inherited);
        }
        float te = em.theta_local;
        if (em.theta_in > kOrderedNegInf) te = fmaxf(te, ordered_to_float(em.theta_in));
        const bool open = te == -INFINITY;
        if (!(te == q_te)) {  // theta moved: requantise the clause bounds
            q_te = te;
            prune = !open && te > 0.0f;
            if (prune) {
                // sum(ub) <= theta * (1 - 2^-20) also covers the rounding of the reference's round-to-nearest
                // clause-order sum of up to 9 scores; everything rounds towards "keep the doc"
                const float scale = __fdiv_ru((float)(kMsSat - 1u), __fmul_rd(te, 0.99999904632568359375f));
                const float x = __fmul_ru(ub, scale);
                q = ((bmask >> lane) & 1u) ? (x < (float)kMsSat ? (uint32_t)ceilf(x) : kMsSat) : 0u;  // NaN -> kMsSat
                if (((bmask >> lane) & 1u) && q == 0u) q = 1u;
                const float x1 = __fmul_ru(ub1, scale), x0 = __fmul_ru(ub0, scale);
                q1 = ((hmask >> lane) & 1u) ? min(q, max(1u, x1 < (float)kMsSat ? (uint32_t)ceilf(x1) : kMsSat)) : q;
                q0 = ((hmask >> lane) & 1u) ? min(q1, max(1u, x0 < (float)kMsSat ? (uint32_t)ceilf(x0) : kMsSat)) : q;
                need_scan = __reduce_add_sync(0xffffffffu, q) >= kMsSat;
            } else {
                q = ((bmask >> lane) & 1u) ? kMsSat : 0u;
                q0 = q1 = q;
                need_scan = bmask != 0;
            }
        }
        // ---- next window: here if bitmap clauses can still matter, else at the next sparse posting
        int w0 = need_scan ? pos : __reduce_min_sync(0xffffffffu, kind == kKindSparse ? nd : kNoMoreDocs);
        if (w0 >= hi) {  // nothing left that could be scored: the rest of the range is only counted
            if (bmask && pos < hi) my_matches += ms_count_range<LIVE>(sh, bmask, seg, pos, hi, lane);
            st_gap += (uint32_t)(hi - pos);
            break;
        }
        if (bmask && w0 > pos) my_matches += ms_count_range<LIVE>(sh, bmask, seg, pos, w0, lane);
        st_gap += (uint32_t)(w0 - pos);
        st_win++;
        st_scan += need_scan;
        st_open += open;
        const int win0 = w0;
        const int base = win0 & ~31;
        int win1 = min(hi, base + kMsW);
        {   // a sparse stream whose cached block ends inside the window (and that has more blocks) ends the window there
            int trunc = 0x7fffffff;
            if (kind == kKindSparse) {
                const WTerm& tc = sh.term[lane];
                if (tc.pos < tc.n && tc.cur <= tc.nb) trunc = cdocs[my_slot * kBlock + tc.n - 1] + 1;
            }
            const int t_all = __reduce_min_sync(0xffffffffu, trunc);
            st_cut += t_all < win1;
            win1 = min(win1, t_all);
        }
        // docs of [win0, win1) inside this lane's word
        uint32_t lmask;
        {
            const int wlo = max(win0 - (base + 32 * lane), 0), whi = min(win1 - (base + 32 * lane), 32);
            lmask = whi <= wlo ? 0u : ((whi >= 32 ? 0xffffffffu : ((1u << whi) - 1u)) & ~((1u << wlo) - 1u));
        }
        // ---- 1. presence of the sparse streams (their postings of this window are all cached)
        const uint32_t act = __ballot_sync(0xffffffffu, kind == kKindSparse && nd < win1);
        uint32_t E = 0;
        if (act) {
            sh.ubits[lane] = 0u;
            __syncwarp();
            for (uint32_t m = act; m; m &= m - 1) {
                const int t = __ffs(m) - 1;
                const int slot = __popc(stream_mask & ((1u << t) - 1u));
                const WTerm& tc = sh.term[t];
                const int32_t* cd = cdocs + slot * kBlock;
                const uint32_t n = tc.n;
                for (uint32_t i = tc.pos + lane;; i += 32) {
                    const int d = i < n ? cd[i] : kNoMoreDocs;
                    const bool in_win = d < win1;
                    if (in_win) atomicOr(&sh.ubits[(d - base) >> 5], 1u << ((d - base) & 31));
                    if (!__all_sync(0xffffffffu, in_win)) break;
                }
            }
            __syncwarp();
            E = sh.ubits[lane];
        }
        // ---- 2. bitmap words: U = docs that count; bit-sliced sum of the quantised bounds -> carry = may beat theta
        uint32_t U = E;
        const int wi = (base >> 5) + lane;
        {
            // all words first (independent loads in flight together), then the arithmetic
            uint32_t wv[kMaxTerms], hv1[PLANES ? kMaxTerms : 1], hv2[PLANES ? kMaxTerms : 1];
#pragma unroll
            for (int t = 0; t < kMaxTerms; t++) {
                wv[t] = (((bmask >> t) & 1u) && lmask) ? (__ldg(sh.bits[t] + wi) & lmask) : 0u;
                if (PLANES) {
                    const bool pl = ((hmask >> t) & 1u) && lmask && need_scan;
                    hv1[t] = pl ? __ldg(sh.hi1[t] + wi) : 0xffffffffu;
                    hv2[t] = pl ? __ldg(sh.hi2[t] + wi) : 0xffffffffu;
                }
            }
            // the next window's line of every bitmap towards L1 while this one is processed
            if (((bmask >> lane) & 1u) && base + kMsW < hi)
                asm volatile("prefetch.global.L1 [%0];" ::"l"(sh.bits[lane] + (base >> 5) + 32));
            uint32_t S[kMsPlanes];
#pragma unroll
            for (int i = 0; i < kMsPlanes; i++) S[i] = 0u;
            uint32_t over = 0u;
#pragma unroll
            for (int t = 0; t < kMaxTerms; t++) {
                if (!((bmask >> t) & 1u)) continue;  // warp-uniform
                const uint32_t w = wv[t];
                sh.cw[t][lane] = w;
                U |= w;
                const uint32_t qt = __shfl_sync(0xffffffffu, q, t);
                const uint32_t qa = __shfl_sync(0xffffffffu, q0, t);
                const uint32_t qb = __shfl_sync(0xffffffffu, q1, t);
                // every posting adds q0, those on the first tf-norm plane q1 - q0 more, those on the second the rest of q;
                // a level whose bound alone beats theta (q >= kMsSat; also: no theta yet / no usable bound) puts its
                // docs into E directly
                if (qa >= kMsSat) {
                    over |= w;
                } else if (need_scan) {
                    ms_add(S, over, w, qa);
                    if (PLANES) {
                        const uint32_t w1 = w & hv1[t];
                        if (qb >= kMsSat) {
                            over |= w1;
                        } else {
                            if (qb != qa) ms_add(S, over, w1, qb - qa);
                            const uint32_t w2 = w & hv2[t];
                            if (qt >= kMsSat) over |= w2;
                            else if (qt != qb) ms_add(S, over, w2, qt - qb);
                        }
                    }
                }
            }
            E |= over;
        }
        // at most kMsSlots docs are scored per window: a fuller window ends at the word where the count is reached
        uint32_t epre = 0, n_e = 0;
        const bool any_e = __any_sync(0xffffffffu, E != 0u);
        if (any_e) {
            uint32_t incl = __popc(E);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += x;
            }
            const uint32_t cutm = __ballot_sync(0xffffffffu, incl > (uint32_t)kMsSlots);
            if (cutm) {  // lanes >= cut leave the window (cut >= 2: a word holds 32 docs)
                const int cut = __ffs(cutm) - 1;
                win1 = base + 32 * cut;
                if (lane >= cut) {
                    E = 0u;
                    U = 0u;
                    lmask = 0u;
                    incl = 0u;
                }
                st_cut++;
            }
            epre = incl - __popc(E);
            n_e = __reduce_max_sync(0xffffffffu, incl);
        }
        uint32_t lw = 0xffffffffu;
        if (LIVE && seg.live) lw = lmask ? reinterpret_cast<const uint32_t*>(seg.live)[wi] : 0u;
        my_matches += __popc(U & lw);
        uint32_t hot = 0;
        if (any_e) {
            st_scored++;
            st_edocs += __popc(E);
            sh.ebits[lane] = E;
            sh.epre[lane] = epre;
            __syncwarp();
            // the column cells this window will read, towards L1 now: the clause-ordered pass below would otherwise
            // pay one DRAM round trip per column clause, one after the other
            for (uint32_t m = col_mask; m; m &= m - 1) {
                const int t = __ffs(m) - 1;
                uint32_t w = sh.cw[t][lane] & E;
                const float* col = sh.col[t] + base + 32 * lane;
                while (w) {
                    const int b = __ffs(w) - 1;
                    w &= w - 1;
                    asm volatile("prefetch.global.L1 [%0];" ::"l"(col + b));
                }
            }
            // ---- 3. exact scores of the docs in E: clauses in clause order (DisjunctionSumScorer::score_sum)
            for (int t = 0; t < T; t++) {
                const int kt = __shfl_sync(0xffffffffu, kind, t);
                if (kt == kKindSparse) {
                    if (!((act >> t) & 1u)) continue;
                    const int slot = __popc(stream_mask & ((1u << t) - 1u));
                    WTerm& tc = sh.term[t];
                    const int32_t* cd = cdocs + slot * kBlock;
                    const float* cs = cscores + slot * kBlock;
                    uint32_t cpos = tc.pos;
                    const uint32_t n = tc.n;
                    for (;;) {
                        const uint32_t i = cpos + lane;
                        const int d = i < n ? cd[i] : kNoMoreDocs;
                        const bool in_win = d < win1;
                        const uint32_t cnt = __popc(__ballot_sync(0xffffffffu, in_win));  // sorted: a prefix
                        if (in_win) {
                            const int idx = d - base;
                            const uint32_t slot = sh.epre[idx >> 5] + __popc(sh.ebits[idx >> 5] & ((1u << (idx & 31)) - 1u));
                            const float sum = __fadd_rn(sh.acc[slot], cs[i]);
                            sh.acc[slot] = sum;
                            if (sum > te) hot |= 1u << (idx >> 5);
                        }
                        cpos += cnt;
                        st_post += cnt;
                        if (cnt < 32) break;
                    }
                    __syncwarp();  // every lane has read this clause's cursor
                    if (lane == 0) tc.pos = cpos;
                    if (lane == t) nd = cpos < n ? cd[cpos] : kNoMoreDocs;  // an emptied cache is refilled below
                    __syncwarp();
                } else if (kt == kKindCol) {
                    uint32_t w = sh.cw[t][lane] & E;
                    if (!__any_sync(0xffffffffu, w != 0u)) continue;
                    const float* col = sh.col[t] + base + 32 * lane;
                    while (w) {
                        const int b = __ffs(w) - 1;
                        w &= w - 1;
                        const uint32_t slot = epre + __popc(E & ((1u << b) - 1u));
                        const float sum = __fadd_rn(sh.acc[slot], __ldg(col + b));
                        sh.acc[slot] = sum;
                        st_gather++;
                        if (sum > te) hot |= 1u << lane;
                    }
                    __syncwarp();
                } else if (kt == kKindBStream) {
                    // a block stream that does not drive windows: seek to this window, add the postings that fall on E
                    if (!__any_sync(0xffffffffu, (sh.cw[t][lane] & E) != 0u)) continue;
                    const int slot = __popc(stream_mask & ((1u << t) - 1u));
                    WTerm& tc = sh.term[t];
                    int32_t* cd = cdocs + slot * kBlock;
                    float* cs = cscores + slot * kBlock;
                    for (;;) {
                        uint32_t cpos = tc.pos;
                        const uint32_t n = tc.n;
                        if (cpos >= n || cd[n - 1] < win0) {  // nothing cached for this window
                            if (tc.cur > tc.nb) break;        // exhausted
                            __syncwarp();                     // every lane has read the cursor
                            if (lane == 0) tc.cur = lower_bound_gallop(tc.blk_last, min(tc.cur, tc.nb), tc.nb, win0);
                            __syncwarp();
                            st_refill++;
                            if (!stream_refill<false, false, false, false>(seg, p, tc, cd, cs, lo, hi, lane, 0, -2147483647 - 1,
                                                                          sh.ubits, hot_unused,
                                                                          mm_unused, INFINITY, mc_unused))
                                break;
                            continue;
                        }
                        const uint32_t i = cpos + lane;
                        const int d = i < n ? cd[i] : kNoMoreDocs;
                        const uint32_t cnt = __popc(__ballot_sync(0xffffffffu, d < win1));  // sorted: a prefix
                        if (d >= win0 && d < win1) {
                            const int idx = d - base;
                            const uint32_t ew = sh.ebits[idx >> 5];
                            if ((ew >> (idx & 31)) & 1u) {
                                const uint32_t slot = sh.epre[idx >> 5] + __popc(ew & ((1u << (idx & 31)) - 1u));
                                const float sum = __fadd_rn(sh.acc[slot], cs[i]);
                                sh.acc[slot] = sum;
                                if (sum > te) hot |= 1u << (idx >> 5);
                            }
                        }
                        st_post += cnt;
                        __syncwarp();  // every lane has read the cursor
                        if (lane == 0) tc.pos = cpos + cnt;
                        __syncwarp();
                        if (cnt < 32 && cpos + cnt < n) break;  // the next cached posting lies beyond the window
                        // else: 32 more may follow, or the cache is used up and the next block may reach into the window
                    }
                    __syncwarp();
                }
            }
            hot = __reduce_or_sync(0xffffffffu, hot);
        }
        // ---- 4. candidates: touched docs (bits of E) whose score beats theta, in docid order
        {
            uint32_t newc_n = 0;
            while (hot) {
                const int s = __ffs(hot) - 1;
                hot &= hot - 1;
                const int idx = s * 32 + lane;
                st_steps++;
                const uint32_t Es = __shfl_sync(0xffffffffu, E, s);
                const uint32_t ps = __shfl_sync(0xffffffffu, epre, s);
                const uint32_t ls = __shfl_sync(0xffffffffu, lw, s);
                const float sc = ((Es >> lane) & 1u) ? sh.acc[ps + __popc(Es & ((1u << lane) - 1u))] : 0.0f;
                const bool cand = ((Es & ls) >> lane) & 1u && (open || sc > te);
                const uint32_t cm = __ballot_sync(0xffffffffu, cand);
                if (!cm || em.overflow) continue;
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
                        continue;
                    }
                    em.run_slot = slot;
                    em.run_cap = cap;
                    em.run_cnt = 0;
                }
                if (cand) {
                    const uint32_t r = __popc(cm & ((1u << lane) - 1u));
                    p.cand_arena[em.run_slot + 1 + em.run_cnt + r] = rg_hit{base + idx + seg.doc_base, sc};
                    if (DEEP) deep_count(reinterpret_cast<uint32_t*>(topk), dmap, sc);
                    else if (newc_n + r < (uint32_t)kNewcW) sh.newc[newc_n + r] = sc;
                }
                em.run_cnt += cn;
                newc_n += cn;
                st_cand += cn;
                if (lane == 0) hdr[em.run_slot] = CandRun{kNone, em.run_cnt};
            }
            __syncwarp();
            // re-arm the accumulator words that were touched (E bits live in the owning lane's word)
            if ((uint32_t)lane < n_e) sh.acc[lane] = 0.0f;
            if ((uint32_t)lane + 32u < n_e) sh.acc[lane + 32] = 0.0f;
            if (DEEP) wtheta_update_deep(em, p, item_idx, dmap, lane, newc_n);
            else wtheta_update(em, p, item_idx, kcap, lane, sh.newc, newc_n);
            __syncwarp();
        }
        pos = win1;
        // ---- 5. refill the sparse streams whose cached block is used up
        {
            bool need = false;
            if (kind == kKindSparse && nd == kNoMoreDocs) {
                const WTerm& tc = sh.term[lane];
                need = tc.pos >= tc.n && tc.cur <= tc.nb;
            }
            for (uint32_t m = __ballot_sync(0xffffffffu, need); m; m &= m - 1) {
                const int t = __ffs(m) - 1;
                const int slot = __popc(stream_mask & ((1u << t) - 1u));
                int first = kNoMoreDocs;
                st_refill++;
                if (stream_refill<false, false, false, false>(seg, p, sh.term[t], cdocs + slot * kBlock, cscores + slot * kBlock,
                                                              lo, hi, lane, 0, -2147483647 - 1,
                                                              sh.ubits, hot_unused, mm_unused,
                                                              INFINITY, mc_unused))
                    first = cdocs[slot * kBlock + sh.term[t].pos];
                if (lane == t) nd = first;
            }
        }
        if (pos >= hi) break;
    }
    my_matches = __reduce_add_sync(0xffffffffu, my_matches);
    if (lane == 0) p.item_matches[item_idx] = my_matches;
    if (p.dbg) {
        st_gather = __reduce_add_sync(0xffffffffu, st_gather);
        st_edocs = __reduce_add_sync(0xffffffffu, st_edocs);
        if (lane == 0) {
            const uint32_t v[13] = {1u, st_win, st_scan, st_open, st_gap, st_post, st_gather, st_refill, st_cand, st_steps,
                                    st_cut, st_scored, st_edocs};
#pragma unroll
            for (int i = 0; i < 13; i++) atomicAdd(p.dbg + i, (unsigned long long)v[i]);
        }
    }
}

template <bool LIVE, bool PLANES, bool DEEP>
static void launch_eval_or_ms_t(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n, size_t wb,
                                uint32_t kcap) {
    const size_t smem = wb * kMsWarps;
    // per launch, not cached: the attribute is per device and engines may live on several
    cudaFuncSetAttribute(k_eval_or_ms<LIVE, PLANES, DEEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const uint32_t ctas = (n + kMsWarps - 1) / kMsWarps;
    k_eval_or_ms<LIVE, PLANES, DEEP><<<ctas, kMsThreads, smem, st>>>(p, item_ids, n, (uint32_t)wb, kcap);
}

template <bool DEEP>
static void launch_eval_or_ms_d(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n,
                                uint32_t max_streams, bool has_live, bool planes) {
    const uint32_t kcap = DEEP ? (uint32_t)kDeepBuckets : (std::min<uint32_t>(p.k, kMaxK) + 31u) & ~31u;
    size_t wb = sizeof(MsWarpShared) + (size_t)kcap * sizeof(float) + (size_t)max_streams * kBlock * 8;
    wb = (wb + 15) & ~size_t(15);
    if (has_live && planes) launch_eval_or_ms_t<true, true, DEEP>(st, p, item_ids, n, wb, kcap);
    else if (has_live) launch_eval_or_ms_t<true, false, DEEP>(st, p, item_ids, n, wb, kcap);
    else if (planes) launch_eval_or_ms_t<false, true, DEEP>(st, p, item_ids, n, wb, kcap);
    else launch_eval_or_ms_t<false, false, DEEP>(st, p, item_ids, n, wb, kcap);
}

void launch_eval_or_ms(cudaStream_t st, const EvalParams& p, const uint32_t* item_ids, uint32_t n,
                       uint32_t max_streams, bool has_live, bool planes) {
    if (!n) return;
    if (p.k > (uint32_t)kMaxK) launch_eval_or_ms_d<true>(st, p, item_ids, n, max_streams, has_live, planes);
    else launch_eval_or_ms_d<false>(st, p, item_ids, n, max_streams, has_live, planes);
}

}  // namespace rg
