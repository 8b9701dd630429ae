"""Constructed indexes for the edges of the disjunction kernels, and an independent numpy model of what they must
return (test_edges_cpu.py checks every fixture against the oracle and the model; test_gpu_edges.py runs them on the
device).  Every index is written with codec.PostingsWriter and explicit norm bytes; scores are BM25 cells
w*(k1+1)*f/(f+cache[norm]) in f32 (bm25_similarity.rs:203-212), a leaf without norms using k1 for cache[norm], added
in clause order from +0.0f."""
import numpy as np

import oracle_binding as ob
from rucene_b200 import codec

F32 = np.float32


# ---- the numpy model -------------------------------------------------------------------------------------------------
def leaf_stats(segs):
    """with_similarity (searcher.rs:306-363): statistics of the largest-max_doc leaf (first among equals), max_doc of
    the whole reader -> (stats leaf index, doc_count, avgdl)"""
    si = max(range(len(segs)), key=lambda i: (segs[i].max_doc, -i))
    s = segs[si]
    max_doc = sum(x.max_doc for x in segs)
    avgdl = codec.bm25_avg_field_length(s.sum_total_term_freq, s.doc_count, max_doc)
    return si, s.doc_count, avgdl


def weight(segs, term, boost):
    si, doc_count, _ = leaf_stats(segs)
    df = int(segs[si].terms["doc_freq"][term])
    return F32(F32(codec.bm25_idf(df, doc_count)) * F32(boost))


def norm_cache(segs, k1, b):
    return codec.bm25_norm_cache(k1, b, leaf_stats(segs)[2])


def cells(w, k1, freqs, norm_vals):
    """norm_vals: cache[norm byte] per posting (k1 in a leaf without norms)"""
    t1 = F32(F32(w) * F32(F32(k1) + F32(1.0)))
    with np.errstate(over="ignore"):   # +inf cells are part of what is tested
        t2 = (t1 * np.asarray(freqs).astype(F32)).astype(F32)
    t3 = (np.asarray(freqs).astype(F32) + np.asarray(norm_vals, F32)).astype(F32)
    return (t2 / t3).astype(F32)


def live_mask(seg):
    if seg.live_docs is None:
        return np.ones(seg.max_doc, bool)
    bits = np.unpackbits(np.asarray(seg.live_docs, np.uint64).view(np.uint8), bitorder="little")
    return bits[:seg.max_doc].astype(bool)


def or_scores(segs, postings, clauses, k1=1.2, b=0.75):
    """Plain-sum disjunction: per leaf (f32 clause-order sums, matched mask).  clauses: [(term, boost)...];
    postings[leaf][term] = (docs, freqs)."""
    cache = norm_cache(segs, k1, b)
    out = []
    for seg, post in zip(segs, postings):
        acc = np.zeros(seg.max_doc, F32)
        hit = np.zeros(seg.max_doc, bool)
        for term, boost in clauses:
            docs, freqs = post[term]
            if len(docs) == 0:
                continue
            nv = np.full(len(docs), F32(k1)) if seg.norms is None else cache[seg.norms[docs]]
            acc[docs] = (acc[docs] + cells(weight(segs, term, boost), k1, freqs, nv)).astype(F32)
            hit[docs] = True
        out.append((acc, hit))
    return out


def total_hits(segs, scored):
    return sum(int(np.count_nonzero(hit & live_mask(seg))) for seg, (_, hit) in zip(segs, scored))


def write_leaf(max_doc, postings, norms, live=None):
    """postings: per term (docs, freqs); live: bool mask or None -> codec.Segment"""
    w = codec.PostingsWriter(doc_version=1, max_doc=max_doc)
    for docs, freqs in postings:
        w.add_term(np.asarray(docs, np.int32), np.asarray(freqs, np.int32))
    words = None
    if live is not None:
        words = np.packbits(np.concatenate([live, np.zeros(-max_doc % 64, bool)]), bitorder="little").view(np.uint64).copy()
    return w.finish(norms=norms, live_docs=words)


def _sorted_postings(mask, freqs):
    docs = np.nonzero(mask)[0].astype(np.int32)
    return docs, np.asarray(freqs)[docs].astype(np.int32)


def sh(*terms):
    """("bool", SHOULD clauses, 0); a term may be (term, boost)"""
    return ("bool", [(ob.SHOULD,) + (t if isinstance(t, tuple) else (t,)) for t in terms], 0)


# ---- 1. spikes: edges of the decode-free kernel and of its column bound ----------------------------------------------
K = 1000               # k of every spike query: seeds per leaf, and at least the spikes of any query
FS = 4                 # seed freq in the two spike columns
STRIDE = 2305          # == 1 mod 32, 128 and 768: successive stride spikes take every offset of a word, a block, a window
RANGE_POSTINGS = (0, 100000)   # 100000: about thirty ranges per (query, leaf), none of them aligned
LIST_STEP = 769        # run starts of the list term: +1 mod 768 from one run to the next
NORM = 108             # every doc's norm byte (a field length of 200)


class SpikeFixture:
    """Two leaves of odd max_doc (the second with deleted docs).  Terms:
    0  column, d % 3 != 0, carries the stride spikes (queried by the A queries)
    1  column, d % 5 != 0, carries the boundary spikes (B queries)
    2  column, d % 7 != 0, plain background
    3  list term: runs of 128 consecutive docids, below the column threshold
    Freq 1 everywhere except: the first K docids of each leaf (seeds) have FS in terms 0 and 1; spikes have distinct
    freqs above FS in their column.  Seeds and spikes are in all three columns.  The seeds of a query score H, every
    spike more, every background doc less (list included), so with k = K the TopDocs are the query's spikes, then
    seeds."""

    MAX_DOCS = (2000001, 1200007)

    def __init__(self):
        self.specs = [sh(0, 2), sh(2, 0), sh((3, 0.25), 0, 2), sh(0, 2, (3, 0.25)),     # A: stride spikes
                      sh(1, 2), sh(2, 1), sh(1, (3, 0.125), 2)]                           # B: boundary spikes
        self.kind = ["A"] * 4 + ["B"] * 3
        self.stride, self.boundary, self.dead_spike = [], [], None
        self.postings, self.segs = [], []
        next_freq = {0: FS + 1, 1: FS + 1}
        for li, M in enumerate(self.MAX_DOCS):
            d = np.arange(M)
            bnd = set()
            den = 256 if li == 0 else 128
            for r in range(1, den):
                bnd.add(M * r // den)
                if li == 0:
                    bnd.add(M * r // den - 1)
            bnd.add(M - 1)
            for lo in self._range_starts(li, M):
                bnd.update((lo - 1, lo))
            bnd = np.array(sorted(bnd), np.int64)
            p0 = K + 200   # the first stride spike: the first place after the seeds where no stride spike is a boundary one
            while True:
                stride = np.arange(p0, M, STRIDE)[:768 if li == 0 else 150]
                if not np.isin(stride, bnd).any():
                    break
                p0 += 1
            special = np.zeros(M, bool)
            special[:K] = True
            special[stride] = True
            special[bnd] = True
            f0 = np.ones(M, np.int32)
            f1 = np.ones(M, np.int32)
            f0[:K] = FS
            f1[:K] = FS
            f0[stride] = np.arange(next_freq[0], next_freq[0] + len(stride))
            next_freq[0] += len(stride)
            f1[bnd] = np.arange(next_freq[1], next_freq[1] + len(bnd))
            next_freq[1] += len(bnd)
            runs = np.arange(K + 64, M - 128, LIST_STEP)[:768 if li == 0 else 300]
            lst = np.zeros(M, bool)
            for s in runs:
                lst[s:s + 128] = True
            post = [_sorted_postings((d % 3 != 0) | special, f0), _sorted_postings((d % 5 != 0) | special, f1),
                    _sorted_postings((d % 7 != 0) | special, np.ones(M, np.int32)),
                    _sorted_postings(lst, np.ones(M, np.int32))]
            live = None
            if li == 1:
                live = (d % 13 != 5) | special   # background deletions, and one deleted spike
                self.dead_spike = int(stride[75])
                live[self.dead_spike] = False
            self.stride.append(stride)
            self.boundary.append(bnd)
            self.postings.append(post)
            self.segs.append(write_leaf(M, post, np.full(M, NORM, np.uint8), live))

    def _range_starts(self, li, M):
        """range starts of the B queries for the explicit RANGE_POSTINGS (search.cu plan_batch: R = ceil(cost / rp),
        at most 256 and max_doc / 128; cost = sum of the clauses' df in the leaf)"""
        d = np.arange(M)
        dfs = {1: np.count_nonzero(d % 5 != 0), 2: np.count_nonzero(d % 7 != 0), 3: 128 * (768 if li == 0 else 300)}
        out = set()
        for rp in RANGE_POSTINGS:
            if not rp:
                continue   # the planner's own grid: a power of two <= 256, on the leaf's max_doc * r / 256 grid
            for terms in ((1, 2), (1, 3, 2)):
                cost = sum(dfs[t] for t in terms) + K + 768   # + the specials (an estimate: R only changes near a step)
                R = max(1, min((cost + rp - 1) // rp, 256, (M + 127) // 128))
                out.update(M * r // R for r in range(1, R))
        return out

    def spikes(self, qi):
        """[(leaf, docid)] of the live spikes of query qi"""
        which = self.stride if self.kind[qi] == "A" else self.boundary
        return [(li, int(x)) for li, xs in enumerate(which) for x in xs if (li, int(x)) != (1, self.dead_spike)]

    def clauses(self, qi):
        return [(c[1], c[2] if len(c) > 2 else 1.0) for c in self.specs[qi][1]]


# ---- 2. ulp-level cases ----------------------------------------------------------------------------------------------
# One leaf, norm byte ULP_NB and freq 1 for the background.  Terms 0-2 are columns for (b), terms 3-4 columns for (a),
# term 5 pads sum_total_term_freq to ULP_TTF so that avgdl (and with it the norm cache) does not depend on the freqs
# chosen below.  The constants were found by a numpy search over boosts, freqs and norm bytes (test_edges_cpu.py
# re-derives every inequality).
ULP_MAX_DOC = 100003
ULP_NB = 108           # field length 200: a large cache entry, so background cells stay low
ULP_TTF = 400000
# (a): the seeds (docids 0..4: the first candidates of the range, so the kernel's theta is H from the first window
# on) and X (docid 2000) score H = cell3 + cell4 of (ULP_A_H); Y (docid 2500) scores the
# next float above H with (ULP_A_Y).  k = 5: X must stay out (ties do not enter), Y must enter.
ULP_A_BOOSTS = (0.5856491923332214, 0.7368105053901672)
ULP_A_H = (102, 16, 41)      # (norm byte, f3, f4)
ULP_A_Y = (103, 8, 41)
ULP_A_SEEDS, ULP_A_X, ULP_A_YDOC = (0, 1, 2, 3, 4), 2000, 2500
# (b): A (docid 3000) has cells a0, a1, a2 in terms 0-2 whose clause-order round-to-nearest sum exceeds C, the
# round-up sum in the kernel's butterfly order ((a0 + a2) + a1); B (docid 1000) scores exactly C.  k = 1.
ULP_B_BOOSTS = (2.102548837661743, 1.6643240451812744, 0.6882572770118713)
ULP_B_A = (100, 21, 37, 30)  # (norm byte, f0, f1, f2)
ULP_B_B = (100, 27, 23, 33)
ULP_B_ADOC, ULP_B_BDOC = 3000, 1000


def ulp_postings():
    """-> (max_doc, postings, norms) of the ulp leaf"""
    M = ULP_MAX_DOC
    d = np.arange(M)
    norms = np.full(M, ULP_NB, np.uint8)
    f = [np.ones(M, np.int32) for _ in range(5)]
    m = [(d % 2 == 0), (d % 3 != 1), (d % 4 != 3), (d % 2 == 1), (d % 5 != 2)]
    for t, v in enumerate(ULP_B_A[1:]):
        f[t][ULP_B_ADOC] = v
    for t, v in enumerate(ULP_B_B[1:]):
        f[t][ULP_B_BDOC] = v
    norms[ULP_B_ADOC], norms[ULP_B_BDOC] = ULP_B_A[0], ULP_B_B[0]
    for doc, (nb, f3, f4) in [(s, ULP_A_H) for s in ULP_A_SEEDS + (ULP_A_X,)] + [(ULP_A_YDOC, ULP_A_Y)]:
        norms[doc] = nb
        f[3][doc], f[4][doc] = f3, f4
    for t in range(3):
        m[t][[ULP_B_ADOC, ULP_B_BDOC]] = True
        m[t][list(ULP_A_SEEDS) + [ULP_A_X, ULP_A_YDOC]] = False
    for t in (3, 4):
        m[t][list(ULP_A_SEEDS) + [ULP_A_X, ULP_A_YDOC]] = True
        m[t][[ULP_B_ADOC, ULP_B_BDOC]] = False
    post = [_sorted_postings(m[t], f[t]) for t in range(5)]
    used = sum(int(p[1].sum()) for p in post)
    post.append((np.array([M - 1], np.int32), np.array([ULP_TTF - used], np.int32)))
    return M, post, norms


def ulp_leaf():
    M, post, norms = ulp_postings()
    return write_leaf(M, post, norms), post


def ulp_specs_a():
    return [sh((3, ULP_A_BOOSTS[0]), (4, ULP_A_BOOSTS[1]))] * 2


def ulp_specs_b():
    return [sh(*[(t, ULP_B_BOOSTS[t]) for t in range(3)])] * 2


def round_up(x64):
    r = F32(x64)
    return r if float(r) >= x64 else np.nextafter(r, F32(np.inf))


def butterfly_round_up(vals):
    """lane i holds vals[i] (0 beyond): __shfl_xor 16..1 with __fadd_ru, lane 0's result"""
    lanes = [F32(0)] * 32
    for i, v in enumerate(vals):
        lanes[i] = F32(v)
    o = 16
    while o:
        lanes = [round_up(float(lanes[i]) + float(lanes[i ^ o])) for i in range(32)]
        o >>= 1
    return lanes[0]


# ---- 3. the limits of the positive-score route -----------------------------------------------------------------------
LIM_MAX_DOC = 30011
LIM_DFS = [0, 1, 3, 129, 700, 4000, 9000, 15000]   # 4000 and up: score columns (df >= max_doc / 8); 700 and up: bitmaps
HOT = 6                                           # limits_leaf(hot=True): freqs 300..599 in this term


def limits_leaf(seed, max_doc=LIM_MAX_DOC, norms=True, hot=False, norm_byte_one=None, live_fraction=None):
    """Random postings of LIM_DFS, norm bytes 95..124 (or none); hot: term HOT's freqs in 300..599 (cells of +inf at
    k1 = 1e6 and a weight near 1e30 from freq 340 on); norm_byte_one: that doc gets norm byte 1, whose cache entry is
    above 1e10 -> (segment, postings)"""
    rng = np.random.default_rng(seed)
    post = []
    for t, df in enumerate(LIM_DFS):
        docs = np.sort(rng.choice(max_doc, size=df, replace=False)).astype(np.int32)
        freqs = np.minimum(rng.geometric(0.4, size=df), 255).astype(np.int32)
        if hot and t == HOT:
            freqs = rng.integers(300, 600, size=df).astype(np.int32)
        post.append((docs, freqs))
    nb = None
    if norms:
        nb = rng.integers(95, 125, size=max_doc).astype(np.uint8)
        if norm_byte_one is not None:
            nb[norm_byte_one] = 1
    live = None if live_fraction is None else rng.random(max_doc) < live_fraction
    return write_leaf(max_doc, post, nb, live), post


def boost_next_to(segs, term, target, above, strict_above):
    """The f32 boost next to the edge of fl(idf * boost) vs target: the smallest boost whose weight is above the edge
    (above=True) or the largest one below it.  strict_above: the edge is "> target" (else ">= target")."""
    si, doc_count, _ = leaf_stats(segs)
    idf = F32(codec.bm25_idf(int(segs[si].terms["doc_freq"][term]), doc_count))
    t = F32(target)

    def is_above(bo):
        w = F32(idf * bo)
        return w > t if strict_above else w >= t
    bo = F32(t / idf)
    while is_above(bo):
        bo = np.nextafter(bo, F32(0))
    while not is_above(bo):
        bo = np.nextafter(bo, F32(np.inf))
    return bo if above else np.nextafter(bo, F32(0))


def weight_edge_boosts(segs):
    """{term: [boost below 1e-20f, at 1e-20f, at or below 1e30f, above 1e30f]} for the column terms 5 and 7"""
    return {t: [boost_next_to(segs, t, 1e-20, False, False), boost_next_to(segs, t, 1e-20, True, False),
                boost_next_to(segs, t, 1e30, False, True), boost_next_to(segs, t, 1e30, True, True)] for t in (5, 7)}


def tiny_boost(segs, term, w):
    """the smallest boost whose weight fl(idf * boost) is at least the subnormal w (the smallest subnormal: exactly)"""
    return boost_next_to(segs, term, w, True, False)
