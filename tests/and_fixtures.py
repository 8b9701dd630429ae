"""Constructed indexes for the edges of the conjunction kernels (eval_and_body: k_eval_and and k_eval_and_ranges, plain
and ReqOpt), and an independent numpy model of what they must return.  test_and_edges_cpu.py checks every fixture
against the oracle and the model, and that each fixture reaches its edge; test_gpu_and_edges.py runs them on the device.

Scores follow edge_fixtures: BM25 cells in f32.  A conjunction adds its required scorers in ConjunctionScorer cost
order (a stable sort by the leaf's df), starting from the cheapest one's score; a FILTER scorer adds +0.0f, and so does
a point range.  ReqOptScorer keeps a sequential f32 (scores_sum, scores_num) over the collected docs of the leaf."""
import types

import numpy as np

import edge_fixtures as E
import oracle_binding as ob
import points_fixtures as pf
import points_oracle as po
from rucene_b200 import codec

F32 = np.float32
R = po.RANGE
MUST, SHOULD, FILTER, MUST_NOT = ob.MUST, ob.SHOULD, ob.FILTER, ob.MUST_NOT


def write_leaf(max_doc, postings, norms, live=None, doc_version=1, use_ef=False, with_pf=True):
    """postings: per term (docs, freqs) -> (codec.Segment, (blocks, ef blocks, bitset blocks))"""
    w = codec.PostingsWriter(doc_version=doc_version, max_doc=max_doc, use_ef=use_ef, with_pf=with_pf)
    for docs, freqs in postings:
        w.add_term(np.asarray(docs, np.int32), np.asarray(freqs, np.int32))
    counts = w.block_counts()
    words = None
    if live is not None:
        words = np.packbits(np.concatenate([live, np.zeros(-max_doc % 64, bool)]), bitorder="little").view(np.uint64).copy()
    return w.finish(norms=norms, live_docs=words), counts


# ---- the numpy model -------------------------------------------------------------------------------------------------
def _clauses(spec):
    return [(c[0], c[1], F32(c[2]) if len(c) > 2 else (F32(0.0) if c[0] & R else F32(1.0))) for c in spec[1]]


def model_leaf(segs, postings, si, spec, points=None, ranges=None, k1=1.2, b=0.75, skip="f32", collected_from=None):
    """The collected docs of leaf si for a conjunction / ReqOpt BooleanQuery spec ("bool", [(occur, id[, boost])], 0)
    (occur | R: id indexes `ranges`, points[si] the leaf's point fields) -> (docs, f32 scores, chain state).
    skip / collected_from: variants of the running-mean rule, to show that a fixture tells them apart:
    "f32" (the scorer's), "ge" (scores_num >= 100), "le" (2 * req <= mean), "double" (the comparison in double),
    "none" (never skip), "opt_only" (the state moves only when the optional side matched); collected_from: the chain
    state (sum, num) the leaf starts from (a scorer that does not start again per leaf)."""
    seg, post = segs[si], postings[si]
    M = seg.max_doc
    cache = E.norm_cache(segs, k1, b)
    cl = _clauses(spec)
    mask = np.ones(M, bool)
    req, opts = [], []
    has_const = False
    for occ, t, boost in cl:
        if occ & R:
            d = pf.model_docs(points[si] if points else {}, ranges[t])
            inr = np.zeros(M, bool)
            if d is not None:
                inr[d] = True
            if (occ & ~R) == MUST_NOT:
                mask &= ~inr
            else:
                mask &= inr
                has_const = True
            continue
        docs, freqs = post[t] if t < len(post) else (np.zeros(0, np.int32), np.zeros(0, np.int32))
        pres = np.zeros(M, bool)
        pres[docs] = True
        if occ == MUST_NOT:
            mask &= ~pres
        elif occ == SHOULD:
            if len(docs):
                opts.append((t, boost, docs, freqs))
        else:
            mask &= pres
            req.append((occ, t, boost, docs, freqs))

    def cell_array(t, boost, docs, freqs):
        out = np.zeros(M, F32)
        nv = np.full(len(docs), F32(k1)) if seg.norms is None else cache[seg.norms[docs]]
        out[docs] = E.cells(E.weight(segs, t, boost), k1, freqs, nv)
        return out

    order = sorted(range(len(req)), key=lambda i: len(req[i][3]))   # stable: clause order among equal df
    score = None
    for i in order:
        occ, t, boost, docs, freqs = req[i]
        c = np.zeros(M, F32) if occ == FILTER else cell_array(t, boost, docs, freqs)
        score = c if score is None else (score + c).astype(F32)
    if score is None:
        score = np.zeros(M, F32)
    elif has_const:
        score = (score + F32(0.0)).astype(F32)
    docs = np.nonzero(mask & E.live_mask(seg))[0]
    sc = score[docs].copy()
    state = (F32(0.0), 0)
    if opts and (req or has_const):
        osum = np.zeros(M, F32)
        ohit = np.zeros(M, bool)
        for t, boost, od, of in opts:
            osum = (osum + cell_array(t, boost, od, of)).astype(F32)
            ohit[od] = True
        s, n = collected_from if collected_from is not None else (F32(0.0), 0)
        for j, d in enumerate(docs):
            r = sc[j]
            if skip != "none" and n > (99 if skip == "ge" else 100):
                mean = F32(s / F32(n))
                two = F32(F32(2.0) * r)
                if skip == "double":
                    skipped = float(two) < float(s) / n
                elif skip == "le":
                    skipped = two <= mean
                else:
                    skipped = two < mean
                if skipped:
                    continue
            if skip != "opt_only" or ohit[d]:
                s = F32(s + r)
                n += 1
            if ohit[d]:
                sc[j] = F32(r + osum[d])
        state = (s, n)
    return docs, sc, state


def model_topdocs(segs, postings, specs, points=None, ranges=None, **kw):
    """SEARCH-mode results of every query: [(global docids, scores, total_hits)] of every collected doc, score
    descending, docid ascending.  kw["carry"]: the ReqOpt chain does not start again per leaf."""
    carry = kw.pop("carry", False)
    out = []
    base = np.cumsum([0] + [s.max_doc for s in segs])
    for spec in specs:
        gd, gs = [], []
        state = None
        for si in range(len(segs)):
            d, s, st = model_leaf(segs, postings, si, spec, points, ranges,
                                  collected_from=state if carry else None, **kw)
            if carry and st[1]:
                state = st
            gd.append(d + base[si])
            gs.append(s)
        gd, gs = np.concatenate(gd), np.concatenate(gs)
        o = np.lexsort((gd, -gs.astype(np.float64)))
        out.append((gd[o], gs[o], len(gd)))
    return out


def same_as_model(got, model, k, label=""):
    """got: (hits, counts, total) of SEARCH mode.  The model does not restate which of several docs that tie at the
    k-th score the heap keeps: above that score the docs must be the model's, at it a subset of the model's."""
    gh, gc, gt = got
    for i, (d, s, n) in enumerate(model):
        m = min(k, n)
        assert int(gt[i]) == n, (label, "query", i, "total_hits", int(gt[i]), n)
        assert int(gc[i]) == m, (label, "query", i, "count")
        g = gh[i][:m]
        assert np.array_equal(g["score"].view(np.uint32), s[:m].view(np.uint32)), (label, "query", i, "scores")
        if m == 0:
            continue
        last = s[m - 1]
        above = g["score"] != last
        assert sorted(g["doc"][above].tolist()) == sorted(d[:m][s[:m] != last].tolist()), (label, "query", i, "docs")
        assert set(g["doc"][~above].tolist()) <= set(d[s == last].tolist()), (label, "query", i, "tied docs")


def queries(specs, ranges=None):
    """specs -> (oracle queries, oracle clauses); a range clause's boost is 0"""
    qs, cs = [], []
    for s in specs:
        qs.append((len(cs), len(s[1]), s[2], 1))
        for c in s[1]:
            cs.append((c[0], c[1], c[2] if len(c) > 2 else (0.0 if c[0] & R else 1.0)))
    return np.array(qs, ob.QUERY_DTYPE), np.array(cs, ob.CLAUSE_DTYPE)


# ---- A. term-led conjunctions ----------------------------------------------------------------------------------------
A_MAX_DOC = 400009
A_LEAD_DFS = (1, 127, 128, 129, 1024, 1025, 7 * 128 + 5, 9 * 128)   # terms 1..8
A_P, A_GALLOP, A_CUT, A_NOT, A_WIDTH = 0, 9, 10, 11, 12
A_CUT_RP = 150          # range_postings of the cut runs: the cut lead (df 572) makes R = 4 items
A_CUT_R = 4
A_VARIANTS = {"v0": (0, False, True), "v1": (1, False, True), "v1_ef_pf": (1, True, True), "v1_ef": (1, True, False)}


class TermLeadFixture:
    """One leaf of A_MAX_DOC docs.  Term 0 (P) is the probe: d % 3 != 2 up to 50 docs before the end, with thousands of
    blocks whose freq widths cycle through 1..31 bits (each block holds a freq 2^w - 1).  Terms 1..8 are leads of
    A_LEAD_DFS docs taken from the probe's edges: each block's first and last docid, the last docid of the last full
    block, the first tail doc, and docs past the last posting.  Term 9 (G) gallops over P: two or three docs per probe
    block, jumps of 0, 1, 2 and 2^k blocks and to the tail; every pair of lead slots across a 32-slot chunk boundary
    falls in one probe block.  Term 10 (C) is cut into A_CUT_R items by range_postings A_CUT_RP: it has docs at each
    item's lo, hi - 1 and hi, and its last full block ends at the last item's lo - 1, so the item before that has no
    tail in scope.  Term 11 (N) is a MUST_NOT on lead-block, probe-block and tail edges.  Term 12 (W) is a lead of 31
    full blocks whose freqs need 1..31 bits."""

    def __init__(self, variant="v1"):
        self.variant = variant
        doc_version, use_ef, with_pf = A_VARIANTS[variant]
        M = A_MAX_DOC
        rng = np.random.default_rng(7)
        d = np.arange(M)
        pmask = (d % 3 != 2) & (d < M - 50)
        self.cut_bounds = [M * r // A_CUT_R for r in range(1, A_CUT_R)]
        for bnd in self.cut_bounds:
            pmask[[bnd - 1, bnd]] = True
        pmask[0] = True
        P = np.nonzero(pmask)[0].astype(np.int32)
        nb = len(P) // 128
        pf_ = np.ones(len(P), np.int64)
        for j in range(nb + 1):
            w = 1 + j % 31
            blk = slice(128 * j, min(len(P), 128 * (j + 1)))
            n = blk.stop - blk.start
            if n == 0:
                continue
            f = rng.integers(1, min(4, 1 << w), n)
            f[(j * 37) % n] = (1 << w) - 1
            pf_[blk] = f
        self.P, self.nb = P, nb
        firsts, lasts, tail = P[0:128 * nb:128], P[127:128 * nb:128], P[128 * nb:]
        self.last_full, self.first_tail = int(lasts[-1]), int(tail[0])
        past = np.array([int(P[-1]) + 1, int(P[-1]) + 7, M - 1], np.int32)
        self.past = past
        pool = np.unique(np.concatenate([firsts, lasts, tail[:4], firsts[::7] + 1, past]))
        post = [(P, pf_.astype(np.int32))]
        leads = []
        for df in A_LEAD_DFS:
            if df == 1:
                docs = np.array([self.last_full], np.int32)
            else:
                must = np.array([P[0], self.last_full, self.first_tail, M - 1])
                rest = np.setdiff1d(pool, must)
                pick = rest[np.linspace(0, len(rest) - 1, df - len(must)).round().astype(int)]
                docs = np.unique(np.concatenate([must, pick]))
                assert len(docs) == df, (df, len(docs))
            leads.append(docs.astype(np.int32))
        for docs in leads:
            post.append((docs, rng.integers(1, 300, len(docs)).astype(np.int32)))
        post.append(self._gallop(P, nb, firsts, lasts, tail, past))
        post.append(self._cut(P, rng))
        not_docs = np.unique(np.concatenate([leads[7][0::128], leads[7][127::128], leads[4][::3],
                                             firsts[::5], lasts[::5], tail[::2], post[A_GALLOP][0][::4]]))
        post.append((not_docs.astype(np.int32), np.ones(len(not_docs), np.int32)))
        wd = P[::60][:31 * 128 + 20]
        wf = np.ones(len(wd), np.int64)
        for j in range(32):
            blk = slice(128 * j, min(len(wd), 128 * (j + 1)))
            n = blk.stop - blk.start
            w = min(j + 1, 31)
            wf[blk] = rng.integers(1, (1 << w), n) if w > 1 else 1
            wf[blk.start + (j * 11) % n] = (1 << w) - 1
        post.append((wd, wf.astype(np.int32)))
        self.postings = [post]
        norms = rng.integers(90, 131, M).astype(np.uint8)
        seg, self.block_counts = write_leaf(M, post, norms, doc_version=doc_version, use_ef=use_ef, with_pf=with_pf)
        self.segs = [seg]

    @staticmethod
    def _gallop(P, nb, firsts, lasts, tail, past):
        blocks, j = [], 0
        for k in range(12):
            for jump in (0, 1, 2, 1 << k):
                if j + jump >= nb:
                    break
                j += jump
                blocks.append(j)
        docs = []
        for j in blocks:
            inner = list(P[128 * j:128 * (j + 1)])
            want = [inner[0], inner[-1]]
            if docs and docs[-1] >= inner[0]:
                want = [x for x in inner if x > docs[-1]][-1:]
            for x in want:
                if len(docs) % 32 == 31:   # the slots on both sides of a chunk boundary: one probe block
                    nxt = [y for y in inner if y > (docs[-1] if docs else -1)]
                    if len(nxt) >= 2:
                        docs += [nxt[0], nxt[1]]
                        continue
                if not docs or x > docs[-1]:
                    docs.append(x)
        docs += [int(t) for t in tail[:3] if t > docs[-1]] + [int(x) for x in past]
        docs = np.array(docs, np.int32)
        return docs, (np.arange(len(docs)) % 200 + 1).astype(np.int32)

    def _cut(self, P, rng):
        M = A_MAX_DOC
        b1, b2, b3 = self.cut_bounds
        must_lo = np.array([0, b1 - 1, b1, b2 - 1, b2, b3 - 1])
        cand = np.setdiff1d(P[P < b3 - 1], must_lo)
        lo_part = np.unique(np.concatenate([must_lo, cand[np.linspace(0, len(cand) - 1, 512 - 6).round().astype(int)]]))
        cand = np.setdiff1d(P[P > b3], [b3])
        hi_part = np.unique(np.concatenate([[b3], cand[np.linspace(0, len(cand) - 1, 58).round().astype(int)], [M - 1]]))
        docs = np.concatenate([lo_part, hi_part]).astype(np.int32)
        assert len(docs) == 572 and docs[511] == b3 - 1, (len(docs), docs[511])
        return docs, rng.integers(1, 50, len(docs)).astype(np.int32)

    def item_bounds(self, df, rp):
        """search.cu plan_batch for a term-led conjunction: R = ceil(df / rp) (at most 256 and the leaf's 128-doc
        blocks), item r = [max_doc * r / R, max_doc * (r + 1) / R)"""
        M = A_MAX_DOC
        Rn = max(1, min(-(-df // rp), 256, (M + 127) // 128))
        return [(M * r // Rn, M * (r + 1) // Rn) for r in range(Rn)]

    @staticmethod
    def specs():
        p = A_P
        sp = [("bool", [(MUST, t), (MUST, p)], 0) for t in range(1, 9)]
        sp += [("bool", [(MUST, p), (MUST, t)], 0) for t in (A_GALLOP, A_CUT, A_WIDTH)]
        sp += [("bool", [(MUST, 8), (MUST, p), (MUST_NOT, A_NOT)], 0),
               ("bool", [(MUST, A_GALLOP), (MUST, p), (MUST_NOT, A_NOT)], 0),
               ("bool", [(MUST, A_WIDTH), (MUST_NOT, A_NOT)], 0),
               ("bool", [(MUST, A_CUT), (MUST, p), (MUST_NOT, A_NOT)], 0),
               ("bool", [(MUST, 8), (FILTER, p)], 0), ("bool", [(FILTER, 5), (MUST, p)], 0),
               ("bool", [(FILTER, A_GALLOP), (FILTER, p), (MUST, A_WIDTH)], 0),
               ("bool", [(MUST, 8, -0.0), (MUST, p)], 0), ("bool", [(MUST, p, -0.0), (MUST, 7)], 0),
               ("bool", [(MUST, 8, -0.0), (FILTER, p)], 0), ("bool", [(MUST, 6, -0.0), (MUST, p, -0.0)], 0),
               ("bool", [(MUST, 5), (MUST, A_WIDTH), (MUST, p)], 0)]
        return sp


# ---- B. ReqOpt -------------------------------------------------------------------------------------------------------
B_A, B_B, B_O, B_N, B_PAD = 0, 1, 2, 3, 4
B_MAX_DOCS = (20011, 1009, 1009, 1013, 3001)   # chain, equal, below, restart, no optional term
B_TTF = 400000
B_BG = (3, 3, 108)        # background (freq a, freq b, norm byte): 2 * req is never below the mean
B_LOW = (1, 1, 100)       # a low required score: 2 * req below the background mean
B_O_SMALL, B_O_BIG = 2, 400
B_K = 5


class ReqOptFixture:
    """MUST a, MUST b, SHOULD o, MUST_NOT n over five leaves.
    Leaf 0 (chain): a on even docs < 6000; 100 collected docs among the first 1030 lead slots (others lack b, are
    deleted or excluded by n), half of them without o; lead slot 1030 is the 101st collected doc (low required score,
    large o: must get o), slot 1031 the 102nd (same, larger o: must not).  Leaf 1 (equal): 101 background docs, a doc z,
    then x with 2 * req == the f32 mean, which is below the exact mean: kept in f32, skipped in double.  Leaf 2 (below):
    the same with y one ulp below the mean: skipped.  Leaf 3 (restart): a low doc with large o as the 5th collected doc:
    the chain starts again from zero.  Leaf 4: no o at all (a plain conjunction), written with EF / BITSET blocks when
    ef=True."""

    def __init__(self, ef=False):
        self.ef = ef
        rng = np.random.default_rng(3)
        self.postings, self.segs, self.counts = [], [], []
        self.decisive = {}
        # leaf 0 first: it fixes the statistics
        self._leaf0(rng)
        self.search = self._find_equal_and_below()
        for li in (1, 2):
            self._leaf_eq(li)
        self._leaf_restart()
        self._leaf_noopt()

    def _finish(self, M, terms, norms, live=None, use_ef=False, with_pf=True):
        """terms: {term: {doc: freq}}"""
        post = []
        for t in range(5):
            m = terms.get(t, {})
            docs = np.array(sorted(m), np.int32)
            post.append((docs, np.array([m[x] for x in docs], np.int32)))
        if len(self.segs) == 0:   # the chain leaf: pad sum_total_term_freq to B_TTF
            used = sum(int(p[1].sum()) for p in post[:4])
            post[B_PAD] = (np.array([M - 1], np.int32), np.array([B_TTF - used], np.int32))
        seg, counts = write_leaf(M, post, norms, live, use_ef=use_ef, with_pf=with_pf)
        self.postings.append(post)
        self.segs.append(seg)
        self.counts.append(counts)

    def _leaf0(self, rng):
        M = B_MAX_DOCS[0]
        terms = {t: {} for t in range(4)}
        norms = np.full(M, 108, np.uint8)
        live = np.ones(M, bool)
        coll = set(np.linspace(3, 1027, 100).round().astype(int).tolist())
        assert len(coll) == 100
        reason = 0
        for p in range(3000):
            d = 2 * p
            terms[B_A][d] = 3
            if p < 1030 and p not in coll:
                r = reason % 3
                reason += 1
                if r != 0:
                    terms[B_B][d] = 3
                if r == 1:
                    live[d] = False
                if r == 2:
                    terms[B_N][d] = 1
                if reason % 2:
                    terms[B_O][d] = B_O_BIG + 50    # not collected: its o must never count
                continue
            fa, fb, nb = B_BG
            terms[B_B][d] = fb
            terms[B_A][d] = fa
            norms[d] = nb
            if p in (1030, 1031) or (p > 1031 and p % 250 == 0):
                terms[B_A][d], terms[B_B][d], norms[d] = B_LOW
                terms[B_O][d] = B_O_BIG + (p - 1030)
            elif p % 2:
                terms[B_O][d] = B_O_SMALL
        for d in range(6000, M, 3):   # noise after the chain: more df for b and o
            terms[B_B][d] = 1
            if d % 2:
                terms[B_O][d] = 1
        self.decisive[0] = (2 * 1030, 2 * 1031)
        self._finish(M, terms, norms, live)

    def _weights(self):
        segs = self.segs[:1] + [types.SimpleNamespace(max_doc=md) for md in B_MAX_DOCS[1:]]
        return ([E.weight(segs, t, 1.0) for t in (B_A, B_B, B_O)], E.norm_cache(segs, 1.2, 0.75))

    def _req(self, fa, fb, nb):
        (wa, wb, _), cache = self._weights()
        ca = E.cells(wa, 1.2, np.asarray(fa), cache[np.asarray(nb)])
        cb = E.cells(wb, 1.2, np.asarray(fb), cache[np.asarray(nb)])
        return (ca + cb).astype(F32)

    def _find_equal_and_below(self):
        """numpy search over (freq a, freq b, norm byte): the background chain of 101 docs, then z (not skipped),
        then x with fl(2 * req_x) == fl(sum / 102) < sum / 102 exactly, and y with 2 * req_y one ulp below that mean"""
        fa, fb, nb = np.meshgrid(np.arange(1, 41), np.arange(1, 41), np.arange(0, 256), indexing="ij")
        fa, fb, nb = fa.ravel(), fb.ravel(), nb.ravel()
        req = self._req(fa, fb, nb)
        r0 = self._req(*[np.array([v]) for v in B_BG])[0]
        s = F32(0.0)
        for _ in range(101):
            s = F32(s + r0)
        mean_bg = F32(s / F32(101))
        zok = F32(2.0) * req >= mean_bg
        sums = (s + req).astype(F32)
        means = (sums / F32(102)).astype(F32)
        below_exact = sums.astype(np.float64) / 102.0 > means.astype(np.float64)
        two = (F32(2.0) * req).astype(F32)
        two_bits = two.view(np.uint32)
        order = np.argsort(two_bits, kind="stable")
        sorted_bits = two_bits[order]

        def find(target_bits, ok):
            pos = np.searchsorted(sorted_bits, target_bits)
            pos = np.minimum(pos, len(sorted_bits) - 1)
            hit = ok & (sorted_bits[pos] == target_bits)
            zi = int(np.nonzero(hit)[0][0])
            return zi, int(order[pos[zi]])

        zx, x = find(means.view(np.uint32), zok & below_exact)
        below = np.nextafter(means, F32(-np.inf)).astype(F32)
        zy, y = find(below.view(np.uint32), zok)
        pick = lambda i: (int(fa[i]), int(fb[i]), int(nb[i]))
        return {"r0": r0, "z_eq": pick(zx), "x": pick(x), "z_below": pick(zy), "y": pick(y)}

    def _leaf_eq(self, li):
        M = B_MAX_DOCS[li]
        terms = {t: {} for t in range(4)}
        norms = np.full(M, 108, np.uint8)
        z, dec = (self.search["z_eq"], self.search["x"]) if li == 1 else (self.search["z_below"], self.search["y"])
        for d in range(101):
            terms[B_A][d], terms[B_B][d], norms[d] = B_BG
            if d % 3 == 0:
                terms[B_O][d] = B_O_SMALL
        for d, (fa, fb, nb) in ((101, z), (102, dec)):
            terms[B_A][d], terms[B_B][d], norms[d] = fa, fb, nb
        terms[B_O][102] = B_O_BIG + (10 if li == 2 else 0)
        for d in range(200, 400, 7):   # docs without a: b and o only
            terms[B_B][d] = 2
            terms[B_O][d] = 2
        self.decisive[li] = (102,)
        self._finish(M, terms, norms)

    def _leaf_restart(self):
        M = B_MAX_DOCS[3]
        terms = {t: {} for t in range(4)}
        norms = np.full(M, 108, np.uint8)
        for d in range(0, 40, 2):
            terms[B_A][d], terms[B_B][d], norms[d] = B_BG
        terms[B_A][8], terms[B_B][8], norms[8] = B_LOW
        terms[B_O][8] = B_O_BIG + 5
        self.decisive[3] = (8,)
        self._finish(M, terms, norms)

    def _leaf_noopt(self):
        M = B_MAX_DOCS[4]
        terms = {t: {} for t in range(4)}
        for d in range(0, 1500):
            terms[B_A][d] = 1 + d % 3
        for d in range(0, 3000, 2):
            terms[B_B][d] = 2
        self._finish(M, terms, np.full(M, 100, np.uint8), use_ef=self.ef, with_pf=False)

    @staticmethod
    def specs():
        a, b, o, n = B_A, B_B, B_O, B_N
        return [("bool", [(MUST, a), (MUST, b), (SHOULD, o), (MUST_NOT, n)], 0),
                ("bool", [(MUST, b), (SHOULD, o), (MUST, a), (MUST_NOT, n)], 0)]


# ---- C. range conjunctions -------------------------------------------------------------------------------------------
C_BLOCKS = 151                       # 150 full 128-doc blocks and a last partial block of 77 docs
C_MAX_DOC = 128 * (C_BLOCKS - 1) + 77
C_BAND = 1 << 20                     # keys of the taken blocks start here
C_S = list(range(0, 7)) + [32] + list(range(33, 40)) + [64] + [131, 133, 135, 150]
C_W127, C_WMV, C_MANY, C_ABOVE, C_OOO = 3, 5, 33, 36, 64   # special blocks of field F
F_MAIN, F_MISS, F_INT, F_LONG, F_SEQ = 0, 1, 2, 3, 4
C_T_ALL, C_T_HALF, C_T1, C_T2, C_T_EQ, C_T_EQ1 = 0, 1, 2, 3, 4, 5
C_SEQ_COUNT = 15001                  # the F_SEQ range: docs 1000..16000 (one key each), every split item's lo
C_SPLIT_RP = 4000                    # range_postings of the split runs: R = 4 range-lead items
LONG_EXTREMES = (-(1 << 63), -1, 0, (1 << 63) - 1)
INT_EXTREMES = (-(1 << 31), (1 << 31) - 1)


def c_key(block, d):
    return C_BAND + block * 1024 + (d % 128)


class RangeFixture:
    """One leaf of C_MAX_DOC docs with point fields, next to a leaf without them.
    F_MAIN (LongPoint): blocks in C_S carry keys from C_BAND up (block B: C_BAND + 1024 B + d % 128), every other block
    keys below C_BAND, blocks 140..149 none.  Read 32 block-table entries at a time from block 0, the taken blocks put
    the 8th of a step at lane 0 (block 32) and at lane 31 (block 64) of a read, leave runs of 24 and 66 blocks between
    them, and end with fewer than 8 before rend = 151.  Block C_W127 has 127 valued docs and 128 values; block C_WMV is
    fully valued with one doc that also has a value past the band; block C_MANY holds a doc with 40 values of which
    only the last is in the band, and C_ABOVE a doc whose only key is above every upper bound; block C_OOO holds
    multi-valued docs uploaded with their keys out of order.  The last partial block is fully valued.
    F_MISS: F_MAIN without doc max_doc - 1.  F_INT / F_LONG: keys at the u32 and u64 extremes.  F_SEQ: key = docid."""

    def __init__(self, ef=False):
        self.ef = ef
        rng = np.random.default_rng(17)
        M = C_MAX_DOC
        d = np.arange(M)
        post = [(d, np.ones(M, np.int32)),                                        # t_all: every doc
                (d[d % 2 == 0], (1 + d[d % 2 == 0] % 5).astype(np.int32))]        # t_half
        t1 = np.sort(rng.choice(M, 3000, replace=False))
        t2 = np.sort(rng.choice(M, 9000, replace=False))
        post += [(t1, rng.integers(1, 20, len(t1))), (t2, rng.integers(1, 20, len(t2)))]
        post += [(np.arange(100, 400), np.ones(300, np.int64)), (np.arange(99, 400), np.ones(301, np.int64))]
        post = [(np.asarray(a, np.int32), np.asarray(f, np.int32)) for a, f in post]
        norms = rng.integers(95, 125, M).astype(np.uint8)
        seg, self.block_counts = write_leaf(M, post, norms, use_ef=ef, with_pf=False)
        seg2, _ = write_leaf(5003, [(np.arange(0, 5003, 3), np.ones(1668)), (np.arange(0, 5003, 2), np.ones(2502))],
                             rng.integers(95, 125, 5003).astype(np.uint8))
        self.segs = [seg, seg2]
        self.postings = [post, [(np.arange(0, 5003, 3, dtype=np.int32), np.ones(1668, np.int32)),
                                (np.arange(0, 5003, 2, dtype=np.int32), np.ones(2502, np.int32))]]
        docs, keys = [], []
        for B in range(C_BLOCKS):
            if 140 <= B < 150:
                continue
            for x in range(128 * B, min(M, 128 * (B + 1))):
                if B == C_W127 and x == 128 * B + 40:
                    continue
                docs.append(x)
                keys.append(c_key(B, x) if B in C_S else B * 64 + x % 64)
        extra = [(128 * C_W127 + 41, c_key(C_W127, 128 * C_W127 + 100)),   # 128 values, 127 docs
                 (128 * C_WMV + 9, 3 * C_BAND)]                             # a value past every band range
        many = 128 * C_MANY + 50
        keys[docs.index(many)] = 17                                         # 40 values, the last one in the band
        extra += [(many, 18 + j) for j in range(38)] + [(many, c_key(C_MANY, many))]
        above = 128 * C_ABOVE + 70
        keys[docs.index(above)] = 3 * C_BAND
        for x in range(128 * C_OOO + 3, 128 * C_OOO + 128, 9):             # out of order: the band key is uploaded first
            extra.append((x, 5))
        self.many_doc, self.above_doc, self.w127_missing = many, above, 128 * C_W127 + 40
        docs = np.array(docs + [e[0] for e in extra], np.int32)
        keys = np.array(keys + [e[1] for e in extra], np.int64)
        perm = rng.permutation(len(docs))
        perm = np.concatenate([perm[perm < len(keys) - len(extra)], perm[perm >= len(keys) - len(extra)]])
        docs, keys = docs[perm], keys[perm]
        miss = docs != M - 1
        ints = np.array([INT_EXTREMES[i % 2] if i % 5 == 0 else int(v) for i, v in
                         enumerate(rng.integers(-(1 << 31), 1 << 31, M))], np.int64)
        lng = np.array([LONG_EXTREMES[i % 4] if i % 3 == 0 else int(v) for i, v in
                        enumerate(rng.integers(-(1 << 62), 1 << 62, M))], np.int64)
        self.points = [{F_MAIN: self._field(8, docs, keys), F_MISS: self._field(8, docs[miss], keys[miss]),
                        F_INT: self._field(4, np.arange(M, dtype=np.int32), ints),
                        F_LONG: self._field(8, np.arange(M, dtype=np.int32), lng),
                        F_SEQ: self._field(8, np.arange(M, dtype=np.int32), np.arange(M, dtype=np.int64))}, {}]
        self.ranges = self._ranges()

    @staticmethod
    def _field(nb, docs, vals):
        return (nb, np.asarray(docs, np.int32), pf.packed_of(nb, vals), vals)

    def _ranges(self):
        L, I = po.long_pack, po.int_pack
        mk = lambda f, lo, hi, nb=8: po.make_range(f, nb, (L if nb == 8 else I)(lo), (L if nb == 8 else I)(hi))
        b2 = 33
        out = [mk(F_MAIN, C_BAND, 2 * C_BAND),                                  # 0: every band block
               mk(F_MAIN, c_key(6, 0), c_key(6, 127)),                          # 1: block 6's min and max
               mk(F_MAIN, c_key(b2, 127), c_key(b2 + 1, 64)),                   # 2: lower = block 33's max
               mk(F_MAIN, 2 * C_BAND, 2 * C_BAND + 5),                          # 3: points in the leaf, none inside
               mk(F_MISS, C_BAND, 2 * C_BAND),                                  # 4: last block misses max_doc - 1
               mk(F_MAIN, c_key(150, 0), c_key(150, 127)),                      # 5: the last partial block
               mk(F_MAIN, c_key(C_W127, 0), c_key(C_W127, 127)),                # 6: 127 docs, 128 values
               mk(F_SEQ, 1000, 1000 + C_SEQ_COUNT - 1),                         # 7: split items
               mk(F_SEQ, 100, 399),                                             # 8: count 300 (= df of t_eq)
               mk(F_INT, INT_EXTREMES[0], INT_EXTREMES[0], 4), mk(F_INT, INT_EXTREMES[1], INT_EXTREMES[1], 4),
               mk(F_INT, INT_EXTREMES[0], INT_EXTREMES[1], 4)]                   # 9..11
        out += [mk(F_LONG, lo, hi) for lo, hi in ((LONG_EXTREMES[0], LONG_EXTREMES[0]), (-1, 0), (-1, -1), (0, 0),
                                                   (LONG_EXTREMES[3], LONG_EXTREMES[3]),
                                                   (LONG_EXTREMES[0], LONG_EXTREMES[3]))]   # 12..17
        out += [mk(F_MAIN, 2, 17), mk(F_MAIN, 5, 5)]                            # 18, 19: keys before a band key
        return np.array(out, po.RANGE_DTYPE)

    def range_count(self, si, ri):
        """PointField::count: keys of the leaf in the range (0 without the field)"""
        r = self.ranges[ri]
        f = int(r["field"])
        if f not in self.points[si]:
            return 0
        nb, _, packed, _ = self.points[si][f]
        keys = np.zeros(len(packed), np.uint64)
        for j in range(nb):
            keys = (keys << np.uint64(8)) | packed[:, j].astype(np.uint64)
        lo = int.from_bytes(bytes(r["lower"][:nb]), "big")
        hi = int.from_bytes(bytes(r["upper"][:nb]), "big")
        return int(np.count_nonzero((keys >= np.uint64(lo)) & (keys <= np.uint64(hi))))

    def split_bounds(self, rp=C_SPLIT_RP):
        """search.cu plan_batch for a range lead: R = ceil(count / rp), items cut on 128-doc block edges"""
        cnt = self.range_count(0, 7)
        Rn = max(1, min(-(-cnt // rp), 256, C_BLOCKS))
        return [(C_BLOCKS * r // Rn * 128, C_MAX_DOC if r + 1 == Rn else C_BLOCKS * (r + 1) // Rn * 128)
                for r in range(Rn)]

    @staticmethod
    def specs(n_ranges):
        ta, th, t1, t2 = C_T_ALL, C_T_HALF, C_T1, C_T2
        sp = [("bool", [(MUST, ta), (FILTER | R, ri)], 0) for ri in range(n_ranges)]          # range leads
        sp += [("bool", [(MUST, th), (FILTER | R, ri)], 0) for ri in (0, 2, 5, 6, 7)]
        sp += [("bool", [(MUST, t1), (FILTER | R, ri)], 0) for ri in (0, 7, 11, 17)]          # term leads, range probes
        sp += [("bool", [(FILTER | R, ri), (SHOULD, t1), (SHOULD, t2)], 0) for ri in (0, 4, 7, 11)]   # range-only ReqOpt
        sp += [("bool", [(MUST, th), (FILTER | R, 0), (SHOULD, t1), (SHOULD, t2)], 0),
               ("bool", [(MUST, ta), (MUST | R, 0), (MUST_NOT | R, 3)], 0),                   # MUST_NOT count 0: dropped
               ("bool", [(MUST, ta), (MUST | R, 7), (MUST_NOT | R, 8), (MUST_NOT, t1)], 0),
               ("bool", [(MUST, th), (MUST | R, 0), (MUST | R, 4)], 0),
               ("bool", [(MUST, C_T_EQ), (FILTER | R, 8)], 0), ("bool", [(MUST, C_T_EQ1), (FILTER | R, 8)], 0),
               ("bool", [(MUST, t2), (MUST_NOT | R, 0)], 0)]
        return sp


def lead_schedule(take, first_block, rend):
    """The range lead's block choice (eval_and_body 1'), replayed: per step the blocks taken, and per read of 32
    block-table entries the lane that took a step's 8th block -> (steps, lanes of 8th takes)"""
    steps, eighth = [], []
    cur = first_block
    while True:
        found = []
        while len(found) < 8 and cur < rend:
            idx = [l for l in range(32) if cur + l < rend and take[cur + l]]
            need = 8 - len(found)
            if len(idx) >= need:
                eighth.append(idx[need - 1])
                found += [cur + l for l in idx[:need]]
                cur += idx[need - 1] + 1
            else:
                found += [cur + l for l in idx]
                cur += min(32, rend - cur)
        if not found:
            return steps, eighth
        steps.append(found)
