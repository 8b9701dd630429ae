// orc_points — 1-D PointRangeQuery (src/core/search/query/point_range_query.rs of zhihu/rucene) inside the oracle's
// BooleanQuery.  TEST INFRASTRUCTURE: the parity reference of the device's range clauses (tests/points_oracle.py binds
// it).
//
// It includes oracle/oracle.cpp unchanged, so the index model, the BM25 weights and every term scorer, conjunction,
// disjunction, ReqOpt / ReqNot scorer and the TopDocs collector are the oracle's.  What is added:
//   PointRangeWeight::create_scorer  point_range_query.rs:502-556, restated literally:
//     None when the leaf has no point values of the field (:508-509, 560); bail on another bytes_per_dim (:517-522);
//     the all_docs_match shortcut (:524-543: every doc has a value and the range covers the field's min and max)
//     -> AllDocsIterator; else DocIdSetBuilder over every point the visitor accepts (visit_by_packed_value,
//     :626-640: lower <= packed <= upper as unsigned byte strings), sorted and deduplicated
//     (util/doc_id_set_builder.rs:224-250); ConstantScoreScorer::new(self.weight = 0f32, ..) (:466-485, 553).
//     In 1-D the BKD traversal only prunes cells wholly outside the range or takes cells wholly inside it, so
//     testing every point gives the same set.
//   Its cost() is DocIdSetBuilder's estimate, which depends on BKD internals; here it is the size of the set.  Any
//   estimate gives the same TopDocs: ConjunctionScorer sums lead1 + lead2 + others in cost order
//   (conjunction_scorer.rs:87-95), and adding the range's +0.0f is the identity for every x except -0.0f, which
//   becomes +0.0f wherever in the sum the addition happens.
//   BooleanWeight::create_scorer (boolean_query.rs:196-279) as oracle.cpp's create_scorer, with range clauses.
#include "../../oracle/oracle.cpp"

#include <map>

namespace {

constexpr int32_t kRangeBit = 0x100;  // orc_clause.occur: a range clause, term_id indexes the range array

struct orc_point_range {
    uint32_t field, bytes_per_dim;
    uint8_t lower[8], upper[8];
};

struct PointFieldData {  // PointValues of one field of one leaf
    uint32_t bytes_per_dim = 0;
    std::vector<int32_t> docs;
    std::vector<uint8_t> packed;  // docs.size() * bytes_per_dim
};

struct PointTable {
    std::map<std::pair<uint32_t, uint32_t>, PointFieldData> fields;  // (leaf, field)
};

// a sorted, deduplicated doc set, or every doc of the leaf (AllDocsIterator)
struct PointScorer : Scorer {
    std::vector<int32_t> docs;
    bool all = false;
    int32_t max_doc = 0, doc = -1;
    size_t idx = 0;
    int32_t doc_id() const override { return doc; }
    int32_t next() override {
        if (all) return doc = doc + 1 >= max_doc ? NO_MORE_DOCS : doc + 1;
        return doc = idx < docs.size() ? docs[idx++] : NO_MORE_DOCS;
    }
    int32_t advance(int32_t target) override {
        if (all) return doc = target >= max_doc ? NO_MORE_DOCS : target;
        while (idx < docs.size() && docs[idx] < target) idx++;
        return next();
    }
    size_t cost() const override { return all ? (size_t)max_doc : docs.size(); }
    float score() override { return 0.0f; }  // ConstantScoreScorer(weight = 0f32)
};

// PointRangeWeight::create_scorer (point_range_query.rs:502-556)
ScorerPtr range_scorer(const PointTable& pts, uint32_t seg_i, const SegmentData& seg, const orc_point_range& r) {
    const auto it = pts.fields.find({seg_i, r.field});
    if (it == pts.fields.end()) return nullptr;  // no point values / no FieldInfo: None
    const PointFieldData& f = it->second;
    const uint32_t n = r.bytes_per_dim;
    if (f.bytes_per_dim != n) throw Error("field was indexed with another bytes_per_dim");
    std::unique_ptr<PointScorer> s(new PointScorer());
    s->max_doc = seg.max_doc;
    const size_t n_points = f.docs.size();
    // all_docs_match: values.doc_count(field) == max_doc and the range covers the field's min and max packed value
    if (n_points) {
        std::vector<int32_t> distinct(f.docs);
        std::sort(distinct.begin(), distinct.end());
        distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
        if ((int32_t)distinct.size() == seg.max_doc) {
            const uint8_t* mn = &f.packed[0];
            const uint8_t* mx = &f.packed[0];
            for (size_t i = 1; i < n_points; i++) {
                const uint8_t* v = &f.packed[i * n];
                if (std::memcmp(v, mn, n) < 0) mn = v;
                if (std::memcmp(v, mx, n) > 0) mx = v;
            }
            if (!(std::memcmp(r.lower, mn, n) > 0 || std::memcmp(r.upper, mx, n) < 0)) {
                s->all = true;
                return ScorerPtr(s.release());
            }
        }
    }
    // build_matching_doc_set: the visitor over every point, then DocIdSetBuilder::build (sorted, deduplicated)
    for (size_t i = 0; i < n_points; i++) {
        const uint8_t* v = &f.packed[i * n];
        if (std::memcmp(v, r.lower, n) < 0) continue;
        if (std::memcmp(v, r.upper, n) > 0) continue;
        s->docs.push_back(f.docs[i]);
    }
    std::sort(s->docs.begin(), s->docs.end());
    s->docs.erase(std::unique(s->docs.begin(), s->docs.end()), s->docs.end());
    return ScorerPtr(s.release());
}

// oracle.cpp's create_scorer (BooleanWeight::create_scorer, boolean_query.rs:196-279) with range clauses
ScorerPtr create_scorer_r(const orc_index& ix, uint32_t seg_i, const orc_query& q, const orc_clause* clauses,
                          const Plan& plan, const PointTable& pts, const orc_point_range* ranges) {
    const SegmentData& seg = ix.segs[seg_i];
    auto is_range = [&](uint32_t ci) { return (clauses[q.clause_begin + ci].occur & kRangeBit) != 0; };
    auto occur_of = [&](uint32_t ci) { return clauses[q.clause_begin + ci].occur & ~kRangeBit; };
    auto sub_scorer = [&](uint32_t ci) -> ScorerPtr {
        const orc_clause& c = clauses[q.clause_begin + ci];
        if (is_range(ci)) return range_scorer(pts, seg_i, seg, ranges[c.term_id]);
        if (c.term_id >= seg.terms.size() || seg.terms[c.term_id].doc_freq <= 0) return nullptr;
        if (c.occur == ORC_FILTER) return ScorerPtr(new FilterTermScorer(seg, seg.terms[c.term_id]));
        return ScorerPtr(new TermScorer(seg, seg.terms[c.term_id], &plan.weights[ci]));
    };
    if (!q.is_boolean) return sub_scorer(0);
    if (q.is_boolean == 2) throw Error("DisjunctionMaxQuery with ranges is not modelled");
    int32_t msm = q.min_should_match;
    std::vector<uint32_t> musts, shoulds, filters, must_nots;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const int occ = occur_of(i);
        (occ == ORC_MUST ? musts : occ == ORC_SHOULD ? shoulds : occ == ORC_FILTER ? filters : must_nots).push_back(i);
    }
    if (msm <= 0) msm = musts.empty() ? 1 : 0;
    if (musts.size() + shoulds.size() + filters.size() + must_nots.size() == 0)
        throw Error("boolean query should at least contain one inner query!");
    // one positive clause: the clause itself; a lone FILTER is ConstantScoreQuery::with_boost(.., 0) (:66-75)
    if (must_nots.empty() && musts.size() + shoulds.size() + filters.size() == 1) {
        const uint32_t ci = musts.size() == 1 ? musts[0] : shoulds.size() == 1 ? shoulds[0] : filters[0];
        return sub_scorer(ci);
    }
    const bool match_all = musts.size() + shoulds.size() + filters.size() == 0;
    musts.insert(musts.end(), filters.begin(), filters.end());
    ScorerPtr must_scorer, should_scorer, must_not_scorer;
    if (match_all) must_scorer.reset(new AllDocsScorer(seg.max_doc));
    if (!musts.empty()) {
        std::vector<ScorerPtr> v;
        for (uint32_t ci : musts) {
            ScorerPtr s = sub_scorer(ci);
            if (!s) return nullptr;
            v.push_back(std::move(s));
        }
        if (v.size() > 1) must_scorer.reset(new ConjunctionScorer(std::move(v)));
        else must_scorer = std::move(v[0]);
    }
    {
        std::vector<ScorerPtr> v;
        for (uint32_t ci : shoulds)
            if (ScorerPtr s = sub_scorer(ci)) v.push_back(std::move(s));
        if (!v.empty()) should_scorer.reset(new DisjunctionSumScorer(std::move(v), true, msm));
    }
    {
        std::vector<ScorerPtr> v;
        for (uint32_t ci : must_nots)
            if (ScorerPtr s = sub_scorer(ci)) v.push_back(std::move(s));
        if (v.size() == 1) must_not_scorer = std::move(v[0]);
        else if (v.size() > 1) must_not_scorer.reset(new DisjunctionSumScorer(std::move(v), false, msm));
    }
    if (must_scorer) {
        if (should_scorer) {
            ScorerPtr ro(new ReqOptScorer(std::move(must_scorer), std::move(should_scorer)));
            if (must_not_scorer) return ScorerPtr(new ReqNotScorer(std::move(ro), std::move(must_not_scorer)));
            return ro;
        }
        if (must_not_scorer) return ScorerPtr(new ReqNotScorer(std::move(must_scorer), std::move(must_not_scorer)));
        return must_scorer;
    }
    if (should_scorer) {
        if (must_not_scorer) return ScorerPtr(new ReqNotScorer(std::move(should_scorer), std::move(must_not_scorer)));
        return should_scorer;
    }
    return nullptr;
}

// oracle.cpp's search_one with range clauses (searcher.rs:487-525; parallel_mode 1: search_parallel)
void search_one_r(const orc_index& ix, const PointTable& pts, const orc_point_range* ranges, const orc_query& q,
                  const orc_clause* clauses, uint32_t k, int parallel_mode, orc_hit* out, uint32_t* out_count,
                  uint64_t* out_total) {
    Plan plan;
    plan.weights.resize(q.n_clauses);
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        const orc_clause& c = clauses[q.clause_begin + i];
        if (!(c.occur & kRangeBit)) make_weight(ix, c.term_id, c.boost, plan.weights[i]);
    }
    TopDocsHeap main(k);
    for (uint32_t si = 0; si < ix.segs.size(); si++) {
        const SegmentData& seg = ix.segs[si];
        ScorerPtr scorer = create_scorer_r(ix, si, q, clauses, plan, pts, ranges);
        if (!scorer) continue;
        if (parallel_mode == 0) {
            bulk_score(*scorer, &seg, [&](int32_t doc, Scorer& s) { main.collect(doc + seg.doc_base, s.score()); });
        } else {
            TopDocsHeap leaf(k);
            bulk_score(*scorer, &seg, [&](int32_t doc, Scorer& s) { leaf.collect(doc + seg.doc_base, s.score()); });
            main.total_hits += leaf.total_hits;
            for (const orc_hit& h : leaf.data) main.add_doc(h.doc, h.score);
        }
    }
    *out_total = main.total_hits;
    std::vector<orc_hit> hits = main.top_docs();
    *out_count = (uint32_t)hits.size();
    for (size_t i = 0; i < hits.size(); i++) out[i] = hits[i];
}

}  // namespace

extern "C" {

void* orc_points_create(void) { return new PointTable(); }
void orc_points_destroy(void* p) { delete static_cast<PointTable*>(p); }

// every 1-D point of one field of leaf seg: docs[i] has the packed value packed[i * bytes_per_dim ..]
int orc_index_add_points(void* p, uint32_t seg, uint32_t field, uint32_t bytes_per_dim, const int32_t* docs,
                         const uint8_t* packed, size_t n) {
    ORC_TRY
    PointTable& pts = *static_cast<PointTable*>(p);
    if (bytes_per_dim == 0 || bytes_per_dim > 8) throw Error("bytes_per_dim must be 1..8");
    if (pts.fields.count({seg, field})) throw Error("field already added for this leaf");
    PointFieldData& f = pts.fields[{seg, field}];
    f.bytes_per_dim = bytes_per_dim;
    f.docs.assign(docs, docs + n);
    f.packed.assign(packed, packed + n * bytes_per_dim);
    return 0;
    ORC_CATCH(-1)
}

// PointRangeWeight::create_scorer's doc set in leaf seg: returns its size (written up to cap), -1 for None
int64_t orc_range_docs(orc_index* ix, void* p, uint32_t seg, const orc_point_range* r, int32_t* out, int64_t cap) {
    ORC_TRY
    ScorerPtr s = range_scorer(*static_cast<PointTable*>(p), seg, ix->segs.at(seg), *r);
    if (!s) return -1;
    int64_t n = 0;
    for (int32_t d = s->next(); d != NO_MORE_DOCS; d = s->next()) {
        if (n < cap) out[n] = d;
        n++;
    }
    return n;
    ORC_CATCH(-2)
}

int orc_search_batch_ranges(orc_index* ix, void* p, const orc_query* queries, uint32_t n_queries,
                            const orc_clause* clauses, const orc_point_range* ranges, uint32_t n_ranges, uint32_t k,
                            int parallel_mode, int n_threads, orc_hit* out_hits, uint32_t* out_counts,
                            uint64_t* out_total) {
    ORC_TRY
    if (ix->segs.empty()) throw Error("index has no segments");
    for (uint32_t i = 0; i < n_queries; i++)
        for (uint32_t c = 0; c < queries[i].n_clauses; c++) {
            const orc_clause& cl = clauses[queries[i].clause_begin + c];
            if ((cl.occur & kRangeBit) && cl.term_id >= n_ranges) throw Error("range index out of bounds");
        }
    const PointTable& pts = *static_cast<PointTable*>(p);
    parallel_for(n_queries, n_threads, [&](uint32_t i) {
        search_one_r(*ix, pts, ranges, queries[i], clauses, k, parallel_mode, out_hits + (size_t)i * k, out_counts + i,
                     out_total + i);
    });
    return 0;
    ORC_CATCH(-1)
}

}  // extern "C"
