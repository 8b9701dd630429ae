// PointRangeQuery through the C++ host mirror (searcher.hpp): two point fields on a synthetic leaf, then a bare
// range, ranges beside terms, a MUST_NOT range and a ReqOpt with a range.  Prints each TopDocs as
// "total_hits doc:score_bits ..." so that the pytest driver can compare it with the oracle.
//   "ts" (LongPoint): doc * 10 for docs not divisible by 7, a second value doc * 10 + 3 for docs divisible by 5
//   "f" (FloatPoint): (doc % 201 - 100) / 4, and -0.0 for docs with doc % 402 == 100 (the others there are +0.0)
#include <cstdio>
#include <cstring>

#include "../../rucene_b200/csrc/host/searcher.hpp"
#include "rucene_codec.h"

int main() {
    using namespace rucene;
    rc_synth_config cfg{0x5EED0001ull, 50000, 500, 1, 2};
    rc_segment* seg = rc_synth_segment(&cfg);
    if (!seg) { std::fprintf(stderr, "synth failed: %s\n", rc_last_error()); return 2; }
    LeafData leaf;
    leaf.doc_file = rc_segment_doc_file(seg, &leaf.doc_len);
    leaf.norms = rc_segment_norms(seg);
    leaf.terms = rc_segment_terms(seg, &leaf.n_terms);
    int64_t st[8];
    rc_segment_stats(seg, st);
    leaf.doc_count = st[0]; leaf.sum_total_term_freq = st[1]; leaf.sum_doc_freq = st[2]; leaf.max_doc = (int32_t)st[3];
    std::unordered_map<std::string, uint32_t> dict;
    for (uint32_t t = 0; t < leaf.n_terms; t++) dict["t" + std::to_string(t)] = t;
    auto term = [](const char* s) { return TermQuery::create(Term::create("body", s)); };
    std::vector<int32_t> ts_docs, f_docs;
    std::string ts_packed, f_packed;
    for (int32_t d = 0; d < leaf.max_doc; d++) {
        if (d % 7 != 0) {
            ts_docs.push_back(d);
            ts_packed += LongPoint::pack((int64_t)d * 10);
        }
        if (d % 5 == 0) {
            ts_docs.push_back(d);
            ts_packed += LongPoint::pack((int64_t)d * 10 + 3);
        }
        f_docs.push_back(d);
        f_packed += FloatPoint::pack(d % 402 == 100 ? -0.0f : (float)(d % 201 - 100) / 4.0f);
    }
    try {
        GpuIndexSearcher searcher({leaf}, "body", dict);
        searcher.upload_points(0, "ts", 8, ts_docs.data(), reinterpret_cast<const uint8_t*>(ts_packed.data()), ts_docs.size());
        searcher.upload_points(0, "f", 4, f_docs.data(), reinterpret_cast<const uint8_t*>(f_packed.data()), f_docs.size());
        const std::vector<QueryPtr> queries = {
            LongPoint::new_range_query("ts", 1000, 200003),
            BooleanQuery::build({term("t2")}, {}, {LongPoint::new_range_query("ts", 50000, 400000)}, {}, 0),
            BooleanQuery::build({term("t1"), FloatPoint::new_range_query("f", -0.0f, 5.0f)}, {}, {},
                                {LongPoint::new_exact_query("ts", 1000)}, 0),
            BooleanQuery::build({}, {term("t1"), term("t7")}, {FloatPoint::new_range_query("f", 0.0f, 25.0f)}, {}, 0),
            BooleanQuery::build({}, {}, {FloatPoint::new_exact_query("f", -0.0f)}, {}, 0),
        };
        for (const QueryPtr& q : queries) {
            TopDocsCollector collector(20);
            searcher.search(*q, collector);
            const TopDocs& top = collector.top_docs();
            std::printf("%llu", (unsigned long long)top.total_hits());
            for (const ScoreDoc& d : top.score_docs()) {
                uint32_t bits;
                std::memcpy(&bits, &d.score, 4);
                std::printf(" %d:%u", d.doc_id(), bits);
            }
            std::printf("\n");
        }
    } catch (const Error& e) {
        std::fprintf(stderr, "error %d: %s\n", e.code, e.what());
        return 1;
    }
    rc_segment_destroy(seg);
    return 0;
}
