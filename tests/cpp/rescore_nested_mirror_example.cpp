// QueryRescorer through the C++ host mirror (searcher.hpp) with rescoring queries that hold pure-SHOULD groups of
// TermQuerys: a first pass on the GPU, then each rescoring request (rescorer.rs:67-115,542-556) through
// rg_rescore_hits_nested.  Prints each rescored TopDocs as "total_hits doc:score_bits ..." so that the pytest driver
// can compare it with the oracle's rescorer.
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
    auto any = [&](const char* a, const char* b) { return BooleanQuery::build({}, {term(a), term(b)}, {}, {}, 0); };
    try {
        GpuIndexSearcher searcher({leaf}, "body", dict);
        QueryPtr first = BooleanQuery::build({}, {term("t1"), term("t2"), term("t3"), term("t5"), term("t9")}, {}, {}, 0);
        const std::vector<RescoreRequest> requests = {
            {BooleanQuery::build({any("t1", "t2"), any("t3", "t4")}, {}, {}, {}, 0), 1.0f, 2.0f, RescoreMode::Total, 15},
            {BooleanQuery::build({term("t5")}, {}, {}, {any("t6", "t7")}, 0), 0.5f, 1.0f, RescoreMode::Multiply, 40},
            {BooleanQuery::build({any("t1", "t2")}, {term("t3"), any("t9", "t8")}, {}, {}, 0), 1.0f, 1.0f,
             RescoreMode::Avg, 20},
        };
        for (const RescoreRequest& req : requests) {
            TopDocsCollector collector(20);
            searcher.search(*first, collector);
            TopDocs top = collector.top_docs();
            QueryRescorer().rescore(searcher, req, top);
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
