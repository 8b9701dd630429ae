// Nested BooleanQuerys through the C++ host mirror (searcher.hpp): pure-SHOULD groups of TermQuerys as MUST, FILTER,
// SHOULD and MUST_NOT clauses on a synthetic leaf.  Prints each TopDocs as "total_hits doc:score_bits ..." so that the
// pytest driver can compare it with the oracle.
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
        const std::vector<QueryPtr> queries = {
            BooleanQuery::build({any("t1", "t2"), any("t3", "t4")}, {}, {}, {}, 0),              // +(a|b) +(c|d)
            BooleanQuery::build({term("t5"), any("t6", "t7")}, {}, {}, {term("t8")}, 0),        // +a +(b|c) -d
            BooleanQuery::build({any("t1", "t2")}, {term("t3")}, {}, {}, 0),                    // +(a|b) c
            BooleanQuery::build({}, {}, {any("t2", "t9")}, {term("t1")}, 0),                    // #(a|b) -c
            BooleanQuery::build({term("t1")}, {}, {}, {any("t2", "t3")}, 0),                    // +a -(b|c)
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
