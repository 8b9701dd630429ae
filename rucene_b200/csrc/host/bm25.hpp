// bm25.hpp — host side of BM25Similarity: what Query::create_weight computes once per
// (query term) before any posting is touched.  Product code (used by librucene_codec.so and
// by the C++ searcher mirror); independent of oracle/.
//
// Reference (paths relative to src/core/ of zhihu/rucene):
//   util/small_float.rs:16-36                         byte315 <-> f32
//   search/similarity/bm25_similarity.rs:33-43        NORM_TABLE
//   search/similarity/bm25_similarity.rs:72-83        avg_field_length
//   search/similarity/bm25_similarity.rs:90-92        encode_norm_value
//   search/similarity/bm25_similarity.rs:99-114       idf (f64 ln, cast to f32)
//   search/similarity/bm25_similarity.rs:161-165      cache[i] = k1*((1-b) + b*(NORM[i]/avgdl))
// Build with -ffp-contract=off: rustc never fuses a*b+c, and the cache must be bit-identical.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace rucene {

inline uint8_t float_to_byte315(float f) {
    int32_t bits;
    std::memcpy(&bits, &f, 4);
    const int32_t zero_point = (63 - 15) << 3;
    int32_t small = bits >> 21;
    if (small <= zero_point) return bits <= 0 ? 0 : 1;
    if (small >= zero_point + 0x100) return 255;
    return (uint8_t)(small - zero_point);
}

inline float byte315_to_float(uint8_t b) {
    if (b == 0) return 0.0f;
    uint32_t bits = ((uint32_t)b << 21) + ((uint32_t)(63 - 15) << 24);
    float f;
    std::memcpy(&f, &bits, 4);
    return f;
}

inline uint8_t encode_norm_value(float boost, int32_t field_length) {
    return float_to_byte315(boost / std::sqrt((float)field_length));
}

struct NormDecodeTable {
    float v[256];
    NormDecodeTable() {
        for (int i = 1; i < 256; i++) {
            float f = byte315_to_float((uint8_t)i);
            v[i] = 1.0f / (f * f);
        }
        v[0] = 1.0f / v[255];
    }
};

inline const NormDecodeTable& norm_decode_table() {
    static const NormDecodeTable t;
    return t;
}

inline float bm25_avg_field_length(int64_t sum_total_term_freq, int64_t doc_count, int64_t max_doc) {
    if (sum_total_term_freq <= 0) return 1.0f;
    if (doc_count == -1) doc_count = max_doc;
    return (float)((double)sum_total_term_freq / (double)doc_count);
}

inline float bm25_idf(int64_t doc_freq, int64_t doc_count) {
    double x = 1.0 + ((double)doc_count - (double)doc_freq + 0.5) / ((double)doc_freq + 0.5);
    return 0.0f + (float)std::log(x);
}

inline void bm25_norm_cache(float k1, float b, float avgdl, float* cache) {
    const NormDecodeTable& t = norm_decode_table();
    for (int i = 0; i < 256; i++) cache[i] = k1 * ((1.0f - b) + b * (t.v[i] / avgdl));
}

}  // namespace rucene
