// codec.cpp — host-side write path of the Lucene50 postings format (DocsAndFreqs field),
// BM25 weight helpers and the synthetic Zipfian index generator (librucene_codec.so).
//
// Format references (paths relative to src/core/ of zhihu/rucene):
//   codec/postings/posting_writer.rs:289-361,457-474,477-589   term/doc/block emission
//   codec/postings/skip_writer.rs:187-290                       multi-level skip data
//   codec/postings/for_util.rs:150-185,374-478                  ForUtil table + write_block
//   util/packed/packed_simd.rs:81-108                           SIMD128 4-lane layout
//   util/packed/packed_misc.rs:474-531,2556-2582,2768-2777      COMPACT formats, BE encoders
//   codec/codec_util.rs:46-124                                  index header / footer
// Compile with -ffp-contract=off: the synthetic generator's math must be reproducible.
#include "rucene_codec.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../host/bm25.hpp"

namespace {

thread_local std::string g_err;
constexpr int kBlock = 128;
constexpr int kMaxSkipLevels = 10;

// ------------------------------------------------------------------ byte sink
struct Bytes {
    std::vector<uint8_t> v;
    size_t size() const { return v.size(); }
    void u8(uint8_t b) { v.push_back(b); }
    void raw(const void* p, size_t n) {
        const uint8_t* s = (const uint8_t*)p;
        v.insert(v.end(), s, s + n);
    }
    void be32(uint32_t x) {
        for (int s = 24; s >= 0; s -= 8) u8((uint8_t)(x >> s));
    }
    void be64(uint64_t x) {
        for (int s = 56; s >= 0; s -= 8) u8((uint8_t)(x >> s));
    }
    void vint(int32_t x) {  // store/io/data_output.rs write_vint: LE base-128
        uint32_t u = (uint32_t)x;
        while (u & ~0x7Fu) {
            u8((uint8_t)((u & 0x7F) | 0x80));
            u >>= 7;
        }
        u8((uint8_t)u);
    }
    void vlong(int64_t x) {
        uint64_t u = (uint64_t)x;
        while (u & ~0x7Full) {
            u8((uint8_t)((u & 0x7F) | 0x80));
            u >>= 7;
        }
        u8((uint8_t)u);
    }
    void clear() { v.clear(); }
};

// zlib CRC-32 (codec footer checksum), slicing-by-8
struct Crc32 {
    uint32_t t[8][256];
    Crc32() {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            t[0][i] = c;
        }
        for (uint32_t i = 0; i < 256; i++)
            for (int s = 1; s < 8; s++) t[s][i] = (t[s - 1][i] >> 8) ^ t[0][t[s - 1][i] & 0xFF];
    }
    uint32_t run(const uint8_t* p, size_t n) const {
        uint32_t c = 0xFFFFFFFFu;
        while (n >= 8) {
            uint32_t a, b;
            std::memcpy(&a, p, 4);
            std::memcpy(&b, p + 4, 4);
            a ^= c;
            c = t[7][a & 0xFF] ^ t[6][(a >> 8) & 0xFF] ^ t[5][(a >> 16) & 0xFF] ^ t[4][a >> 24] ^
                t[3][b & 0xFF] ^ t[2][(b >> 8) & 0xFF] ^ t[1][(b >> 16) & 0xFF] ^ t[0][b >> 24];
            p += 8;
            n -= 8;
        }
        while (n--) c = t[0][(c ^ *p++) & 0xFF] ^ (c >> 8);
        return c ^ 0xFFFFFFFFu;
    }
};
const Crc32 kCrc;

// ------------------------------------------------------------------ ForUtil write side
// COMPACT table (FormatAndBits::fastest(128, bpv, 0.0)): PackedSingleBlock for bpv 1,2,4,
// Packed (big-endian bit stream) otherwise; bits_per_value is never widened at ratio 0.
inline int compact_format_id(int bpv) { return (bpv == 1 || bpv == 2 || bpv == 4) ? 1 : 0; }

void forutil_table(int32_t out[32]) {
    for (int bpv = 1; bpv <= 32; bpv++) out[bpv - 1] = (compact_format_id(bpv) << 5) | (bpv - 1);
}

// SIMD128 layout: value n -> lane n&3, slot n>>2; each lane is an LSB-first stream of b-bit
// fields over the lane's little-endian 32-bit words, vector j of the payload = words j of the
// four lanes.
void pack_simd128(const uint32_t* v, int b, uint8_t* out) {
    if (b == 32) {
        std::memcpy(out, v, 512);
        return;
    }
    uint32_t words[32 * 4];
    std::memset(words, 0, sizeof(uint32_t) * (size_t)b * 4);
    for (int n = 0; n < kBlock; n++) {
        int lane = n & 3, slot = n >> 2;
        int bit = slot * b;
        int w = bit >> 5, s = bit & 31;
        uint64_t val = (uint64_t)v[n] << s;
        words[w * 4 + lane] |= (uint32_t)val;
        if (s + b > 32) words[(w + 1) * 4 + lane] |= (uint32_t)(val >> 32);
    }
    std::memcpy(out, words, (size_t)b * 16);
}

// Packed: one MSB-first big-endian bit stream, value n at bit n*b.
void pack_be_stream(const uint32_t* v, int b, uint8_t* out) {
    std::memset(out, 0, (size_t)b * 16);
    for (int n = 0; n < kBlock; n++) {
        uint64_t bit = (uint64_t)n * b;
        for (int k = b - 1; k >= 0; k--, bit++)
            if ((v[n] >> k) & 1) out[bit >> 3] |= (uint8_t)(0x80u >> (bit & 7));
    }
}

// PackedSingleBlock: 64/b values per big-endian 64-bit long, value i of a long at bits [i*b, i*b+b).
void pack_single_block(const uint32_t* v, int b, uint8_t* out) {
    int per = 64 / b;
    int longs = (kBlock + per - 1) / per;
    for (int L = 0; L < longs; L++) {
        uint64_t x = 0;
        for (int i = 0; i < per && L * per + i < kBlock; i++) x |= (uint64_t)v[L * per + i] << (i * b);
        for (int k = 0; k < 8; k++) out[L * 8 + k] = (uint8_t)(x >> (56 - 8 * k));
    }
}

// ForUtil::write_block: all-equal -> code 0 + vint; else code = bits_required(OR) + payload.
int write_block(const int32_t* data, int doc_version, uint8_t* out) {
    bool all_equal = true;
    uint32_t orv = 0;
    for (int i = 0; i < kBlock; i++) {
        all_equal &= data[i] == data[0];
        orv |= (uint32_t)data[i];
    }
    if (all_equal) {
        Bytes tmp;
        tmp.u8(0);
        tmp.vint(data[0]);
        std::memcpy(out, tmp.v.data(), tmp.size());
        return (int)tmp.size();
    }
    int b = 32 - __builtin_clz(orv);
    out[0] = (uint8_t)b;
    const uint32_t* u = (const uint32_t*)data;
    if (doc_version > 0) pack_simd128(u, b, out + 1);
    else if (compact_format_id(b)) pack_single_block(u, b, out + 1);
    else pack_be_stream(u, b, out + 1);
    return 1 + 16 * b;
}

// ---- the reference's other doc-block encodings (dormant in the open-source writer:
// EfWriterMeta.use_ef is never set, posting_writer.rs:46; production indexes carry them).
// EfWriterMeta, posting_writer.rs:33-57; filled at :335 (ef_upper_doc) and :472 (ef_base_doc).
struct EfWriterMeta {
    int32_t ef_base_doc = -1, ef_upper_doc = 0;
    bool use_ef = false, with_pf = true;
};
inline int64_t ushr64(int64_t x, int n) { return (int64_t)((uint64_t)x >> n); }
inline int64_t num_longs_for_bits(int64_t n) { return ushr64(n + 63, 6); }  // elias_fano_encoder.rs:308-311
// EliasFanoEncoder::pack_value, elias_fano_encoder.rs:334-345 (the spill word is assigned, not or-ed)
inline void ef_pack_value(int64_t value, std::vector<int64_t>& a, int num_bits, int64_t pack_index) {
    if (num_bits == 0) return;
    int64_t bit_pos = (int64_t)num_bits * pack_index;
    size_t index = (size_t)ushr64(bit_pos, 6);
    int at = (int)(bit_pos & 63);
    a[index] |= (int64_t)((uint64_t)value << at);
    if (at + num_bits > 64) a[index + 1] = ushr64(value, 64 - at);
}
// EliasFanoEncoder::new + encode_next for one block, elias_fano_encoder.rs:46-146,214-253
struct EfEncoder {
    int64_t num_values, upper_bound;
    int num_low_bits = 0;
    int64_t lower_bits_mask;
    std::vector<int64_t> upper, lower, index;
    int64_t num_encoded = 0, last_encoded = 0, num_index_entries, index_interval = 256, current_entry_index = 0;
    int n_index_entry_bits;
    EfEncoder(int64_t nv, int64_t ub) : num_values(nv), upper_bound(ub) {
        if (nv > 0 && ub < 0) throw std::runtime_error("upper_bound should not be negative");
        int64_t fac = ub / nv;
        if (fac > 0) num_low_bits = 63 - __builtin_clzll((uint64_t)fac);
        lower_bits_mask = ushr64(INT64_MAX, 63 - num_low_bits);
        lower.assign((size_t)num_longs_for_bits(nv * num_low_bits), 0);
        int64_t high_clear = ushr64(ub > 0 ? ub : 0, num_low_bits);
        if (high_clear > 2 * nv) throw std::runtime_error("ef: num_high_bits_clear > 2 * num_values");
        upper.assign((size_t)num_longs_for_bits(high_clear + nv), 0);
        int64_t max_high_value = ushr64(ub, num_low_bits);
        int64_t n_entries = max_high_value / index_interval;
        num_index_entries = n_entries >= 0 ? n_entries : 0;
        int64_t max_index_entry = max_high_value + nv - 1;
        n_index_entry_bits = max_index_entry <= 0 ? 0 : 64 - __builtin_clzll((uint64_t)max_index_entry);
        index.assign((size_t)num_longs_for_bits(num_index_entries * n_index_entry_bits), 0);
    }
    int encode_size() const { return (int)((upper.size() + lower.size() + index.size()) << 3); }  // :207-212
    void encode_next(int64_t x) {
        if (num_encoded >= num_values) throw std::runtime_error("encode_next called too often");
        if (last_encoded > x) throw std::runtime_error("ef: value smaller than previous");
        if (x > upper_bound) throw std::runtime_error("ef: value larger than upper bound");
        int64_t high_value = ushr64(x, num_low_bits);
        int64_t bit = num_encoded + high_value;  // encode_upper_bits :313-317
        upper[(size_t)ushr64(bit, 6)] |= (int64_t)((uint64_t)1 << (bit & 63));
        ef_pack_value(x & lower_bits_mask, lower, num_low_bits, num_encoded);
        last_encoded = x;
        int64_t index_value = (current_entry_index + 1) * index_interval;
        while (index_value <= high_value) {
            ef_pack_value(index_value + num_encoded, index, n_index_entry_bits, current_entry_index);
            current_entry_index++;
            index_value += index_interval;
        }
        num_encoded++;
    }
};
inline void raw_longs(Bytes& o, const std::vector<int64_t>& a) {  // write_data :347-355: raw LE memory
    for (int64_t x : a)
        for (int k = 0; k < 8; k++) o.u8((uint8_t)((uint64_t)x >> (8 * k)));
}
// ForUtil::write_block with an EfWriterMeta, for_util.rs:396-478 (doc-delta blocks only).
// Returns false when the block falls through to the PF encoding.
bool write_block_other(const int32_t* data, int pf_bits, const EfWriterMeta& meta, Bytes& o) {
    if (!meta.use_ef) return false;
    const int encoded_size = 16 * pf_bits;  // encoded_sizes[num_bits - 1]
    EfEncoder ef(kBlock, (int64_t)(meta.ef_upper_doc - meta.ef_base_doc - 1));
    if (ef.encode_size() > 4 * kBlock) return false;  // MAX_ENCODED_SIZE :33
    int32_t doc = meta.ef_base_doc < 0 ? 0 : meta.ef_base_doc;
    int32_t min_doc = INT32_MAX, max_doc = 0;
    for (int i = 0; i < kBlock; i++) {
        doc += data[i];
        max_doc = std::max(max_doc, doc);
        min_doc = std::min(min_doc, doc);
        ef.encode_next((int64_t)(doc - meta.ef_base_doc - 1));
    }
    // FixedBitSet::resize / encode_size, bit_set.rs:193-204,480-484
    const size_t num_words = (size_t)((((max_doc - min_doc + 1) - 1) >> 6) + 1);
    if ((int)(num_words << 3) <= encoded_size) {
        std::vector<int64_t> bits(num_words, 0);
        doc = meta.ef_base_doc < 0 ? 0 : meta.ef_base_doc;
        for (int i = 0; i < kBlock; i++) {
            doc += data[i];
            const int32_t b = doc - min_doc;
            bits[(size_t)b >> 6] |= (int64_t)((uint64_t)1 << (b & 63));
        }
        o.u8(2u << 6);  // EncodeType::BITSET
        o.vint(min_doc);
        o.u8((uint8_t)num_words);
        raw_longs(o, bits);
        return true;
    }
    if (!meta.with_pf || ef.encode_size() <= encoded_size) {  // EliasFanoEncoder::serialize :255-262
        o.u8(1u << 6);  // EncodeType::EF
        o.vlong(ef.upper_bound);
        raw_longs(o, ef.upper);
        raw_longs(o, ef.lower);
        raw_longs(o, ef.index);
        return true;
    }
    return false;
}

void write_index_header(Bytes& o, int version, const uint8_t id[16], const char* suffix) {
    static const char* codec = "Lucene50PostingsWriterDoc";
    o.be32(0x3FD76C17u);
    o.vint((int32_t)std::strlen(codec));
    o.raw(codec, std::strlen(codec));
    o.be32((uint32_t)version);
    o.raw(id, 16);
    size_t sl = std::strlen(suffix);
    o.u8((uint8_t)sl);
    o.raw(suffix, sl);
    // ForUtil::with_output: PackedInts version 2 then the 32 format codes
    o.vint(2);
    int32_t tbl[32];
    forutil_table(tbl);
    for (int i = 0; i < 32; i++) o.vint(tbl[i]);
}

void write_footer(Bytes& o) {
    o.be32(~0x3FD76C17u);
    o.be32(0);
    uint32_t crc = kCrc.run(o.v.data(), o.size());
    o.be64((uint64_t)crc);
}

// ------------------------------------------------------------------ skip writer
struct SkipWriter {
    int levels = 1;
    Bytes buf[kMaxSkipLevels];
    int32_t last_doc[kMaxSkipLevels];
    int64_t last_fp[kMaxSkipLevels];
    bool initialized = false;
    int64_t term_fp = 0;

    void configure(int32_t max_doc) {
        levels = 1;
        if (max_doc > kBlock) {
            int64_t x = max_doc / kBlock;
            while (x >= 8) {
                x /= 8;
                levels++;
            }
        }
        levels = std::min(levels, kMaxSkipLevels);
    }
    void reset(int64_t doc_fp) {
        term_fp = doc_fp;
        initialized = false;
    }
    void buffer(int32_t doc, uint32_t num_docs, int64_t fp) {
        if (!initialized) {
            for (int i = 0; i < kMaxSkipLevels; i++) {
                buf[i].clear();
                last_doc[i] = 0;
                last_fp[i] = term_fp;
            }
            initialized = true;
        }
        int n = 1;
        uint32_t d = num_docs / kBlock;
        while (d % 8 == 0 && n < levels) {
            n++;
            d /= 8;
        }
        int64_t child = 0;
        for (int lv = 0; lv < n; lv++) {
            buf[lv].vint(doc - last_doc[lv]);
            last_doc[lv] = doc;
            buf[lv].vlong(fp - last_fp[lv]);
            last_fp[lv] = fp;
            int64_t here = (int64_t)buf[lv].size();
            if (lv != 0) buf[lv].vlong(child);
            child = here;
        }
    }
    // returns the file position where the skip data starts
    int64_t flush(Bytes& out) {
        int64_t at = (int64_t)out.size();
        if (!initialized) return at;
        for (int lv = levels - 1; lv >= 1; lv--) {
            if (buf[lv].size() > 0) {
                out.vlong((int64_t)buf[lv].size());
                out.raw(buf[lv].v.data(), buf[lv].size());
            }
        }
        out.raw(buf[0].v.data(), buf[0].size());
        return at;
    }
};

// ------------------------------------------------------------------ postings writer
struct PostingsWriter {
    Bytes out;
    int version = 1;
    SkipWriter skip;
    int32_t dbuf[kBlock], fbuf[kBlock];
    int upto = 0;
    int32_t last_doc = 0, last_block_doc = -1;
    EfWriterMeta ef_meta;
    uint64_t ef_blocks = 0, bitset_blocks = 0;
    int32_t doc_count = 0;
    int64_t term_fp = 0;
    int64_t ttf = 0;
    uint64_t blocks_written = 0;

    void start_term() {
        term_fp = (int64_t)out.size();
        last_doc = 0;
        last_block_doc = -1;
        doc_count = 0;
        upto = 0;
        ttf = 0;
        skip.reset(term_fp);
        ef_meta.ef_base_doc = -1;  // EfWriterMeta::reset :52-56
        ef_meta.ef_upper_doc = 0;
    }
    void add_doc(int32_t doc, int32_t freq) {
        if (last_block_doc != -1 && upto == 0)
            skip.buffer(last_block_doc, (uint32_t)doc_count, (int64_t)out.size());
        int32_t delta = doc - last_doc;
        if (doc < 0 || (doc_count > 0 && delta <= 0)) throw std::runtime_error("docs out of order");
        if (freq < 1) throw std::runtime_error("freq must be >= 1");
        dbuf[upto] = delta;
        fbuf[upto] = freq;
        upto++;
        doc_count++;
        ttf += freq;
        if (upto == kBlock) {
            uint8_t tmp[1 + 512];
            ef_meta.ef_upper_doc = doc;  // :335
            bool other = false;
            if (ef_meta.use_ef) {
                bool all_equal = true;
                uint32_t orv = 0;
                for (int i = 0; i < kBlock; i++) {
                    all_equal &= dbuf[i] == dbuf[0];
                    orv |= (uint32_t)dbuf[i];
                }
                if (!all_equal) {  // the all-equal shortcut comes first (:402-405)
                    const size_t before = out.size();
                    other = write_block_other(dbuf, 32 - __builtin_clz(orv), ef_meta, out);
                    if (other) (out.v[before] >> 6) == 1 ? ef_blocks++ : bitset_blocks++;
                }
            }
            int n = 0;
            if (!other) {
                n = write_block(dbuf, version, tmp);
                out.raw(tmp, (size_t)n);
            }
            n = write_block(fbuf, version, tmp);
            out.raw(tmp, (size_t)n);
            blocks_written++;
        }
        last_doc = doc;
        if (upto == kBlock) {  // finish_doc
            last_block_doc = last_doc;
            upto = 0;
            ef_meta.ef_base_doc = last_block_doc;  // :472
        }
    }
    void finish_term(rg_term_state* st) {
        if (doc_count <= 0) throw std::runtime_error("term without postings");
        int32_t singleton = -1;
        if (doc_count == 1) {
            singleton = dbuf[0];
        } else {
            for (int i = 0; i < upto; i++) {
                if (fbuf[i] == 1) {
                    out.vint((int32_t)(((uint32_t)dbuf[i] << 1) | 1u));
                } else {
                    out.vint((int32_t)((uint32_t)dbuf[i] << 1));
                    out.vint(fbuf[i]);
                }
            }
        }
        int64_t skip_offset = -1;
        if (doc_count > kBlock) skip_offset = skip.flush(out) - term_fp;
        st->doc_freq = doc_count;
        st->singleton_doc_id = singleton;
        st->total_term_freq = ttf;
        st->doc_start_fp = term_fp;
        st->skip_offset = skip_offset;
        upto = 0;
        last_doc = 0;
        doc_count = 0;
    }
};

// ------------------------------------------------------------------ deterministic math
// Series built from IEEE +,*,/ only (no libm), so every host produces the same index bytes.
double det_log(double x) {  // x > 0
    int e;
    double m = std::frexp(x, &e);  // m in [0.5,1), exact
    m *= 2.0;
    e -= 1;
    if (m > 1.4142135623730951) {
        m *= 0.5;
        e += 1;
    }
    double t = (m - 1.0) / (m + 1.0);
    double t2 = t * t;
    double term = t, sum = 0.0;
    for (int k = 1; k <= 27; k += 2) {
        sum += term / (double)k;
        term *= t2;
    }
    return (double)e * 0.6931471805599453 + 2.0 * sum;
}
double det_exp(double x) {
    double kf = std::floor(x / 0.6931471805599453 + 0.5);
    double r = x - kf * 0.6931471805599453;
    double term = 1.0, sum = 1.0;
    for (int i = 1; i <= 18; i++) {
        term *= r / (double)i;
        sum += term;
    }
    return std::ldexp(sum, (int)kf);
}

inline uint64_t splitmix(uint64_t& s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
inline uint64_t mix64(uint64_t x) {
    uint64_t s = x;
    return splitmix(s);
}

int hw_threads() {
    unsigned n = std::thread::hardware_concurrency();
    return n ? (int)n : 1;
}

template <class F>
void parallel_tasks(size_t n, int n_threads, F&& f) {
    if (n_threads <= 1 || n <= 1) {
        for (size_t i = 0; i < n; i++) f(i);
        return;
    }
    std::atomic<size_t> next{0};
    std::atomic<bool> failed{false};
    std::string err;
    std::vector<std::thread> ts;
    int nt = (int)std::min<size_t>((size_t)n_threads, n);
    for (int t = 0; t < nt; t++)
        ts.emplace_back([&] {
            try {
                for (;;) {
                    size_t i = next.fetch_add(1);
                    if (i >= n || failed.load()) break;
                    f(i);
                }
            } catch (const std::exception& e) {
                if (!failed.exchange(true)) err = e.what();
            }
        });
    for (auto& t : ts) t.join();
    if (failed.load()) throw std::runtime_error(err);
}

}  // namespace

struct rc_writer {
    PostingsWriter pw;
    bool finished = false;
};

struct rc_segment {
    std::vector<uint8_t> doc_file;
    std::vector<uint8_t> norms;
    std::vector<rg_term_state> terms;
    int64_t doc_count = 0, sum_ttf = 0, sum_df = 0, max_doc = 0, blocks = 0;
};

struct rc_blocks {
    std::vector<uint8_t> stream;
    std::vector<uint64_t> offsets;
    std::vector<int32_t> values;
};

#define RC_TRY try {
#define RC_CATCH(ret)                 \
    }                                 \
    catch (const std::exception& e) { \
        g_err = e.what();             \
        return ret;                   \
    }

extern "C" {

const char* rc_last_error(void) { return g_err.c_str(); }
int rc_hardware_threads(void) { return hw_threads(); }

rc_writer* rc_writer_create(int doc_version, int32_t max_doc, const uint8_t segment_id[16],
                            const char* suffix) {
    RC_TRY
    if (doc_version < 0 || doc_version > 1) throw std::runtime_error("doc_version must be 0 or 1");
    rc_writer* w = new rc_writer();
    w->pw.version = doc_version;
    w->pw.skip.configure(max_doc);
    write_index_header(w->pw.out, doc_version, segment_id, suffix ? suffix : "");
    return w;
    RC_CATCH(nullptr)
}
int rc_writer_add_term(rc_writer* w, const int32_t* docs, const int32_t* freqs, int32_t n,
                       rg_term_state* out_state) {
    RC_TRY
    if (w->finished) throw std::runtime_error("writer already finished");
    if (n <= 0) throw std::runtime_error("term needs at least one posting");
    w->pw.start_term();
    for (int32_t i = 0; i < n; i++) w->pw.add_doc(docs[i], freqs[i]);
    w->pw.finish_term(out_state);
    return 0;
    RC_CATCH(-1)
}
// test hooks for the reference's own EliasFanoEncoder unit tests (elias_fano_encoder.rs:398-448)
int64_t rc_ef_num_longs_for_bits(int64_t n) { return num_longs_for_bits(n); }
void rc_ef_pack_value(int64_t value, int64_t* longs, int n_longs, int num_bits, int64_t pack_index) {
    std::vector<int64_t> a(longs, longs + n_longs);
    ef_pack_value(value, a, num_bits, pack_index);
    std::copy(a.begin(), a.end(), longs);
}
int rc_ef_encode(const int64_t* values, int64_t n, int64_t upper_bound, int64_t* out_longs, int cap,
                 int32_t out_geom[4]) {
    RC_TRY
    EfEncoder ef(n, upper_bound);
    for (int64_t i = 0; i < n; i++) ef.encode_next(values[i]);
    out_geom[0] = ef.num_low_bits;
    out_geom[1] = (int32_t)ef.upper.size();
    out_geom[2] = (int32_t)ef.lower.size();
    out_geom[3] = (int32_t)ef.index.size();
    if ((int)(ef.upper.size() + ef.lower.size() + ef.index.size()) > cap) throw std::runtime_error("rc_ef_encode: cap");
    int64_t* o = out_longs;
    o = std::copy(ef.upper.begin(), ef.upper.end(), o);
    o = std::copy(ef.lower.begin(), ef.lower.end(), o);
    std::copy(ef.index.begin(), ef.index.end(), o);
    return 0;
    RC_CATCH(-1)
}
int rc_writer_set_ef(rc_writer* w, int use_ef, int with_pf) {
    RC_TRY
    w->pw.ef_meta.use_ef = use_ef != 0;
    w->pw.ef_meta.with_pf = with_pf != 0;
    return 0;
    RC_CATCH(-1)
}
void rc_writer_block_counts(rc_writer* w, uint64_t out[3]) {
    out[0] = w->pw.blocks_written;
    out[1] = w->pw.ef_blocks;
    out[2] = w->pw.bitset_blocks;
}
int rc_writer_finish(rc_writer* w) {
    RC_TRY
    if (!w->finished) {
        write_footer(w->pw.out);
        w->finished = true;
    }
    return 0;
    RC_CATCH(-1)
}
const uint8_t* rc_writer_data(rc_writer* w, size_t* len) {
    *len = w->pw.out.size();
    return w->pw.out.v.data();
}
void rc_writer_forutil_table(rc_writer*, int32_t out[32]) { forutil_table(out); }
void rc_writer_destroy(rc_writer* w) { delete w; }

int rc_forutil_write_block(const int32_t data[128], int doc_version, uint8_t* out) {
    return write_block(data, doc_version, out);
}

uint8_t rc_float_to_byte315(float f) { return rucene::float_to_byte315(f); }
float rc_byte315_to_float(uint8_t b) { return rucene::byte315_to_float(b); }
uint8_t rc_encode_norm_value(float boost, int32_t len) { return rucene::encode_norm_value(boost, len); }
float rc_bm25_idf(int64_t df, int64_t dc) { return rucene::bm25_idf(df, dc); }
float rc_bm25_avg_field_length(int64_t s, int64_t dc, int64_t md) {
    return rucene::bm25_avg_field_length(s, dc, md);
}
void rc_bm25_norm_cache(float k1, float b, float avgdl, float out_cache[256]) {
    rucene::bm25_norm_cache(k1, b, avgdl, out_cache);
}

// Synthetic segment: term t (rank r=t+1) targets df = max(1, N/(r+1)); docids by geometric gap
// sampling with p = df/N; freq = 1 + min(leading-zero count of a random word, 254) (P(1)=1/2);
// doc length ~ lognormal(ln 200, 0.5) -> norm byte via encode_norm_value.
rc_segment* rc_synth_segment(const rc_synth_config* cfg) {
    RC_TRY
    if (cfg->max_doc <= 0 || cfg->n_terms == 0) throw std::runtime_error("bad synth config");
    const int64_t N = cfg->max_doc;
    const uint32_t V = cfg->n_terms;
    int nt = cfg->n_threads > 0 ? cfg->n_threads : hw_threads();
    std::unique_ptr<rc_segment> seg(new rc_segment());
    seg->max_doc = N;
    seg->terms.resize(V);
    seg->norms.resize((size_t)N);

    // norms
    {
        const size_t chunk = 1 << 16;
        size_t n_chunks = ((size_t)N + chunk - 1) / chunk;
        parallel_tasks(n_chunks, nt, [&](size_t c) {
            size_t end = std::min((size_t)N, (c + 1) * chunk);
            for (size_t d = c * chunk; d < end; d++) {
                uint64_t h = mix64(cfg->seed ^ 0xD0C1E57ull ^ ((uint64_t)d * 0x9E3779B97F4A7C15ull));
                double u = 0.0;
                for (int k = 0; k < 4; k++) u += (double)((h >> (16 * k)) & 0xFFFF) / 65536.0;
                double z = (u - 2.0) * 1.7320508075688772;  // ~N(0,1)
                double len = std::floor(200.0 * det_exp(0.5 * z) + 0.5);
                if (len < 1.0) len = 1.0;
                if (len > 10000.0) len = 10000.0;
                seg->norms[d] = rucene::encode_norm_value(1.0f, (int32_t)len);
            }
        });
    }

    // term groups of roughly equal expected postings
    struct Group {
        uint32_t t0, t1;
        Bytes bytes;
        int64_t ttf = 0, df = 0, blocks = 0;
    };
    std::vector<Group> groups;
    {
        const int64_t target = 1 << 21;
        int64_t acc = 0;
        uint32_t start = 0;
        for (uint32_t t = 0; t < V; t++) {
            acc += std::max<int64_t>(1, N / ((int64_t)t + 2));
            if (acc >= target || t + 1 == V) {
                Group g;
                g.t0 = start;
                g.t1 = t + 1;
                groups.push_back(std::move(g));
                start = t + 1;
                acc = 0;
            }
        }
    }
    parallel_tasks(groups.size(), nt, [&](size_t gi) {
        Group& g = groups[gi];
        PostingsWriter pw;
        pw.version = cfg->doc_version;
        pw.skip.configure((int32_t)N);
        for (uint32_t t = g.t0; t < g.t1; t++) {
            int64_t df_target = std::max<int64_t>(1, N / ((int64_t)t + 2));
            double p = (double)df_target / (double)N;
            double log1mp = det_log(1.0 - p);
            uint64_t rs = cfg->seed ^ ((uint64_t)(t + 1) * 0xD1B54A32D192ED03ull);
            pw.start_term();
            int64_t doc = -1;
            int32_t n = 0;
            for (;;) {
                uint64_t r = splitmix(rs);
                double u = (double)((r >> 11) + 1) / 9007199254740992.0;  // (0,1]
                double gap = 1.0 + std::floor(det_log(u) / log1mp);
                if (!(gap < (double)N + 1.0)) break;
                doc += (int64_t)gap;
                if (doc >= N) break;
                uint64_t fr = splitmix(rs);
                int32_t freq = 1 + std::min(fr ? __builtin_clzll(fr) : 64, 254);
                pw.add_doc((int32_t)doc, freq);
                n++;
            }
            rg_term_state st{};
            if (n == 0) {
                st.doc_freq = 0;
                st.singleton_doc_id = -1;
                st.total_term_freq = 0;
                st.doc_start_fp = (int64_t)pw.out.size();
                st.skip_offset = -1;
            } else {
                pw.finish_term(&st);
                g.ttf += st.total_term_freq;
                g.df += st.doc_freq;
            }
            seg->terms[t] = st;
        }
        g.blocks = (int64_t)pw.blocks_written;
        g.bytes = std::move(pw.out);
    });

    // stitch: header | group regions | footer; term regions are position independent apart
    // from doc_start_fp (skip data stores only deltas)
    Bytes file;
    uint8_t id[16];
    for (int i = 0; i < 16; i++) id[i] = (uint8_t)(mix64(cfg->seed + (uint64_t)i) & 0xFF);
    write_index_header(file, cfg->doc_version, id, "");
    size_t total = file.size();
    for (auto& g : groups) total += g.bytes.size();
    file.v.reserve(total + 16);
    for (auto& g : groups) {
        int64_t base = (int64_t)file.size();
        for (uint32_t t = g.t0; t < g.t1; t++) seg->terms[t].doc_start_fp += base;
        file.raw(g.bytes.v.data(), g.bytes.size());
        seg->sum_ttf += g.ttf;
        seg->sum_df += g.df;
        seg->blocks += g.blocks;
        std::vector<uint8_t>().swap(g.bytes.v);
    }
    write_footer(file);
    seg->doc_file = std::move(file.v);
    seg->doc_count = N;
    return seg.release();
    RC_CATCH(nullptr)
}
void rc_segment_destroy(rc_segment* s) { delete s; }
const uint8_t* rc_segment_doc_file(const rc_segment* s, size_t* len) {
    *len = s->doc_file.size();
    return s->doc_file.data();
}
const uint8_t* rc_segment_norms(const rc_segment* s) { return s->norms.data(); }
const rg_term_state* rc_segment_terms(const rc_segment* s, uint32_t* n) {
    *n = (uint32_t)s->terms.size();
    return s->terms.data();
}
void rc_segment_stats(const rc_segment* s, int64_t out[8]) {
    out[0] = s->doc_count;
    out[1] = s->sum_ttf;
    out[2] = s->sum_df;
    out[3] = s->max_doc;
    out[4] = s->blocks;
    out[5] = s->sum_df;
    out[6] = out[7] = 0;
}
void rc_segment_forutil_table(const rc_segment*, int32_t out[32]) { forutil_table(out); }

rc_blocks* rc_synth_blocks(uint64_t seed, uint32_t n_blocks, int mode, int param,
                           int doc_version) {
    RC_TRY
    if (mode == 1 && (param < 0 || param > 32)) throw std::runtime_error("width must be 0..32");
    std::unique_ptr<rc_blocks> b(new rc_blocks());
    b->offsets.resize(n_blocks);
    b->values.resize((size_t)n_blocks * kBlock);
    int nt = hw_threads();
    const uint32_t chunk = 8192;
    uint32_t n_chunks = (n_blocks + chunk - 1) / chunk;
    std::vector<Bytes> parts(n_chunks);
    std::vector<std::vector<uint32_t>> rel(n_chunks);
    parallel_tasks(n_chunks, nt, [&](size_t c) {
        uint32_t end = std::min(n_blocks, (uint32_t)(c + 1) * chunk);
        uint8_t tmp[1 + 512];
        for (uint32_t i = (uint32_t)c * chunk; i < end; i++) {
            uint64_t rs = seed ^ ((uint64_t)(i + 1) * 0xA0761D6478BD642Full);
            int width = mode == 0 ? 1 + (int)(splitmix(rs) % 32) : param;
            int32_t* v = &b->values[(size_t)i * kBlock];
            if (width == 0) {
                int32_t x = (int32_t)(splitmix(rs) & 0x7FFFFFFF);
                for (int k = 0; k < kBlock; k++) v[k] = x;
            } else {
                uint32_t mask = width == 32 ? 0xFFFFFFFFu : ((1u << width) - 1);
                for (int k = 0; k < kBlock; k++) v[k] = (int32_t)((uint32_t)splitmix(rs) & mask);
                int pos = (int)(splitmix(rs) % kBlock);
                v[pos] = (int32_t)((uint32_t)v[pos] | (1u << (width - 1)));  // force the top bit
                {  // never all-equal (all-equal blocks use code 0)
                    int other = (pos + 1) % kBlock;
                    if (v[other] == v[pos]) v[other] = (int32_t)((uint32_t)v[pos] ^ 1u);
                }
            }
            rel[c].push_back((uint32_t)parts[c].size());
            int n = write_block(v, doc_version, tmp);
            parts[c].raw(tmp, (size_t)n);
        }
    });
    size_t total = 0;
    for (auto& p : parts) total += p.size();
    b->stream.reserve(total + 64);
    for (uint32_t c = 0; c < n_chunks; c++) {
        uint64_t base = b->stream.size();
        for (size_t k = 0; k < rel[c].size(); k++) b->offsets[(size_t)c * chunk + k] = base + rel[c][k];
        b->stream.insert(b->stream.end(), parts[c].v.begin(), parts[c].v.end());
    }
    b->stream.resize(b->stream.size() + 64, 0);  // tail padding so vector over-reads stay in bounds
    return b.release();
    RC_CATCH(nullptr)
}
const uint8_t* rc_blocks_stream(const rc_blocks* b, size_t* len) {
    *len = b->stream.size();
    return b->stream.data();
}
const uint64_t* rc_blocks_offsets(const rc_blocks* b, uint32_t* n) {
    *n = (uint32_t)b->offsets.size();
    return b->offsets.data();
}
const int32_t* rc_blocks_values(const rc_blocks* b) { return b->values.data(); }
void rc_blocks_forutil_table(int32_t out[32]) { forutil_table(out); }
void rc_blocks_destroy(rc_blocks* b) { delete b; }

}  // extern "C"
