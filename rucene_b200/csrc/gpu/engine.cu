// engine.cu — engine lifecycle, segment upload (parse `.doc`, build the HBM index image) and the
// ForUtil block-decode entry points of include/rucene_gpu.h.
//
// Upload replaces what Lucene50PostingsReader::open + BlockDocIterator::reset/refill_docs +
// Lucene50SkipReader do lazily per query (codec/postings/posting_reader.rs:85-158,460-561;
// codec/postings/skip_reader.rs:460-511): headers are parsed once, every block's payload bytes
// are copied UNCHANGED into a 16-byte aligned slot, and level 0 of the skip list becomes the
// flat `blk_last` table (last docid per block).
#include <algorithm>
#include <atomic>
#include <cstring>
#include <memory>
#include <thread>

#include "engine.hpp"

namespace rg {

thread_local std::string g_last_error;

int translate_exception() {
    try {
        throw;
    } catch (const CudaError& e) {
        g_last_error = e.what();
        return (e.code == cudaErrorNoDevice || e.code == cudaErrorInsufficientDriver) ? RG_ENODEVICE
                                                                                       : RG_ECUDA;
    } catch (const ArgError& e) {
        g_last_error = e.what();
        return RG_EINVAL;
    } catch (const Unsupported& e) {
        g_last_error = e.what();
        return RG_EUNSUPPORTED;
    } catch (const OutOfArena& e) {
        g_last_error = e.what();
        return RG_ENOMEM;
    } catch (const std::bad_alloc&) {
        g_last_error = "host allocation failed";
        return RG_ENOMEM;
    } catch (const std::exception& e) {
        g_last_error = e.what();
        return RG_EINVAL;
    }
}

namespace {

// ---------------------------------------------------------------- host byte reader
struct In {
    const uint8_t* p;
    size_t len, pos;
    In(const uint8_t* b, size_t l, size_t at = 0) : p(b), len(l), pos(at) {}
    uint8_t u8() {
        if (pos >= len) throw ArgError("`.doc` truncated");
        return p[pos++];
    }
    int32_t vint() {
        uint32_t v = 0;
        for (int shift = 0; shift < 35; shift += 7) {
            uint8_t b = u8();
            v |= (uint32_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) return (int32_t)v;
        }
        throw ArgError("invalid vint");
    }
    int64_t vlong() {
        uint64_t v = 0;
        for (int shift = 0; shift < 63; shift += 7) {
            uint8_t b = u8();
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) return (int64_t)v;
        }
        throw ArgError("invalid vlong");
    }
    uint32_t be32() {
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) v = (v << 8) | u8();
        return v;
    }
    const uint8_t* take(size_t n) {
        if (pos + n > len) throw ArgError("`.doc` truncated");
        const uint8_t* r = p + pos;
        pos += n;
        return r;
    }
};

struct DocHeader {
    int version = 0;
    uint32_t sb_mask = 0;
    int enc_size[33];  // payload bytes for num_bits b (index b)
    size_t body_start = 0;
};

void format_sizes(int version, const int32_t table[32], DocHeader& h) {
    h.version = version;
    h.sb_mask = 0;
    h.enc_size[0] = 0;
    for (int i = 0; i < 32; i++) {
        int code = table[i];
        int fmt = code >> 5, bpv = (code & 31) + 1;
        if (fmt != 0 && fmt != 1) throw ArgError("ForUtil table: invalid format id");
        if (version > 0) {
            h.enc_size[i + 1] = 16 * (i + 1);  // SIMD_ENCODE_SIZE, for_util.rs:44-52
        } else {
            if (bpv != i + 1)
                throw Unsupported("ForUtil table widens bits_per_value (non-COMPACT writer)");
            if (fmt == 1) {
                h.sb_mask |= 1u << i;
                int per = 64 / bpv;
                h.enc_size[i + 1] = ((kBlock + per - 1) / per) * 8;
            } else {
                h.enc_size[i + 1] = (kBlock * bpv + 7) / 8;
            }
        }
    }
}

// codec/codec_util.rs:46-57,75-124 + for_util.rs:120-148
DocHeader parse_doc_header(const uint8_t* file, size_t len) {
    In in(file, len);
    if (in.be32() != 0x3FD76C17u) throw ArgError("`.doc`: bad codec magic");
    int n = in.vint();
    static const char* codec = "Lucene50PostingsWriterDoc";
    if (n != (int)strlen(codec) || memcmp(in.take((size_t)n), codec, (size_t)n) != 0)
        throw ArgError("`.doc`: codec name mismatch");
    int version = (int)in.be32();
    if (version < 0 || version > 1) throw ArgError("`.doc`: unsupported version");
    in.take(16);
    int sl = in.u8();
    in.take((size_t)sl);
    if (in.vint() != 2) throw ArgError("`.doc`: PackedInts version must be 2");
    int32_t table[32];
    for (int i = 0; i < 32; i++) table[i] = in.vint();
    DocHeader h;
    format_sizes(version, table, h);
    h.body_start = in.pos;
    return h;
}

// scalar host decode of one block part (only for the last block of a term, whose last docid is
// not in the skip list)
void host_unpack(const uint8_t* part, int b, int version, uint32_t sb_mask, int32_t* out) {
    if (version > 0) {
        const uint32_t mask = b == 32 ? 0xffffffffu : ((1u << b) - 1u);
        for (int n = 0; n < kBlock; n++) {
            int lane = n & 3, q = n >> 2;
            int bit = q * b, j = bit >> 5, s = bit & 31;
            uint32_t lo, hi = 0;
            memcpy(&lo, part + 16 * j + 4 * lane, 4);
            if (s + b > 32) memcpy(&hi, part + 16 * (j + 1) + 4 * lane, 4);
            uint64_t x = ((uint64_t)hi << 32) | lo;
            out[n] = (int32_t)((uint32_t)(x >> s) & mask);
        }
    } else if ((sb_mask >> (b - 1)) & 1u) {
        int per = 64 / b;
        const uint64_t mask = b == 64 ? ~0ull : ((1ull << b) - 1);
        for (int n = 0; n < kBlock; n++) {
            int L = n / per, i = n % per;
            uint64_t x = 0;
            for (int k = 0; k < 8; k++) x = (x << 8) | part[8 * L + k];
            out[n] = (int32_t)((x >> (i * b)) & mask);
        }
    } else {
        for (int n = 0; n < kBlock; n++) {
            uint64_t bit = (uint64_t)n * b;
            uint32_t v = 0;
            for (int k = 0; k < b; k++, bit++) v = (v << 1) | ((part[bit >> 3] >> (7 - (bit & 7))) & 1u);
            out[n] = (int32_t)v;
        }
    }
}

struct BlockSrc {
    const uint8_t* doc_src;
    const uint8_t* freq_src;
    uint16_t doc_sz, freq_sz;  // payload bytes (0 when constant)
    uint8_t bd, bf;
    uint8_t enc;     // EncodeType of the doc part: 0 PF, 1 EF, 2 BITSET (for_util.rs:505-513)
    int32_t hdr[4];  // EF: {num_low_bits, n_upper_longs, n_lower_longs, 0}; BITSET: {min_doc, num_words, 0, 0}
    int32_t doc_const, freq_const;
    int32_t last_doc;
};

// EliasFanoEncoder geometry of a block (util/packed/elias_fano_encoder.rs:62-123): number of low
// bits and the sizes of the upper / lower / index long arrays that follow vlong(upper_bound).
struct EfGeom {
    int num_low_bits;
    uint32_t n_upper, n_lower, n_index;
};
inline EfGeom ef_geom(int64_t upper_bound) {
    if (upper_bound < 0) throw ArgError("corrupt EF block: negative upper bound");
    auto longs_for_bits = [](int64_t n) { return (uint32_t)((uint64_t)(n + 63) >> 6); };
    EfGeom g{};
    const int64_t nv = kBlock, fac = upper_bound / nv;
    g.num_low_bits = fac > 0 ? 63 - __builtin_clzll((uint64_t)fac) : 0;
    const int64_t max_high = (int64_t)((uint64_t)upper_bound >> g.num_low_bits);
    g.n_lower = longs_for_bits(nv * g.num_low_bits);
    g.n_upper = longs_for_bits(max_high + nv);
    const int64_t n_entries = max_high / 256;  // DEFAULT_INDEX_INTERVAL
    const int64_t max_index_entry = max_high + nv - 1;
    const int entry_bits = max_index_entry <= 0 ? 0 : 64 - __builtin_clzll((uint64_t)max_index_entry);
    g.n_index = longs_for_bits(n_entries * entry_bits);
    return g;
}
inline uint64_t le64(const uint8_t* p) {
    uint64_t v;
    memcpy(&v, p, 8);
    return v;
}
// last docid of an EF / BITSET block (host side; only for the one block skip level 0 does not cover)
int32_t other_block_last_doc(const BlockSrc& b, int32_t ef_base_doc) {
    if (b.enc == 2) {  // min_doc + highest set bit
        for (int w = b.hdr[1] - 1; w >= 0; w--) {
            const uint64_t x = le64(b.doc_src + 8 * (size_t)w);
            if (x) return b.hdr[0] + 64 * w + 63 - __builtin_clzll(x);
        }
        throw ArgError("corrupt BITSET block: no bit set");
    }
    // EF: value 127 = ((position of the 128th set upper bit - 127) << L) | low[127]
    const int L = b.hdr[0];
    int64_t pos = -1;
    int seen = 0;
    for (int w = 0; w < b.hdr[1] && pos < 0; w++) {
        uint64_t x = le64(b.doc_src + 8 * (size_t)w);
        while (x) {
            const int bit = __builtin_ctzll(x);
            x &= x - 1;
            if (++seen == kBlock) {
                pos = 64 * (int64_t)w + bit;
                break;
            }
        }
    }
    if (pos < 0) throw ArgError("corrupt EF block: fewer than 128 upper bits");
    int64_t low = 0;
    if (L) {
        const uint8_t* lo = b.doc_src + 8 * (size_t)b.hdr[1];
        const int64_t bitpos = (int64_t)L * (kBlock - 1);
        const size_t wi = (size_t)(bitpos >> 6);
        const int at = (int)(bitpos & 63);
        uint64_t v = le64(lo + 8 * wi) >> at;
        if (at + L > 64) v |= le64(lo + 8 * (wi + 1)) << (64 - at);
        low = (int64_t)(v & ((1ull << L) - 1));
    }
    return (int32_t)((((pos - (kBlock - 1)) << L) | low) + 1 + ef_base_doc);
}

// all docids of an EF / BITSET block (host side, upload-time validation); returns how many were found (<= 128)
int other_block_docs(const BlockSrc& b, int32_t ef_base_doc, int32_t* out) {
    int n = 0;
    if (b.enc == 2) {
        for (int w = 0; w < b.hdr[1]; w++) {
            uint64_t x = le64(b.doc_src + 8 * (size_t)w);
            while (x) {
                if (n == kBlock) return kBlock + 1;
                out[n++] = b.hdr[0] + 64 * w + __builtin_ctzll(x);
                x &= x - 1;
            }
        }
        return n;
    }
    const int L = b.hdr[0];
    const uint8_t* lo = b.doc_src + 8 * (size_t)b.hdr[1];
    for (int w = 0; w < b.hdr[1] && n < kBlock; w++) {
        uint64_t x = le64(b.doc_src + 8 * (size_t)w);
        while (x && n < kBlock) {
            const int64_t pos = 64 * (int64_t)w + __builtin_ctzll(x);
            x &= x - 1;
            int64_t low = 0;
            if (L) {
                const int64_t bitpos = (int64_t)L * n;
                const size_t wi = (size_t)(bitpos >> 6);
                const int at = (int)(bitpos & 63);
                uint64_t v = le64(lo + 8 * wi) >> at;
                if (at + L > 64) v |= le64(lo + 8 * (wi + 1)) << (64 - at);
                low = (int64_t)(v & ((1ull << L) - 1));
            }
            const int64_t doc = (((pos - n) << L) | low) + 1 + ef_base_doc;
            if (doc < 0 || doc > 0x7ffffffe) return -1;
            out[n++] = (int32_t)doc;
        }
    }
    return n;
}

struct TermParse {
    uint32_t n_blocks = 0;
    const uint8_t* tail_src = nullptr;
    uint32_t tail_bytes = 0, tail_n = 0;
    int32_t tail_base = 0;
    uint64_t enc_bytes = 0;
};

inline uint32_t part_units(int sz) { return sz == 0 ? 1u : (uint32_t)((sz + 15) / 16); }

// Walk one term's region (posting_writer.rs:334-351,491-502 layout; skip level 0 per
// skip_writer.rs:209-226,241-259).
void parse_term(const uint8_t* file, size_t len, const DocHeader& h, const rg_term_state& ts, int32_t max_doc,
                std::vector<BlockSrc>& blocks, TermParse& tp) {
    const int df = ts.doc_freq;
    tp = TermParse();
    if (df <= 0) return;
    if (df == 1) {
        if (ts.singleton_doc_id < 0 || ts.singleton_doc_id >= max_doc) throw ArgError("singleton_doc_id outside [0, max_doc)");
        tp.tail_n = 1;
        return;
    }
    if (ts.doc_start_fp < 0 || (size_t)ts.doc_start_fp > len) throw ArgError("doc_start_fp out of range");
    In in(file, len, (size_t)ts.doc_start_fp);
    const uint32_t nb = (uint32_t)(df / kBlock);
    tp.n_blocks = nb;
    const size_t first = blocks.size();
    std::vector<size_t> block_fp(nb + 1);
    for (uint32_t i = 0; i < nb; i++) {
        block_fp[i] = in.pos;
        BlockSrc b{};
        uint8_t code = in.u8();
        b.enc = code >> 6;
        if (b.enc == 3) throw Unsupported("EncodeType::FULL doc blocks are unimplemented in the reference too");
        if (b.enc == 1) {  // EF, ForUtil::read_other_encode_block (for_util.rs:346-362)
            const EfGeom g = ef_geom(in.vlong());
            b.hdr[0] = g.num_low_bits;
            b.hdr[1] = (int32_t)g.n_upper;
            b.hdr[2] = (int32_t)g.n_lower;
            b.doc_src = in.take(8 * (size_t)(g.n_upper + g.n_lower));
            in.take(8 * (size_t)g.n_index);  // the skip index inside the block is not needed on the device
            b.doc_sz = (uint16_t)(16 + 8 * (g.n_upper + g.n_lower));
        } else if (b.enc == 2) {  // BITSET (:363-368)
            b.hdr[0] = in.vint();
            b.hdr[1] = in.u8();
            b.doc_src = in.take(8 * (size_t)b.hdr[1]);
            b.doc_sz = (uint16_t)(16 + 8 * b.hdr[1]);
        } else {
            b.bd = code & 0x3f;
            if (b.bd > 32) throw ArgError("corrupt doc block header");
            if (b.bd == 0) {
                b.doc_const = in.vint();
            } else {
                b.doc_sz = (uint16_t)h.enc_size[b.bd];
                b.doc_src = in.take(b.doc_sz);
            }
        }
        code = in.u8();
        b.bf = code & 0x3f;  // ForUtil::read_block: num_bits = code & 0x3F
        if (b.bf > 32) throw ArgError("corrupt freq block header");
        if (b.bf == 0) {
            b.freq_const = in.vint();
        } else {
            b.freq_sz = (uint16_t)h.enc_size[b.bf];
            b.freq_src = in.take(b.freq_sz);
        }
        blocks.push_back(b);
    }
    block_fp[nb] = in.pos;
    // vint tail
    tp.tail_n = (uint32_t)(df % kBlock);
    tp.tail_src = file + in.pos;
    size_t tail_start = in.pos;
    int64_t tail_delta_sum = 0;
    for (uint32_t i = 0; i < tp.tail_n; i++) {
        uint32_t code = (uint32_t)in.vint();
        tail_delta_sum += code >> 1;
        if (!(code & 1)) in.vint();
    }
    tp.tail_bytes = (uint32_t)(in.pos - tail_start);
    tp.enc_bytes = in.pos - (size_t)ts.doc_start_fp;
    // last docid of each full block: skip level 0, then a host decode for the uncovered block
    uint32_t n0 = df > kBlock ? (uint32_t)((df - 1) / kBlock) : 0;
    int32_t last = 0;
    if (n0 > 0) {
        if (ts.skip_offset < 0) throw ArgError("doc_freq > 128 but no skip_offset");
        In sk(file, len, (size_t)(ts.doc_start_fp + ts.skip_offset));
        int trimmed = df % kBlock == 0 ? df - 1 : df;  // skip_reader.rs:307-313
        int levels = 1;
        for (int64_t x = trimmed / kBlock; x >= 8; x /= 8) levels++;
        levels = std::min(levels, 10);
        for (int lv = levels - 1; lv >= 1; lv--) {
            int64_t length = sk.vlong();
            sk.take((size_t)length);
        }
        int64_t fp = ts.doc_start_fp;
        for (uint32_t i = 0; i < n0; i++) {
            last += sk.vint();
            fp += sk.vlong();
            if ((size_t)fp != block_fp[i + 1]) throw ArgError("skip data disagrees with block layout");
            blocks[first + i].last_doc = last;
        }
    }
    for (uint32_t i = n0; i < nb; i++) {  // at most one block
        const BlockSrc& b = blocks[first + i];
        if (b.enc) {
            last = other_block_last_doc(b, i == 0 ? -1 : last);
            blocks[first + i].last_doc = last;
            continue;
        }
        int64_t sum = 0;
        if (b.bd == 0) {
            sum = (int64_t)b.doc_const * kBlock;
        } else {
            int32_t vals[kBlock];
            host_unpack(b.doc_src, b.bd, h.version, h.sb_mask, vals);
            for (int k = 0; k < kBlock; k++) sum += vals[k];
        }
        last = (int32_t)(last + sum);
        blocks[first + i].last_doc = last;
    }
    tp.tail_base = nb ? last : 0;
    // The kernels index norms / live docs / windows with these docids: a corrupt file must fail here
    // (RG_EINVAL), not as an out-of-bounds device access.
    int32_t prev = -1;
    for (uint32_t i = 0; i < nb; i++) {
        const BlockSrc& b = blocks[first + i];
        if (b.last_doc <= prev || b.last_doc >= max_doc || (int64_t)b.last_doc - prev < kBlock)
            throw ArgError("corrupt postings: block last docids must increase by >= 128 and stay below max_doc");
        if (b.enc) {  // EF / BITSET: every docid of the block, decoded here once, must be increasing in (prev, last_doc]
            int32_t docs[kBlock];
            if (other_block_docs(b, prev, docs) != kBlock) throw ArgError("corrupt EF/BITSET doc block: not 128 docids");
            int32_t q = prev;
            for (int k = 0; k < kBlock; k++) {
                if (docs[k] <= q) throw ArgError("corrupt EF/BITSET doc block: docids not increasing");
                q = docs[k];
            }
            if (q != b.last_doc) throw ArgError("corrupt EF/BITSET doc block: disagrees with the skip data");
        }
        prev = b.last_doc;
    }
    if (tp.tail_n && (int64_t)tp.tail_base + tail_delta_sum >= (int64_t)max_doc)
        throw ArgError("corrupt postings: vint tail runs past max_doc");
}

int hw_threads() {
    unsigned n = std::thread::hardware_concurrency();
    return n ? (int)std::min(n, 64u) : 1;
}

template <class F>
void parallel_chunks(size_t n, F&& f) {
    int nt = (int)std::min<size_t>((size_t)hw_threads(), n);
    if (nt <= 1) {
        for (size_t i = 0; i < n; i++) f(i);
        return;
    }
    std::atomic<size_t> next{0};
    std::atomic<int> code{0};
    std::string msg;
    std::vector<std::thread> ts;
    for (int t = 0; t < nt; t++)
        ts.emplace_back([&] {
            for (;;) {
                size_t i = next.fetch_add(1);
                if (i >= n || code.load()) break;
                try {
                    f(i);
                } catch (...) {
                    int c = translate_exception();
                    int expected = 0;
                    if (code.compare_exchange_strong(expected, c)) msg = g_last_error;
                }
            }
        });
    for (auto& t : ts) t.join();
    if (int c = code.load()) {
        if (c == RG_EUNSUPPORTED) throw Unsupported(msg);
        throw ArgError(msg);
    }
}

template <class T>
void upload(DevBuf<T>& dst, const T* src, size_t n, cudaStream_t st) {
    dst.alloc(n);
    if (n) RG_CUDA_CHECK(cudaMemcpyAsync(dst.p, src, n * sizeof(T), cudaMemcpyHostToDevice, st));
}

}  // namespace

void build_segment(rg_engine* e, Segment& seg, int32_t doc_base, int32_t max_doc,
                   const uint8_t* file, size_t len, const uint8_t* norms, const uint64_t* live,
                   const rg_term_state* terms, uint32_t n_terms) {
    const DocHeader h = parse_doc_header(file, len);
    // pass 1: parse term regions in parallel chunks
    const size_t n_chunks = std::max<size_t>(1, std::min<size_t>(256, (n_terms + 63) / 64));
    struct Chunk {
        uint32_t t0, t1;
        std::vector<BlockSrc> blocks;
        std::vector<TermParse> tp;
        uint64_t blk_base = 0, unit_base = 0, tail_base = 0, units = 0, tail_bytes = 0;
    };
    std::vector<Chunk> chunks(n_chunks);
    {
        // balance by doc_freq
        uint64_t total = 0;
        for (uint32_t t = 0; t < n_terms; t++) total += (uint64_t)std::max(terms[t].doc_freq, 0) + 16;
        uint64_t per = total / n_chunks + 1, acc = 0;
        size_t c = 0;
        chunks[0].t0 = 0;
        for (uint32_t t = 0; t < n_terms; t++) {
            acc += (uint64_t)std::max(terms[t].doc_freq, 0) + 16;
            if (acc >= per && c + 1 < n_chunks) {
                chunks[c].t1 = t + 1;
                c++;
                chunks[c].t0 = t + 1;
                acc = 0;
            }
        }
        chunks[c].t1 = n_terms;
        for (size_t i = c + 1; i < n_chunks; i++) chunks[i].t0 = chunks[i].t1 = n_terms;
    }
    parallel_chunks(n_chunks, [&](size_t ci) {
        Chunk& ch = chunks[ci];
        ch.tp.resize(ch.t1 - ch.t0);
        for (uint32_t t = ch.t0; t < ch.t1; t++) {
            parse_term(file, len, h, terms[t], max_doc, ch.blocks, ch.tp[t - ch.t0]);
        }
        for (const BlockSrc& b : ch.blocks) ch.units += part_units(b.doc_sz) + part_units(b.freq_sz);
        for (const TermParse& tp : ch.tp) ch.tail_bytes += tp.tail_bytes;
    });
    uint64_t n_blocks = 0, units = 0, tail_bytes = 0;
    for (Chunk& ch : chunks) {
        ch.blk_base = n_blocks;
        ch.unit_base = units;
        ch.tail_base = tail_bytes;
        n_blocks += ch.blocks.size();
        units += ch.units;
        tail_bytes += ch.tail_bytes;
    }
    if (units + 8 >= (1ull << 32)) throw Unsupported("segment image exceeds 64 GiB of block payload");
    if (n_blocks >= (1ull << 32) || tail_bytes >= (1ull << 32)) throw Unsupported("segment too large");
    // pass 2: fill the host staging image
    std::vector<uint4> h_arena(units + 8);
    std::vector<int32_t> h_last(n_blocks + 1);
    std::vector<BlockDesc> h_desc(n_blocks + 1);
    std::vector<uint8_t> h_tails(tail_bytes + 16);
    std::vector<TermDev> h_terms(n_terms);
    seg.host_terms.assign(n_terms, TermHost());
    parallel_chunks(n_chunks, [&](size_t ci) {
        Chunk& ch = chunks[ci];
        uint64_t blk = ch.blk_base, unit = ch.unit_base, tail = ch.tail_base;
        size_t bi = 0;
        for (uint32_t t = ch.t0; t < ch.t1; t++) {
            const TermParse& tp = ch.tp[t - ch.t0];
            const rg_term_state& ts = terms[t];
            TermDev td{};
            td.blk_begin = (uint32_t)blk;
            td.n_blocks = tp.n_blocks;
            td.tail_off = (uint32_t)tail;
            td.tail_n = tp.tail_n;
            td.doc_freq = std::max(ts.doc_freq, 0);
            td.tail_base = tp.tail_base;
            td.singleton_doc = ts.doc_freq == 1 ? ts.singleton_doc_id : -1;
            td.singleton_freq = ts.doc_freq == 1 ? (int32_t)ts.total_term_freq : 0;
            h_terms[t] = td;
            seg.host_terms[t].doc_freq = td.doc_freq;
            seg.host_terms[t].n_blocks = tp.n_blocks;
            seg.host_terms[t].enc_bytes = tp.enc_bytes;
            seg.host_terms[t].tail_n = tp.tail_n;
            seg.host_terms[t].tail_base = tp.tail_base;
            for (uint32_t i = 0; i < tp.n_blocks; i++, bi++, blk++) {
                const BlockSrc& b = ch.blocks[bi];
                const uint32_t du = part_units(b.doc_sz), fu = part_units(b.freq_sz);
                uint8_t* dst = reinterpret_cast<uint8_t*>(&h_arena[unit]);
                if (b.enc) {  // 16-byte header, then the raw little-endian longs
                    memcpy(dst, b.hdr, 16);
                    memcpy(dst + 16, b.doc_src, (size_t)b.doc_sz - 16);
                } else if (b.bd) {
                    memcpy(dst, b.doc_src, b.doc_sz);
                } else {
                    memcpy(dst, &b.doc_const, 4);
                }
                uint8_t* fdst = dst + 16 * (size_t)du;
                if (b.bf) memcpy(fdst, b.freq_src, b.freq_sz);
                else memcpy(fdst, &b.freq_const, 4);
                h_last[blk] = b.last_doc;
                h_desc[blk].off16 = (uint32_t)unit;
                h_desc[blk].bits = (uint32_t)b.bd | ((uint32_t)b.bf << 8) | (du << 16) | ((uint32_t)b.enc << 24);
                unit += du + fu;
            }
            if (tp.tail_bytes) {
                memcpy(&h_tails[tail], tp.tail_src, tp.tail_bytes);
                tail += tp.tail_bytes;
            }
        }
    });
    cudaStream_t st = e->stream;
    upload(seg.arena, h_arena.data(), h_arena.size(), st);
    upload(seg.blk_last, h_last.data(), h_last.size(), st);
    upload(seg.blk_desc, h_desc.data(), h_desc.size(), st);
    upload(seg.tails, h_tails.data(), h_tails.size(), st);
    upload(seg.terms, h_terms.data(), h_terms.size(), st);
    if (norms) {
        upload(seg.norms, norms, (size_t)max_doc, st);
        for (int64_t i = 0; i < (int64_t)max_doc; i++) seg.norm_seen[norms[i]] = 1;
    }
    if (live) upload(seg.live, live, ((size_t)max_doc + 63) / 64, st);
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    for (const Chunk& ch : chunks)
        for (const BlockSrc& b : ch.blocks) {
            seg.has_other_enc = seg.has_other_enc || b.enc != 0;
            seg.block_enc_bytes += 2ull + (b.doc_sz ? b.doc_sz : 1u) + (b.freq_sz ? b.freq_sz : 1u);
        }
    seg.n_blocks_total = n_blocks;
    e->col_budget_floats = 0;
    e->local_budget_floats = 0;
    seg.doc_base = doc_base;
    seg.max_doc = max_doc;
    seg.dev.arena = seg.arena.p;
    seg.dev.blk_last = seg.blk_last.p;
    seg.dev.blk_desc = seg.blk_desc.p;
    seg.dev.tails = seg.tails.p;
    seg.dev.terms = seg.terms.p;
    seg.dev.norms = seg.norms.p;
    seg.dev.live = seg.live.p;
    seg.dev.doc_base = doc_base;
    seg.dev.max_doc = max_doc;
    seg.dev.n_terms = n_terms;
    seg.dev.version = h.version;
    seg.dev.sb_mask = h.sb_mask;
    // ---- presence bitmaps of the dense terms (device-side: one warp per block sets 128 bits)
    seg.bitmap_slot.assign(n_terms, -1);
    if (!(e->cfg.flags & RG_CFG_NO_BITMAPS)) {
        // score columns need the bitmaps of the terms with df >= max_doc/64 only; k_eval_or_ms wants them down to /1024
        const uint64_t bitmap_den = (e->cfg.flags & RG_CFG_MAXSCORE) ? kBitmapDen : kColumnDen;
        std::vector<uint32_t> dense;
        for (uint32_t t = 0; t < n_terms; t++)
            if ((uint64_t)std::max(terms[t].doc_freq, 0) * bitmap_den >= (uint64_t)max_doc && terms[t].doc_freq >= 2)
                dense.push_back(t);
        std::sort(dense.begin(), dense.end(), [&](uint32_t a, uint32_t b) {
            return terms[a].doc_freq != terms[b].doc_freq ? terms[a].doc_freq > terms[b].doc_freq : a < b;
        });
        seg.bitmap_words = (((uint64_t)max_doc + 31) / 32 + 64 + 3) & ~3ull;
        size_t free_b = 0, total_b = 0;
        RG_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
        const uint64_t budget = std::max<uint64_t>(64ull << 20, (uint64_t)free_b / 5);  // bytes: a fifth of the free HBM
        const size_t n_bm = (size_t)std::min<uint64_t>(dense.size(), budget / (seg.bitmap_words * 4));
        if (n_bm) {
            dense.resize(n_bm);
            seg.bitmaps.alloc(n_bm * seg.bitmap_words);
            RG_CUDA_CHECK(cudaMemsetAsync(seg.bitmaps.p, 0, seg.bitmaps.bytes(), st));
            std::vector<ColumnJob> jobs(n_bm);
            uint32_t units = 0;
            for (size_t i = 0; i < n_bm; i++) {
                const uint32_t t = dense[i];
                seg.bitmap_slot[t] = (int32_t)i;
                seg.bitmap_terms.push_back(t);
                jobs[i] = ColumnJob{0u, t, 0u, 0.0f, seg.bitmaps.p + i * seg.bitmap_words, units, 0u};
                units += seg.host_terms[t].n_blocks + (seg.host_terms[t].tail_n ? 1u : 0u);
            }
            DevBuf<SegDev> d_seg;
            DevBuf<ColumnJob> d_jobs;
            upload(d_seg, &seg.dev, 1, st);
            upload(d_jobs, jobs.data(), jobs.size(), st);
            launch_build_bitmaps(st, d_seg.p, d_jobs.p, (uint32_t)n_bm, units);
            RG_CUDA_CHECK(cudaGetLastError());
            e->launches++;
            RG_CUDA_CHECK(cudaStreamSynchronize(st));
        }
    }
    seg.device_bytes = seg.arena.bytes() + seg.blk_last.bytes() + seg.blk_desc.bytes() + seg.tails.bytes() +
                       seg.terms.bytes() + seg.norms.bytes() + seg.live.bytes() + seg.bitmaps.bytes();
}

// Lucene's norm table maps byte 0 to an infinite length, so a norm cache usually holds +inf at [0]: what matters is the
// entries that norm bytes of the leaf actually select (f / (f + inf) would be a score of exactly 0).
void refresh_cache_small(rg_engine* e) {
    const size_t n_caches = e->h_caches.size() / 256;
    for (Segment& sg : e->segs) {
        sg.cache_small.assign(n_caches, 1);
        for (size_t c = 0; c < n_caches; c++)
            for (int i = 0; i < 256; i++)
                if (sg.norm_seen[i] && !(e->h_caches[c * 256 + i] >= 0.0f && e->h_caches[c * 256 + i] <= 1e10f)) sg.cache_small[c] = 0;
    }
}

}  // namespace rg

using namespace rg;

void rg_engine::sync_tables() {
    if (segs_dirty) {
        std::vector<SegDev> h(segs.size());
        for (size_t i = 0; i < segs.size(); i++) h[i] = segs[i].dev;
        d_segs.alloc(std::max<size_t>(1, h.size()));
        if (!h.empty())
            RG_CUDA_CHECK(cudaMemcpyAsync(d_segs.p, h.data(), h.size() * sizeof(SegDev),
                                          cudaMemcpyHostToDevice, stream));
        RG_CUDA_CHECK(cudaStreamSynchronize(stream));
        segs_dirty = false;
    }
    if (caches_dirty) {
        d_caches.alloc(std::max<size_t>(256, h_caches.size()));
        if (!h_caches.empty())
            RG_CUDA_CHECK(cudaMemcpyAsync(d_caches.p, h_caches.data(), h_caches.size() * sizeof(float),
                                          cudaMemcpyHostToDevice, stream));
        RG_CUDA_CHECK(cudaStreamSynchronize(stream));
        caches_dirty = false;
    }
}

struct rg_blockset {
    DevBuf<uint4> arena;
    DevBuf<BlockDesc> desc;
    DevBuf<int32_t> out;
    uint32_t n_blocks = 0;
    int version = 0;
    uint32_t sb_mask = 0;
    uint64_t enc_bytes = 0;
};

#define RG_TRY try {
#define RG_CATCH \
    }            \
    catch (...) { return translate_exception(); }

extern "C" {

const char* rg_last_error(rg_engine*) { return g_last_error.c_str(); }

int rg_engine_create(const rg_config* cfg, rg_engine** out) {
    RG_TRY
    if (!out) throw ArgError("out is null");
    *out = nullptr;
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || count == 0) {
        g_last_error = std::string("no CUDA device: ") + cudaGetErrorString(ce) +
                       " (librucene_gpu has no CPU fallback)";
        cudaGetLastError();
        return RG_ENODEVICE;
    }
    std::unique_ptr<rg_engine> e(new rg_engine());
    if (cfg) e->cfg = *cfg;
    int dev = e->cfg.device;
    if (dev < 0) RG_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= count) throw ArgError("device ordinal out of range");
    RG_CUDA_CHECK(cudaSetDevice(dev));
    e->device = dev;
    RG_CUDA_CHECK(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
    e->stream = e->own_stream;
    RG_CUDA_CHECK(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    for (auto& ev : e->list_jobs_done) RG_CUDA_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    RG_CUDA_CHECK(cudaEventCreate(&e->ev0));
    RG_CUDA_CHECK(cudaEventCreate(&e->ev1));
    RG_CUDA_CHECK(cudaEventCreate(&e->ev2));
    RG_CUDA_CHECK(cudaEventCreate(&e->ev3));
    for (auto& ev : e->rescore_ev) RG_CUDA_CHECK(cudaEventCreate(&ev));
    e->range_postings_set = e->cfg.range_postings != 0;  // else the planner picks per batch (plan_batch)
    if (e->cfg.range_postings == 0) e->cfg.range_postings = 1u << 15;
    if (const char* v = getenv("RG_OR_COL_DEN")) e->or_col_den = std::max(1, atoi(v));  // tuning knob (bench sweeps)
    if (const char* v = getenv("RG_COLUMN_SWEEP")) e->column_sweep = atoi(v) != 0;      // A/B knob
    *out = e.release();
    return RG_OK;
    RG_CATCH
}

void rg_engine_destroy(rg_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    if (e->ev0) cudaEventDestroy(e->ev0);
    if (e->ev1) cudaEventDestroy(e->ev1);
    if (e->ev2) cudaEventDestroy(e->ev2);
    if (e->ev3) cudaEventDestroy(e->ev3);
    for (auto& ev : e->rescore_ev)
        if (ev) cudaEventDestroy(ev);
    for (auto& ev : e->list_jobs_done)
        if (ev) cudaEventDestroy(ev);
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    if (e->own_stream) cudaStreamDestroy(e->own_stream);
    delete e;
}

int rg_engine_set_stream(rg_engine* e, void* s) {
    RG_TRY
    if (!e) throw ArgError("engine is null");
    e->stream = s ? reinterpret_cast<cudaStream_t>(s) : e->own_stream;
    return RG_OK;
    RG_CATCH
}

uint64_t rg_engine_launch_count(rg_engine* e) { return e ? e->launches : 0; }

int rg_engine_set_flags(rg_engine* e, uint32_t flags) {
    RG_TRY
    if (!e) throw ArgError("engine is null");
    // RG_CFG_NO_BITMAPS acts at upload time: it cannot be cleared once a segment went up without bitmaps
    e->cfg.flags = flags;
    return RG_OK;
    RG_CATCH
}

int rg_engine_column_stats(rg_engine* e, uint64_t out[4]) {
    RG_TRY
    if (!e || !out) throw ArgError("null argument");
    out[0] = e->col_cache.size();
    out[1] = e->col_floats * sizeof(float);
    out[2] = e->col_builds;
    out[3] = e->col_hits;
    return RG_OK;
    RG_CATCH
}

int rg_engine_list_stats(rg_engine* e, uint64_t out[4]) {
    RG_TRY
    if (!e || !out) throw ArgError("null argument");
    out[0] = e->list_cache.size();
    out[1] = e->list_floats * sizeof(float);
    out[2] = e->list_builds;
    out[3] = e->list_hits;
    return RG_OK;
    RG_CATCH
}

float rg_engine_last_kernel_ms(rg_engine* e, const char* which) {
    if (!e || !which) return -1.f;
    std::string w(which);
    if (w == "decode") return e->last_decode_ms;
    if (w == "eval") return e->last_eval_ms;
    if (w == "replay") return e->last_replay_ms;
    if (w == "run") return e->last_run_ms;
    if (w == "rescore") {
        if (e->rescore_timed && cudaEventSynchronize(e->rescore_ev[1]) == cudaSuccess) {
            cudaEventElapsedTime(&e->last_rescore_ms, e->rescore_ev[0], e->rescore_ev[1]);
            e->rescore_timed = false;
        }
        cudaGetLastError();
        return e->last_rescore_ms;
    }
    return -1.f;
}

uint64_t rg_engine_index_bytes(rg_engine* e) {
    uint64_t b = 0;
    if (e)
        for (auto& s : e->segs) {
            b += s.device_bytes;
            for (auto& f : s.points) b += f.second.bytes();
        }
    return b;
}

int rg_points_upload(rg_engine* e, uint32_t seg_ord, uint32_t field, uint32_t bytes_per_dim, const int32_t* docs,
                     const uint8_t* packed, size_t n) {
    RG_TRY
    if (!e || (n && (!docs || !packed))) throw ArgError("null argument");
    if (seg_ord >= e->segs.size()) throw ArgError("rg_points_upload: leaf not uploaded");
    if (bytes_per_dim != 4 && bytes_per_dim != 8) throw ArgError("rg_points_upload: bytes_per_dim must be 4 or 8");
    Segment& seg = e->segs[seg_ord];
    if (seg.points.count(field)) throw ArgError("rg_points_upload: field already uploaded for this leaf");
    const int32_t max_doc = seg.max_doc;
    if (n > 0xffffffffull) throw ArgError("rg_points_upload: more than 2^32 - 1 points");  // offsets are u32
    for (size_t i = 0; i < n; i++)
        if (docs[i] < 0 || docs[i] >= max_doc) throw ArgError("rg_points_upload: docid outside [0, max_doc)");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    // the packed bytes as a big-endian unsigned integer: compares exactly as the byte strings do
    std::vector<uint64_t> key(n);
    for (size_t i = 0; i < n; i++) {
        uint64_t v = 0;
        for (uint32_t j = 0; j < bytes_per_dim; j++) v = v << 8 | packed[i * bytes_per_dim + j];
        key[i] = v;
    }
    // CSR in docid order, keys ascending within a doc
    std::vector<uint32_t> offsets((size_t)max_doc + 1, 0);
    for (size_t i = 0; i < n; i++) offsets[(size_t)docs[i] + 1]++;
    for (size_t d = 0; d < (size_t)max_doc; d++) offsets[d + 1] += offsets[d];
    std::vector<uint64_t> csr(n);
    {
        std::vector<uint32_t> pos(offsets.begin(), offsets.end() - 1);
        for (size_t i = 0; i < n; i++) csr[pos[(size_t)docs[i]]++] = key[i];
    }
    for (size_t d = 0; d < (size_t)max_doc; d++) std::sort(csr.begin() + offsets[d], csr.begin() + offsets[d + 1]);
    const size_t n_blk = ((size_t)max_doc + kBlock - 1) / kBlock;
    std::vector<RangeBlock> blocks(n_blk, RangeBlock{~0ull, 0ull, 0u, 0u});
    for (size_t d = 0; d < (size_t)max_doc; d++) {
        RangeBlock& b = blocks[d / kBlock];
        const uint32_t o0 = offsets[d], o1 = offsets[d + 1];
        if (o0 == o1) continue;
        b.docs++;
        b.values += o1 - o0;
        b.min = std::min(b.min, csr[o0]);
        b.max = std::max(b.max, csr[o1 - 1]);
    }
    PointField pf;
    pf.bytes_per_dim = bytes_per_dim;
    cudaStream_t st = e->stream;
    upload(pf.offsets, offsets.data(), offsets.size(), st);
    upload(pf.blocks, blocks.data(), blocks.size(), st);
    std::vector<uint32_t> k32;
    if (bytes_per_dim == 4) k32.assign(csr.begin(), csr.end());
    pf.keys.alloc(n * bytes_per_dim);
    if (n)
        RG_CUDA_CHECK(cudaMemcpyAsync(pf.keys.p, bytes_per_dim == 8 ? (const void*)csr.data() : (const void*)k32.data(),
                                      n * bytes_per_dim, cudaMemcpyHostToDevice, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));  // the host vectors go out of scope
    std::sort(key.begin(), key.end());
    pf.sorted = std::move(key);
    seg.points.emplace(field, std::move(pf));
    e->generation++;  // batches prepared before this upload are stale
    return RG_OK;
    RG_CATCH
}

int rg_segment_upload(rg_engine* e, uint32_t seg_ord, int32_t doc_base, int32_t max_doc,
                      const uint8_t* doc_file, size_t doc_len, const uint8_t* norms,
                      const uint64_t* live_docs, const rg_term_state* terms, uint32_t n_terms) {
    RG_TRY
    if (!e || !doc_file || (!terms && n_terms)) throw ArgError("null argument");
    if (seg_ord != e->segs.size()) throw ArgError("segments must be uploaded in leaf order (seg_ord == #uploaded)");
    if (seg_ord >= 65535) throw ArgError("too many segments");
    if (max_doc <= 0 || doc_base < 0) throw ArgError("bad max_doc/doc_base");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    Segment seg;
    build_segment(e, seg, doc_base, max_doc, doc_file, doc_len, norms, live_docs, terms, n_terms);
    e->segs.push_back(std::move(seg));
    e->segs_dirty = true;
    e->generation++;  // batches prepared before this upload are stale (rg_batch_run checks)
    refresh_cache_small(e);
    return RG_OK;
    RG_CATCH
}

int rg_norm_cache_set(rg_engine* e, uint32_t cache_id, const float cache[256]) {
    RG_TRY
    if (!e || !cache) throw ArgError("null argument");
    if (cache_id >= 4096) throw ArgError("cache_id out of range");
    if (e->h_caches.size() < (size_t)(cache_id + 1) * 256) e->h_caches.resize((size_t)(cache_id + 1) * 256, 0.f);
    memcpy(&e->h_caches[(size_t)cache_id * 256], cache, 256 * sizeof(float));
    e->caches_dirty = true;
    e->generation++;
    if (e->cache_nonneg.size() <= cache_id) e->cache_nonneg.resize(cache_id + 1, 0);
    bool nonneg = true;
    for (int i = 0; i < 256; i++) nonneg = nonneg && cache[i] >= 0.0f;  // false for NaN as well
    e->cache_nonneg[cache_id] = nonneg ? 1 : 0;
    refresh_cache_small(e);
    for (Segment& sg : e->segs)  // and so are the high tf-norm planes of this cache
        for (auto it = sg.tf_planes.begin(); it != sg.tf_planes.end();)
            it = it->first.first == cache_id ? sg.tf_planes.erase(it) : std::next(it);
    // score columns / scored lists computed with the previous contents of this cache are no longer valid
    for (auto it = e->col_cache.begin(); it != e->col_cache.end();) {
        if (std::get<3>(it->first) == cache_id) {
            e->col_floats -= it->second->len;
            it = e->col_cache.erase(it);
        } else {
            ++it;
        }
    }
    for (auto it = e->list_cache.begin(); it != e->list_cache.end();) {
        if (std::get<3>(it->first) == cache_id) {
            e->list_floats -= it->second->len;
            it = e->list_cache.erase(it);
        } else {
            ++it;
        }
    }
    return RG_OK;
    RG_CATCH
}

// ---------------------------------------------------------------- block codec entry points
int rg_segment_decode(rg_engine* e, uint32_t seg_ord, uint64_t first_block, uint64_t n_blocks, int32_t* out,
                      uint64_t stats[4]) {
    RG_TRY
    if (!e || !stats) throw ArgError("null argument");
    if (seg_ord >= e->segs.size()) throw ArgError("no such segment");
    const Segment& seg = e->segs[seg_ord];
    if (first_block > seg.n_blocks_total) throw ArgError("first_block out of range");
    n_blocks = std::min<uint64_t>(n_blocks, seg.n_blocks_total - first_block);
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    DevBuf<int32_t> d_out;
    d_out.alloc(std::max<uint64_t>(1, n_blocks) * 2 * kBlock);
    if (out) RG_CUDA_CHECK(cudaMemsetAsync(d_out.p, 0, d_out.bytes(), st));
    RG_CUDA_CHECK(cudaEventRecord(e->ev0, st));
    launch_decode_segment(st, seg.arena.p, seg.blk_desc.p, (uint32_t)first_block, (uint32_t)n_blocks, d_out.p,
                          seg.dev.version, seg.dev.sb_mask);
    RG_CUDA_CHECK(cudaGetLastError());
    if (n_blocks) e->launches++;
    RG_CUDA_CHECK(cudaEventRecord(e->ev1, st));
    if (out) RG_CUDA_CHECK(cudaMemcpyAsync(out, d_out.p, n_blocks * 2 * kBlock * 4, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    RG_CUDA_CHECK(cudaEventElapsedTime(&e->last_decode_ms, e->ev0, e->ev1));
    stats[0] = seg.n_blocks_total ? seg.block_enc_bytes * n_blocks / seg.n_blocks_total : 0;  // pro rata
    stats[1] = n_blocks * 2 * kBlock * 4;
    stats[2] = n_blocks;
    stats[3] = seg.n_blocks_total;
    return RG_OK;
    RG_CATCH
}


static void table_to_header(int doc_version, const int32_t forutil_table[32], DocHeader& h) {
    if (!forutil_table) throw ArgError("forutil_table is null");
    if (doc_version < 0 || doc_version > 1) throw ArgError("doc_version must be 0 or 1");
    format_sizes(doc_version, forutil_table, h);
}

int rg_forutil_decode(rg_engine* e, const uint8_t* stream, size_t len, const uint64_t* offsets,
                      uint32_t n_blocks, int doc_version, const int32_t forutil_table[32],
                      int32_t* out) {
    RG_TRY
    if (!e || !stream || !offsets || !out) throw ArgError("null argument");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    DocHeader h;
    table_to_header(doc_version, forutil_table, h);
    for (uint32_t i = 0; i < n_blocks; i++) {  // bounds + header validation on the host
        if (offsets[i] >= len) throw ArgError("block offset out of range");
        int b = stream[offsets[i]] & 0x3f;
        if (b > 32) throw ArgError("corrupt block header");
        size_t need = b ? (size_t)1 + (size_t)h.enc_size[b] : 2;
        if (offsets[i] + need > len) throw ArgError("block runs past the end of the stream");
    }
    DevBuf<uint8_t> d_stream;
    DevBuf<uint64_t> d_off;
    DevBuf<int32_t> d_out;
    d_stream.alloc(len + 64);
    d_off.alloc(std::max<uint32_t>(n_blocks, 1));
    d_out.alloc((size_t)std::max<uint32_t>(n_blocks, 1) * kBlock);
    cudaStream_t st = e->stream;
    RG_CUDA_CHECK(cudaMemsetAsync(d_stream.p + len, 0, 64, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(d_stream.p, stream, len, cudaMemcpyHostToDevice, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(d_off.p, offsets, (size_t)n_blocks * 8, cudaMemcpyHostToDevice, st));
    RG_CUDA_CHECK(cudaEventRecord(e->ev0, st));
    launch_decode_raw(st, d_stream.p, d_off.p, n_blocks, d_out.p, h.version, h.sb_mask);
    RG_CUDA_CHECK(cudaGetLastError());
    if (n_blocks) e->launches++;
    RG_CUDA_CHECK(cudaEventRecord(e->ev1, st));
    RG_CUDA_CHECK(cudaMemcpyAsync(out, d_out.p, (size_t)n_blocks * kBlock * 4, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    RG_CUDA_CHECK(cudaEventElapsedTime(&e->last_decode_ms, e->ev0, e->ev1));
    return RG_OK;
    RG_CATCH
}

int rg_blockset_stage(rg_engine* e, const uint8_t* stream, size_t len, const uint64_t* offsets,
                      uint32_t n_blocks, int doc_version, const int32_t forutil_table[32],
                      rg_blockset** out) {
    RG_TRY
    if (!e || !stream || !offsets || !out) throw ArgError("null argument");
    RG_CUDA_CHECK(cudaSetDevice(e->device));
    DocHeader h;
    table_to_header(doc_version, forutil_table, h);
    std::unique_ptr<rg_blockset> bs(new rg_blockset());
    bs->n_blocks = n_blocks;
    bs->version = h.version;
    bs->sb_mask = h.sb_mask;
    std::vector<BlockDesc> desc(std::max<uint32_t>(n_blocks, 1));
    uint64_t units = 0;
    for (uint32_t i = 0; i < n_blocks; i++) {
        if (offsets[i] >= len) throw ArgError("block offset out of range");
        int b = stream[offsets[i]] & 0x3f;
        if (b > 32) throw ArgError("corrupt block header");
        int sz = b ? h.enc_size[b] : 0;
        if (offsets[i] + 1 + (size_t)(b ? sz : 1) > len) throw ArgError("block runs past the end of the stream");
        desc[i].off16 = (uint32_t)units;
        desc[i].bits = (uint32_t)b | (part_units(sz) << 16);
        units += part_units(sz);
        if (units >= (1ull << 32)) throw Unsupported("block set exceeds 64 GiB");
    }
    std::vector<uint4> arena(units + 8);
    parallel_chunks((n_blocks + 65535) / 65536, [&](size_t c) {
        uint32_t end = (uint32_t)std::min<uint64_t>(n_blocks, (c + 1) * 65536ull);
        for (uint32_t i = (uint32_t)(c * 65536ull); i < end; i++) {
            const uint8_t* p = stream + offsets[i];
            int b = p[0] & 0x3f;
            uint8_t* dst = reinterpret_cast<uint8_t*>(&arena[desc[i].off16]);
            if (b) {
                memcpy(dst, p + 1, (size_t)h.enc_size[b]);
            } else {
                In in(stream, len, (size_t)offsets[i] + 1);
                int32_t v = in.vint();
                memcpy(dst, &v, 4);
            }
        }
    });
    for (uint32_t i = 0; i < n_blocks; i++) {
        int b = desc[i].bits & 0xff;
        if (b) bs->enc_bytes += 1 + (uint64_t)h.enc_size[b];
        else {
            In in(stream, len, (size_t)offsets[i] + 1);
            size_t p0 = in.pos;
            in.vint();
            bs->enc_bytes += 1 + (in.pos - p0);
        }
    }
    cudaStream_t st = e->stream;
    upload(bs->arena, arena.data(), arena.size(), st);
    upload(bs->desc, desc.data(), desc.size(), st);
    bs->out.alloc((size_t)std::max<uint32_t>(n_blocks, 1) * kBlock);
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    *out = bs.release();
    return RG_OK;
    RG_CATCH
}

int rg_blockset_decode(rg_engine* e, rg_blockset* bs) {
    RG_TRY
    if (!e || !bs) throw ArgError("null argument");
    cudaStream_t st = e->stream;
    RG_CUDA_CHECK(cudaEventRecord(e->ev0, st));
    launch_decode_staged(st, bs->arena.p, bs->desc.p, bs->n_blocks, bs->out.p, bs->version, bs->sb_mask);
    RG_CUDA_CHECK(cudaGetLastError());
    if (bs->n_blocks) e->launches++;
    RG_CUDA_CHECK(cudaEventRecord(e->ev1, st));
    return RG_OK;
    RG_CATCH
}

int rg_blockset_fetch(rg_engine* e, rg_blockset* bs, int32_t* out) {
    RG_TRY
    if (!e || !bs || !out) throw ArgError("null argument");
    cudaStream_t st = e->stream;
    RG_CUDA_CHECK(cudaMemcpyAsync(out, bs->out.p, (size_t)bs->n_blocks * kBlock * 4, cudaMemcpyDeviceToHost, st));
    RG_CUDA_CHECK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&e->last_decode_ms, e->ev0, e->ev1);
    cudaGetLastError();
    return RG_OK;
    RG_CATCH
}

int rg_blockset_stats(rg_engine*, rg_blockset* bs, uint64_t out[4]) {
    if (!bs || !out) return RG_EINVAL;
    out[0] = bs->enc_bytes;
    out[1] = (uint64_t)bs->n_blocks * 512;
    out[2] = bs->n_blocks;
    out[3] = bs->arena.bytes() + bs->desc.bytes();
    return RG_OK;
}

void rg_blockset_destroy(rg_engine*, rg_blockset* bs) { delete bs; }

}  // extern "C"
