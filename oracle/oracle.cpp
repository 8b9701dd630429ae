/*
 * oracle.cpp — CPU restatement of zhihu/rucene's IndexSearcher hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  Every function cites the reference
 * file:line it follows; paths are relative to src/core/ of zhihu/rucene.
 * Compile with -ffp-contract=off: the reference (rustc) never contracts a*b+c
 * into an FMA and BM25 bit-exactness depends on that.
 *
 * Not a copy: the reference is Rust with trait objects, macro-unrolled SSE and
 * mmap inputs; this is a from-scratch C++ restatement of the same algorithms.
 */
#include "oracle.h"

#include <emmintrin.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

namespace orc {

constexpr int BLOCK_SIZE = 128;          // codec/postings/posting_format.rs
constexpr int MAX_DATA_SIZE = 147;       // codec/postings/for_util.rs:42
constexpr int MAX_ENCODED_SIZE = 512;    // for_util.rs:33
constexpr int32_t NO_MORE_DOCS = INT32_MAX;  // search/mod.rs:59
constexpr int MAX_SKIP_LEVELS = 10;      // posting_reader.rs:49

static thread_local std::string g_err;

struct Error : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// ---------------------------------------------------------------------------
// store/io/data_input.rs:78-111 (vint), :127- (vlong); big-endian ints :58-76
// ---------------------------------------------------------------------------
struct Input {
    const uint8_t* base = nullptr;
    int64_t len = 0;
    int64_t pos = 0;
    Input() = default;
    Input(const uint8_t* b, int64_t l, int64_t p = 0) : base(b), len(l), pos(p) {}
    uint8_t read_byte() {
        if (pos >= len) throw Error("read past EOF");
        return base[pos++];
    }
    int32_t read_vint() {
        int8_t b = (int8_t)read_byte();
        if (b >= 0) return b;
        int32_t i = b & 0x7f;
        b = (int8_t)read_byte();
        i |= (b & 0x7f) << 7;
        if (b >= 0) return i;
        b = (int8_t)read_byte();
        i |= (b & 0x7f) << 14;
        if (b >= 0) return i;
        b = (int8_t)read_byte();
        i |= (b & 0x7f) << 21;
        if (b >= 0) return i;
        b = (int8_t)read_byte();
        i |= (int32_t)((uint32_t)(b & 0x0f) << 28);
        if (((uint8_t)b & 0xf0) != 0) throw Error("Invalid vInt detected");
        return i;
    }
    int64_t read_vlong() {
        int64_t v = 0;
        for (int shift = 0; shift < 63; shift += 7) {
            int8_t b = (int8_t)read_byte();
            v |= (int64_t)(b & 0x7f) << shift;
            if (b >= 0) return v;
        }
        throw Error("Invalid vLong detected");
    }
    int32_t read_int() {
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) v = (v << 8) | read_byte();
        return (int32_t)v;
    }
    int64_t read_long() {
        uint64_t v = 0;
        for (int i = 0; i < 8; i++) v = (v << 8) | read_byte();
        return (int64_t)v;
    }
    void seek(int64_t p) {
        if (p < 0 || p > len) throw Error("seek out of range");
        pos = p;
    }
    int64_t file_pointer() const { return pos; }
    // store/io/mmap_index_input.rs:246-251 — zero-copy window
    const uint8_t* get_and_advance(size_t n) {
        if (pos + (int64_t)n > len) throw Error("read past EOF");
        const uint8_t* p = base + pos;
        pos += (int64_t)n;
        return p;
    }
    void read_exact(uint8_t* dst, size_t n) { std::memcpy(dst, get_and_advance(n), n); }
};

// ---------------------------------------------------------------------------
// util/packed/packed_simd.rs:81-163 — SIMD128Packer, 4-lane interleaved codec.
// TRANSFER: 0 none, 1 delta (trans_to_delta / trans_from_delta :347-374)
// ---------------------------------------------------------------------------
struct DeltaState {
    uint32_t base;
};

static inline __m128i to_delta(DeltaState& st, __m128i data) {  // packed_simd.rs:347-361
    __m128i prev = _mm_or_si128(_mm_slli_si128(data, 4), _mm_set_epi32(0, 0, 0, (int)st.base));
    __m128i deltas = _mm_sub_epi32(data, prev);
    st.base = (uint32_t)_mm_cvtsi128_si32(_mm_srli_si128(data, 12));
    return deltas;
}
static inline __m128i from_delta(DeltaState& st, __m128i delta) {  // packed_simd.rs:363-374
    __m128i a = _mm_add_epi32(delta, _mm_slli_si128(delta, 4));
    __m128i b = _mm_add_epi32(a, _mm_slli_si128(a, 8));
    __m128i v = _mm_add_epi32(b, _mm_set1_epi32((int)st.base));
    st.base = (uint32_t)_mm_cvtsi128_si32(_mm_srli_si128(v, 12));
    return v;
}

template <int B, bool DELTA>
static void simd_pack_t(const uint32_t* data, uint8_t* enc, DeltaState* st) {  // :81-108
    const __m128i* in = (const __m128i*)data;
    __m128i* out = (__m128i*)enc;
    __m128i buffer = _mm_setzero_si128();
#pragma GCC unroll 32
    for (int i = 0; i < 32; i++) {
        __m128i v = _mm_loadu_si128(in + i);
        if (DELTA) v = to_delta(*st, v);
        const int inner_pos = i * B % 32;
        buffer = _mm_or_si128(buffer, _mm_slli_epi32(v, inner_pos));
        const int new_pos = inner_pos + B;
        if (new_pos >= 32) {
            _mm_storeu_si128(out++, buffer);
            buffer = (new_pos > 32) ? _mm_srli_epi32(v, 32 - inner_pos) : _mm_setzero_si128();
        }
    }
}

template <int B, bool DELTA>
static void simd_unpack_t(const uint8_t* enc, uint32_t* data, DeltaState* st) {  // :126-163
    const __m128i* in = (const __m128i*)enc;
    __m128i* out = (__m128i*)data;
    const __m128i mask = _mm_set1_epi32((int)((1u << B) - 1));
    __m128i buffer = _mm_loadu_si128(in);
#pragma GCC unroll 32
    for (int i = 0; i < 32; i++) {
        const int inner_pos = i * B % 32;
        const int new_pos = inner_pos + B;
        __m128i v;
        if (new_pos >= 32) {
            in++;
            if (new_pos == 32) {
                v = buffer;
                // the reference re-loads here even after the last vector (i==31), reading 16
                // bytes beyond the payload; the value is never used, so we skip that read.
                if (i < 31) buffer = _mm_loadu_si128(in);
            } else {
                const int remain = 32 - inner_pos;
                __m128i temp = _mm_loadu_si128(in);
                v = _mm_and_si128(_mm_or_si128(buffer, _mm_slli_epi32(temp, remain)), mask);
                buffer = _mm_srli_epi32(temp, B - remain);
            }
        } else {
            v = _mm_and_si128(buffer, mask);
            buffer = _mm_srli_epi32(buffer, B);
        }
        if (DELTA) v = from_delta(*st, v);
        _mm_storeu_si128(out + i, v);
    }
}

template <bool DELTA>
static void simd_pack(const uint32_t* data, uint8_t* enc, int bits, DeltaState* st) {  // :169-207
    switch (bits) {
#define C(N) case N: simd_pack_t<N, DELTA>(data, enc, st); break;
        C(1) C(2) C(3) C(4) C(5) C(6) C(7) C(8) C(9) C(10) C(11) C(12) C(13) C(14) C(15) C(16)
        C(17) C(18) C(19) C(20) C(21) C(22) C(23) C(24) C(25) C(26) C(27) C(28) C(29) C(30) C(31)
#undef C
        case 32: std::memcpy(enc, data, 512); break;  // direct_copy_to :57-59
        case 0: break;
        default: throw Error("simd pack: bits > 32");
    }
}
template <bool DELTA>
static void simd_unpack(const uint8_t* enc, uint32_t* data, int bits, DeltaState* st) {  // :209-252
    switch (bits) {
#define C(N) case N: simd_unpack_t<N, DELTA>(enc, data, st); break;
        C(1) C(2) C(3) C(4) C(5) C(6) C(7) C(8) C(9) C(10) C(11) C(12) C(13) C(14) C(15) C(16)
        C(17) C(18) C(19) C(20) C(21) C(22) C(23) C(24) C(25) C(26) C(27) C(28) C(29) C(30) C(31)
#undef C
        case 32: std::memcpy(data, enc, 512); break;  // direct_copy_from :61-65
        case 0: break;
        default: throw Error("simd unpack: bits > 32");
    }
}

static int simd_max_bits(const uint32_t* data) {  // packed_simd.rs:376-392
    uint32_t r = 0;
    for (int i = 0; i < 128; i++) r |= data[i];
    return r == 0 ? 0 : 32 - __builtin_clz(r);
}

// ---------------------------------------------------------------------------
// util/packed/packed_misc.rs — Format (:380-466), FormatAndBits::fastest (:474-531),
// BulkOperationPacked (:2405-2446, decode :2655-2680, encode :2556-2582),
// BulkOperationPackedSingleBlock (:2686-2777, :2829-2875)
// ---------------------------------------------------------------------------
enum Format { PACKED = 0, PACKED_SINGLE_BLOCK = 1 };

static bool single_block_supported(int bpv) {  // Packed64SingleBlock::is_supported
    static const int ok[] = {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 16, 21, 32};
    for (int v : ok)
        if (v == bpv) return true;
    return false;
}

static int64_t format_byte_count(int format, int value_count, int bpv) {  // :403-418
    if (format == PACKED) return ((int64_t)value_count * bpv + 7) / 8;
    int vpb = 64 / bpv;
    return (int64_t)((value_count + vpb - 1) / vpb) * 8;
}

static float overhead_per_value(int format, int bpv) {  // :449-458
    if (format == PACKED) return 0.f;
    int vpb = 64 / bpv;
    int overhead = 64 % bpv;
    return (float)overhead / (float)vpb;
}

static void fastest_format(int value_count, int bpv, float ratio, int* out_format,
                           int* out_bpv) {  // :484-531
    if (value_count == -1) value_count = INT32_MAX;
    ratio = std::max(0.0f, ratio);
    ratio = std::min(7.0f, ratio);
    float per_value = ratio * (float)bpv;
    int max_bpv = bpv + (int)per_value;
    int actual = -1;
    int format = PACKED;
    const int three_blocks_max = INT32_MAX / 3;
    if (bpv <= 8 && max_bpv >= 8) actual = 8;
    else if (bpv <= 16 && max_bpv >= 16) actual = 16;
    else if (bpv <= 32 && max_bpv >= 32) actual = 32;
    else if (bpv <= 64 && max_bpv >= 64) actual = 64;
    else if (value_count <= three_blocks_max && bpv <= 24 && max_bpv >= 24) actual = 24;
    else if (value_count <= three_blocks_max && bpv <= 48 && max_bpv >= 48) actual = 48;
    else {
        for (int b = bpv; b <= max_bpv; b++) {
            if (single_block_supported(b)) {
                float overhead = overhead_per_value(PACKED_SINGLE_BLOCK, b);
                float acceptable = per_value + (float)bpv - (float)b;
                if (overhead <= acceptable) {
                    actual = b;
                    format = PACKED_SINGLE_BLOCK;
                    break;
                }
            }
        }
        if (actual < 0) actual = bpv;
    }
    *out_format = format;
    *out_bpv = actual;
}

struct BulkOp {
    int format = PACKED;
    int bpv = 0;
    // Packed
    int byte_block_count = 0, byte_value_count_ = 0;
    int32_t int_mask = 0;
    // SingleBlock
    int value_count = 0;
    int64_t mask64 = 0;

    static BulkOp make(int format, int bpv) {
        BulkOp op;
        op.format = format;
        op.bpv = bpv;
        if (format == PACKED) {  // :2424-2453
            int blocks = bpv;
            while ((blocks & 1) == 0) blocks >>= 1;
            int long_value_count = 64 * blocks / bpv;
            int bbc = 8 * blocks, bvc = long_value_count;
            while ((bbc & 1) == 0 && (bvc & 1) == 0) {
                bbc >>= 1;
                bvc >>= 1;
            }
            op.byte_block_count = bbc;
            op.byte_value_count_ = bvc;
            int64_t mask = bpv == 64 ? -1 : (int64_t)(((uint64_t)1 << bpv) - 1);
            op.int_mask = (int32_t)mask;
        } else {  // :2694-2701 (bulk_operation_of :2379-2387 does no is_supported check)
            op.value_count = 64 / bpv;
            op.mask64 = ((int64_t)1 << bpv) - 1;
        }
        return op;
    }
    int byte_value_count() const { return format == PACKED ? byte_value_count_ : value_count; }
    int bytes_per_iteration() const { return format == PACKED ? byte_block_count : 8; }

    // decode_byte_to_int — Packed :2655-2680, SingleBlock :2829-2841 (+ :2739-2755, :2700-2709)
    int decode(const uint8_t* blocks, int32_t* values, int iterations) const {
        int vo = 0;
        if (format == PACKED) {
            int32_t next_value = 0;
            int bits_left = bpv;
            int bo = 0;
            for (int i = 0; i < iterations * byte_block_count; i++) {
                int32_t bytes = blocks[bo++];
                if (bits_left > 8) {
                    bits_left -= 8;
                    next_value |= (int32_t)((uint32_t)bytes << bits_left);
                } else {
                    int bits = 8 - bits_left;
                    values[vo++] = next_value | (bytes >> bits);
                    while (bits >= bpv) {
                        bits -= bpv;
                        values[vo++] = (bytes >> bits) & int_mask;
                    }
                    bits_left = bpv - bits;
                    next_value = (int32_t)((uint32_t)(bytes & ((1 << bits) - 1)) << bits_left);
                }
            }
        } else {
            for (int i = 0; i < iterations; i++) {
                uint64_t block = 0;
                for (int k = 0; k < 8; k++) block = (block << 8) | blocks[i * 8 + k];
                values[vo++] = (int32_t)((int64_t)block & mask64);
                for (int k = 1; k < value_count; k++) {
                    block >>= bpv;
                    values[vo++] = (int32_t)((int64_t)block & mask64);
                }
            }
        }
        return vo;
    }
    // encode_int_to_byte — Packed :2556-2582, SingleBlock :2866-2875 (+ :2768-2777, :2711-2718)
    int encode(const int32_t* values, uint8_t* blocks, int iterations) const {
        int bo = 0;
        if (format == PACKED) {
            int32_t next_block = 0;
            int bits_left = 8;
            int vo = 0;
            for (int i = 0; i < byte_value_count_ * iterations; i++) {
                uint32_t v = (uint32_t)values[vo++];
                if (bpv < bits_left) {
                    next_block |= (int32_t)(v << (bits_left - bpv));
                    bits_left -= bpv;
                } else {
                    int bits = bpv - bits_left;
                    blocks[bo++] = (uint8_t)(next_block | (int32_t)(v >> bits));
                    while (bits >= 8) {
                        bits -= 8;
                        blocks[bo++] = (uint8_t)(v >> bits);
                    }
                    bits_left = 8 - bits;
                    next_block = (int32_t)((v & ((1u << bits) - 1)) << bits_left);
                }
            }
        } else {
            for (int i = 0; i < iterations; i++) {
                uint64_t block = (uint32_t)values[i * value_count];
                for (int k = 1; k < value_count; k++)
                    block |= (uint64_t)(uint32_t)values[i * value_count + k] << (k * bpv);
                for (int k = 1; k <= 8; k++) blocks[bo++] = (uint8_t)(block >> (64 - (k << 3)));
            }
        }
        return bo;
    }
};

static int compute_iterations(const BulkOp& op) {  // for_util.rs:60-62
    return (int)std::ceil((float)BLOCK_SIZE / (float)op.byte_value_count());
}

static int max_data_size() {  // for_util.rs:64-97
    int m = 0;
    for (int format = 0; format < 2; format++)
        for (int bpv = 1; bpv <= 32; bpv++) {
            BulkOp op = BulkOp::make(format, bpv);
            m = std::max(m, compute_iterations(op) * op.byte_value_count());
        }
    return m;
}

// ---------------------------------------------------------------------------
// codec/postings/for_util.rs:103-148 (with_input), :187-243 (read_block), :263-272 (skip_block)
// ---------------------------------------------------------------------------
enum EncodeType { PF = 0, EF = 1, BITSET = 2, FULL = 3 };

struct ForUtil {
    int encoded_sizes[32];
    int iterations[32];
    BulkOp decoders[32];

    void init_from_codes(const int32_t codes[32]) {
        for (int i = 0; i < 32; i++) {
            int code = codes[i];
            int format_id = code >> 5;
            int bpv = (code & 31) + 1;
            if (format_id != PACKED && format_id != PACKED_SINGLE_BLOCK)
                throw Error("Invalid format id");
            encoded_sizes[i] = (int)format_byte_count(format_id, BLOCK_SIZE, bpv);
            decoders[i] = BulkOp::make(format_id, bpv);
            iterations[i] = compute_iterations(decoders[i]);
        }
    }
    void with_input(Input& in) {  // :120-148
        int v = in.read_vint();
        if (v != 2) throw Error("PackedInts version must be 2");  // packed_misc.rs:47-68
        int32_t codes[32];
        for (int i = 0; i < 32; i++) codes[i] = in.read_vint();
        init_from_codes(codes);
    }
    // read_block :187-243.  encode_type != nullptr only for doc-delta blocks.
    void read_block(Input& in, uint8_t* encoded, int32_t* decoded, EncodeType* encode_type,
                    bool by_simd) const {
        uint8_t code = in.read_byte();
        if (encode_type) {
            EncodeType et = (EncodeType)(code >> 6);
            if (et != PF) {
                *encode_type = et;
                return;
            }
        }
        int num_bits = code & 0x3F;
        if (num_bits > 32) throw Error("corrupt block header");
        if (num_bits == 0) {  // ALL_VALUES_EQUAL
            int32_t value = in.read_vint();
            for (int i = 0; i < BLOCK_SIZE; i++) decoded[i] = value;
            return;
        }
        if (by_simd) {
            const uint8_t* enc = in.get_and_advance((size_t)num_bits * BLOCK_SIZE / 8);
            simd_unpack<false>(enc, (uint32_t*)decoded, num_bits, nullptr);
        } else {
            int esz = encoded_sizes[num_bits - 1];
            in.read_exact(encoded, (size_t)esz);
            decoders[num_bits - 1].decode(encoded, decoded, iterations[num_bits - 1]);
        }
    }
    void skip_block(Input& in) const {  // :263-272
        int num_bits = in.read_byte();
        if (num_bits == 0) {
            in.read_vint();
            return;
        }
        if (num_bits > 32) throw Error("corrupt block header");
        in.seek(in.file_pointer() + encoded_sizes[num_bits - 1]);
    }
};

// ---------------------------------------------------------------------------
// codec/postings/skip_reader.rs — Lucene50SkipReader (docs-only fields)
// ---------------------------------------------------------------------------
static int ilog(int64_t x, int base) {  // util/math.rs:21-32
    int ret = 0;
    while (x >= base) {
        x /= base;
        ret++;
    }
    return ret;
}

struct SkipReader {
    int max_levels = MAX_SKIP_LEVELS;
    int number_of_skip_levels = 0;
    int number_of_levels_to_buffer = 1;
    int doc_count = 0;
    Input stream[MAX_SKIP_LEVELS];
    bool has_stream[MAX_SKIP_LEVELS];
    int64_t skip_pointer[MAX_SKIP_LEVELS];
    int64_t skip_interval[MAX_SKIP_LEVELS];
    int64_t num_skipped[MAX_SKIP_LEVELS];
    int32_t skip_doc[MAX_SKIP_LEVELS];
    int32_t last_doc = 0;
    int64_t child_pointer[MAX_SKIP_LEVELS];
    int64_t last_child_pointer = 0;
    int64_t doc_pointer[MAX_SKIP_LEVELS];
    int64_t last_doc_pointer = 0;

    explicit SkipReader(const Input& base_stream) {  // :222-299
        for (int i = 0; i < MAX_SKIP_LEVELS; i++) {
            has_stream[i] = false;
            skip_pointer[i] = child_pointer[i] = num_skipped[i] = 0;
            skip_doc[i] = 0;
            doc_pointer[i] = 0;
            skip_interval[i] = i == 0 ? BLOCK_SIZE : skip_interval[i - 1] * 8;
        }
        stream[0] = base_stream;
        has_stream[0] = true;
    }
    static int trim(int df) { return df % BLOCK_SIZE == 0 ? df - 1 : df; }  // :307-313

    void init(int64_t skip_ptr, int64_t doc_base_pointer, int df) {  // :315-356
        df = trim(df);
        skip_pointer[0] = skip_ptr;
        doc_count = df;
        for (int i = 0; i < MAX_SKIP_LEVELS; i++) {
            skip_doc[i] = 0;
            num_skipped[i] = 0;
            child_pointer[i] = 0;
        }
        for (int i = 1; i < number_of_skip_levels; i++) has_stream[i] = false;
        load_skip_levels();
        last_doc_pointer = doc_base_pointer;
        for (int i = 0; i < MAX_SKIP_LEVELS; i++) doc_pointer[i] = doc_base_pointer;
    }
    void load_skip_levels() {  // :460-511
        if ((int64_t)doc_count <= skip_interval[0]) number_of_skip_levels = 1;
        else number_of_skip_levels = 1 + ilog((int64_t)doc_count / skip_interval[0], 8);
        if (number_of_skip_levels > max_levels) number_of_skip_levels = max_levels;
        stream[0].seek(skip_pointer[0]);
        int to_buffer = number_of_levels_to_buffer;
        for (int i = number_of_skip_levels - 1; i >= 1; i--) {
            int64_t length = stream[0].read_vlong();
            skip_pointer[i] = stream[0].file_pointer();
            // buffered (SkipBuffer :24-92) and cloned streams both address the level by
            // absolute file position, so one representation serves both branches.
            stream[i] = stream[0];
            has_stream[i] = true;
            if (to_buffer > 0) to_buffer--;
            stream[0].seek(stream[0].file_pointer() + length);
        }
        skip_pointer[0] = stream[0].file_pointer();
    }
    int32_t read_skip_data(int level) {  // :431-453 (no positions/payloads)
        int32_t delta = stream[level].read_vint();
        int64_t pointer = stream[level].read_vlong();
        doc_pointer[level] += pointer;
        return delta;
    }
    void set_last_skip_data(int level) {  // :410-429
        last_doc = skip_doc[level];
        last_child_pointer = child_pointer[level];
        last_doc_pointer = doc_pointer[level];
    }
    void seek_child(int level) {  // :385-408
        stream[level].seek(last_child_pointer);
        num_skipped[level] = num_skipped[level + 1] - skip_interval[level + 1];
        skip_doc[level] = last_doc;
        if (level > 0) child_pointer[level] = stream[level].read_vlong() + skip_pointer[level - 1];
        doc_pointer[level] = last_doc_pointer;
    }
    bool load_next_skip(int level) {  // :513-539
        set_last_skip_data(level);
        num_skipped[level] += skip_interval[level];
        if (num_skipped[level] > (int64_t)doc_count) {
            skip_doc[level] = INT32_MAX;
            if (number_of_skip_levels > level) number_of_skip_levels = level;
            return false;
        }
        skip_doc[level] += read_skip_data(level);
        if (level != 0) child_pointer[level] = stream[level].read_vlong() + skip_pointer[level - 1];
        return true;
    }
    int32_t skip_to(int32_t target) {  // :554-584
        int level = 0;
        while (level < number_of_skip_levels - 1 && target > skip_doc[level + 1]) level++;
        while (level >= 0) {
            if (target > skip_doc[level]) {
                if (!load_next_skip(level)) continue;
            } else {
                if (level > 0 && last_child_pointer > stream[level - 1].file_pointer())
                    seek_child(level - 1);
                level--;
            }
        }
        return (int32_t)(num_skipped[0] - skip_interval[0] - 1);
    }
    int32_t doc() const { return last_doc; }
    int64_t doc_ptr() const { return last_doc_pointer; }
    int32_t next_skip_doc() const { return skip_doc[0]; }
};

// ---------------------------------------------------------------------------
// Scorer / DocIterator — search/mod.rs:66-156, search/scorer/mod.rs:85-99
// ---------------------------------------------------------------------------
struct Scorer {
    virtual ~Scorer() = default;
    virtual int32_t doc_id() const = 0;
    virtual int32_t next() = 0;
    virtual int32_t advance(int32_t target) = 0;
    virtual size_t cost() const = 0;
    virtual float score() = 0;
};
using ScorerPtr = std::unique_ptr<Scorer>;

// ---------------------------------------------------------------------------
// codec/postings/posting_reader.rs:343-794 — BlockDocIterator (PF blocks)
// ---------------------------------------------------------------------------
// util/packed/elias_fano_encoder.rs:24-146,255-262 (read side: geometry + the three long arrays),
// util/packed/elias_fano_decoder.rs:23-330 (next_value / advance_to_value / current_index),
// util/bit_set.rs:193-251,351-376,453-460 (FixedBitSet pieces the BITSET blocks use).
// The open-source writer never emits these blocks (EfWriterMeta.use_ef is never set,
// posting_writer.rs:46) but the reader handles them (posting_reader.rs:501-561,612-647,649-789).
// ---------------------------------------------------------------------------
static const int64_t NO_MORE_VALUES = -1;
static inline int64_t ushr64(int64_t x, int n) { return (int64_t)((uint64_t)x >> n); }
static inline int clz64(int64_t x) { return x == 0 ? 64 : __builtin_clzll((uint64_t)x); }
static inline int ctz64(int64_t x) { return x == 0 ? 64 : __builtin_ctzll((uint64_t)x); }
static inline int popc64(int64_t x) { return __builtin_popcountll((uint64_t)x); }

struct EliasFanoEncoder {  // as rebuilt by get_encoder / rebuild_not_with_check + deserialize2
    int64_t num_values = 0, upper_bound = 0;
    int num_low_bits = 0;
    int64_t lower_bits_mask = 0;
    std::vector<int64_t> upper_longs, lower_longs, upper_zero_bit_position_index;
    int64_t num_encoded = 0, last_encoded = 0;
    int64_t num_index_entries = 0, index_interval = 256;
    int n_index_entry_bits = 0;
    static int64_t num_longs_for_bits(int64_t n) { return ushr64(n + 63, 6); }  // :308-311
    void rebuild(int64_t nv, int64_t ub) {  // :48-146 and :148-205 agree on every derived field
        num_values = nv;
        upper_bound = ub;
        num_encoded = nv;
        last_encoded = ub;
        num_low_bits = 0;
        if (nv > 0) {
            int64_t fac = ub / nv;
            if (fac > 0) num_low_bits = 64 - 1 - clz64(fac);
        }
        lower_bits_mask = ushr64(INT64_MAX, 64 - 1 - num_low_bits);
        lower_longs.assign((size_t)num_longs_for_bits(nv * num_low_bits), 0);
        upper_longs.assign((size_t)num_longs_for_bits(ushr64(ub, num_low_bits) + nv), 0);
        int64_t max_high_value = ushr64(ub, num_low_bits);
        int64_t n_entries = max_high_value / index_interval;
        num_index_entries = n_entries >= 0 ? n_entries : 0;
        int64_t max_index_entry = max_high_value + nv - 1;
        n_index_entry_bits = max_index_entry <= 0 ? 0 : 64 - clz64(max_index_entry);
        upper_zero_bit_position_index.assign((size_t)num_longs_for_bits(num_index_entries * n_index_entry_bits), 0);
    }
    static void read_data2(std::vector<int64_t>& buf, Input& in) {  // :367-374: raw little-endian memory
        for (auto& x : buf) {
            uint8_t b[8];
            in.read_exact(b, 8);
            uint64_t v = 0;
            for (int i = 0; i < 8; i++) v |= (uint64_t)b[i] << (8 * i);
            x = (int64_t)v;
        }
    }
    void deserialize2(Input& in) {  // :278-285
        num_encoded = num_values;
        last_encoded = upper_bound;
        read_data2(upper_longs, in);
        read_data2(lower_longs, in);
        read_data2(upper_zero_bit_position_index, in);
    }
};

struct EliasFanoDecoder {
    const EliasFanoEncoder* e = nullptr;
    int64_t num_encoded = 0, ef_index = -1, set_bit_for_index = -1, num_index_entries = 0, index_mask = 0;
    int64_t cur_high_long = 0;
    void refresh(const EliasFanoEncoder* enc) {  // new() :36-46
        e = enc;
        num_encoded = enc->num_encoded;
        ef_index = -1;
        set_bit_for_index = -1;
        num_index_entries = enc->num_index_entries;
        index_mask = ((int64_t)1 << enc->n_index_entry_bits) - 1;
        cur_high_long = 0;
    }
    int64_t current_index() const {  // :60-68
        if (ef_index < 0) throw Error("index before sequence");
        if (ef_index >= num_encoded) throw Error("index after sequence");
        return ef_index;
    }
    static int64_t unpack_value(const std::vector<int64_t>& a, int num_bits, int64_t pack_index, int64_t mask) {
        if (num_bits == 0) return 0;  // :96-108
        int64_t bit_pos = pack_index * num_bits;
        size_t index = (size_t)ushr64(bit_pos, 6);
        int bit_pos_at_index = (int)(bit_pos & 63);
        int64_t value = ushr64(a.at(index), bit_pos_at_index);
        if (bit_pos_at_index + num_bits > 64) value |= (int64_t)((uint64_t)a.at(index + 1) << (64 - bit_pos_at_index));
        return value & mask;
    }
    int64_t current_low_value() const { return unpack_value(e->lower_longs, e->num_low_bits, ef_index, e->lower_bits_mask); }
    int64_t combine(int64_t high, int64_t low) const { return (int64_t)((uint64_t)high << e->num_low_bits) | low; }
    bool to_after_current_high_bit() {  // :122-134
        ef_index++;
        if (ef_index >= num_encoded) return false;
        set_bit_for_index++;
        size_t hi = (size_t)ushr64(set_bit_for_index, 6);
        cur_high_long = ushr64(e->upper_longs.at(hi), (int)(set_bit_for_index & 63));
        return true;
    }
    void to_next_high_long() {  // :136-142
        set_bit_for_index += 64 - (set_bit_for_index & 63);
        cur_high_long = e->upper_longs.at((size_t)ushr64(set_bit_for_index, 6));
    }
    void to_next_high_value() {  // :143-148
        while (cur_high_long == 0) to_next_high_long();
        set_bit_for_index += ctz64(cur_high_long);
    }
    int64_t next_value() {  // :154-160
        if (!to_after_current_high_bit()) return NO_MORE_VALUES;
        to_next_high_value();
        return combine(set_bit_for_index - ef_index, current_low_value());
    }
    static int select_bit(int64_t x, int r) {  // bit_util.rs:215-248: index of the r-th 1 bit, -1 if none
        int s = -1;
        uint64_t u = (uint64_t)x;
        while (u != 0 && r > 0) {
            int ntz = __builtin_ctzll(u);
            u = ntz + 1 >= 64 ? 0 : u >> (ntz + 1);
            s += ntz + 1;
            r--;
        }
        return r > 0 ? -1 : s;
    }
    int64_t advance_to_value(int64_t target) {  // :186-318
        ef_index++;
        if (ef_index >= num_encoded) return NO_MORE_VALUES;
        set_bit_for_index++;
        size_t high_index = (size_t)ushr64(set_bit_for_index, 6);
        int64_t upper_long = e->upper_longs.at(high_index);
        cur_high_long = ushr64(upper_long, (int)(set_bit_for_index & 63));
        int64_t high_target = ushr64(target, e->num_low_bits);
        int64_t index_entry_index = (high_target / e->index_interval) - 1;
        if (index_entry_index >= 0) {
            if (index_entry_index >= num_index_entries) index_entry_index = num_index_entries - 1;
            int64_t index_high_value = (index_entry_index + 1) * e->index_interval;
            if (index_high_value > high_target) throw Error("ef: index_high_value > high_target");
            if (index_high_value > (set_bit_for_index - ef_index)) {
                set_bit_for_index = unpack_value(e->upper_zero_bit_position_index, e->n_index_entry_bits,
                                                 index_entry_index, index_mask);
                ef_index = set_bit_for_index - index_high_value;
                high_index = (size_t)ushr64(set_bit_for_index, 6);
                upper_long = e->upper_longs.at(high_index);
                cur_high_long = ushr64(upper_long, (int)(set_bit_for_index & 63));
            }
            if (!(ef_index < num_encoded)) throw Error("ef: index past the sequence");
        }
        int cur_set_bits = popc64(cur_high_long);
        int cur_clear_bits = 64 - cur_set_bits - (int)(set_bit_for_index & 63);
        while ((set_bit_for_index - ef_index + cur_clear_bits) < high_target) {
            ef_index += cur_set_bits;
            if (ef_index >= num_encoded) return NO_MORE_VALUES;
            set_bit_for_index += 64 - (set_bit_for_index & 63);
            high_index++;
            upper_long = e->upper_longs.at(high_index);
            cur_high_long = upper_long;
            cur_set_bits = popc64(cur_high_long);
            cur_clear_bits = 64 - cur_set_bits;
        }
        while (cur_high_long == 0) {
            set_bit_for_index += 64 - (set_bit_for_index & 63);
            high_index++;
            upper_long = e->upper_longs.at(high_index);
            cur_high_long = upper_long;
        }
        int rank = (int)(high_target - (set_bit_for_index - ef_index));
        if (rank > 64) throw Error("ef: rank > 64");
        if (rank >= 1) {
            int clear_bit_for_value = select_bit(~cur_high_long, rank);
            if (clear_bit_for_value < 0 || clear_bit_for_value > 63) throw Error("ef: select failed");
            set_bit_for_index += clear_bit_for_value + 1;
            int one_bits_before_clear_bit = clear_bit_for_value - rank + 1;
            ef_index += one_bits_before_clear_bit;
            if (ef_index >= num_encoded) return NO_MORE_VALUES;
            if ((set_bit_for_index & 63) == 0) {
                high_index++;
                upper_long = e->upper_longs.at(high_index);
                cur_high_long = upper_long;
            } else {
                cur_high_long = ushr64(upper_long, (int)(set_bit_for_index & 63));
            }
            while (cur_high_long == 0) {
                set_bit_for_index += 64 - (set_bit_for_index & 63);
                high_index++;
                upper_long = e->upper_longs.at(high_index);
                cur_high_long = upper_long;
            }
        }
        set_bit_for_index += ctz64(cur_high_long);
        int64_t current_value = combine(set_bit_for_index - ef_index, current_low_value());
        while (current_value < target) {
            current_value = next_value();
            if (current_value == NO_MORE_VALUES) return NO_MORE_VALUES;
        }
        return current_value;
    }
};

struct FixedBitSet {
    std::vector<int64_t> bits;
    size_t num_bits = 0, num_words = 0;
    static size_t bits2words(size_t n) { return (size_t)((((int32_t)n - 1) >> 6) + 1); }  // :480-484
    void resize(size_t n) {  // :193-200
        size_t w = bits2words(n);
        if (w != bits.size()) {
            bits.resize(w, 0);
            num_words = w;
            num_bits = num_words << 6;
        }
    }
    void clear_all() { std::fill(bits.begin(), bits.end(), 0); }
    bool get(size_t index) const { return (bits.at(index >> 6) & ((int64_t)1 << (index & 63))) != 0; }
    int32_t next_set_bit(size_t index) const {  // :351-376
        size_t i = index >> 6;
        int64_t word = bits.at(i) >> (index & 63);  // arithmetic shift, as in the reference
        if (word != 0) return (int32_t)(index + (size_t)ctz64(word));
        for (;;) {
            i++;
            if (i >= num_words) break;
            word = bits[i];
            if (word != 0) return (int32_t)((i << 6) + (size_t)ctz64(word));
        }
        return NO_MORE_DOCS;
    }
    uint32_t count_ones_before_index2(int32_t doc_upto, size_t bit_index, size_t end_index) const {  // :206-251
        uint32_t count = (uint32_t)doc_upto;
        if (end_index > bit_index) {
            size_t start_high = bit_index >> 6, end_high = end_index >> 6;
            if (start_high < end_high) {
                uint64_t remain = (uint64_t)bits.at(start_high) >> (bit_index & 63);
                if (remain != 0) count += (uint32_t)__builtin_popcountll(remain);
                start_high++;
                for (size_t i = start_high; i < end_high; i++)
                    if (bits.at(i) != 0) count += (uint32_t)popc64(bits[i]);
                size_t low_value = end_index & 63;
                if (low_value > 0) {
                    int64_t value = bits.at(end_high) & (int64_t)(((uint64_t)1 << low_value) - 1);
                    if (value > 0) count += (uint32_t)popc64(value);
                }
            } else {
                size_t end_remain = end_index & 63;
                if (end_remain > 0) {
                    int64_t value = bits.at(end_high) & (int64_t)(((uint64_t)1 << end_remain) - 1);
                    if (value > 0) {
                        value = value >> (bit_index & 63);
                        if (value > 0) count += (uint32_t)popc64(value);
                    }
                }
            }
        }
        return count;
    }
};

// ---------------------------------------------------------------------------
struct SegmentData;

struct BlockDocIterator {
    uint8_t encoded[MAX_ENCODED_SIZE];
    int32_t doc_delta_buffer[MAX_DATA_SIZE];
    int32_t freq_buffer[MAX_DATA_SIZE];
    int doc_buffer_upto = 0;
    std::unique_ptr<SkipReader> skipper;
    bool skipped = false;
    Input doc_in;
    bool index_has_freq = true;
    int doc_freq = 0;
    int64_t total_term_freq = 0;
    int doc_upto = 0;
    int32_t doc = -1;
    int32_t accum = 0;
    int32_t freq = 0;
    int64_t doc_term_start_fp = 0;
    int64_t skip_offset = 0;
    int32_t next_skip_doc = 0;
    bool needs_freq = true;
    int32_t singleton_doc_id = -1;
    const ForUtil* for_util = nullptr;
    bool use_simd = false;
    // other block encodings (:394-400)
    EncodeType encode_type = PF;
    EliasFanoEncoder ef_encoder;
    EliasFanoDecoder ef_decoder;
    bool has_ef_decoder = false;
    int32_t ef_base_doc = -1;
    int ef_base_total = 0;
    FixedBitSet doc_bits;
    int32_t bits_min_doc = 0;
    int32_t bits_index = 0;

    BlockDocIterator(const Input& file, const ForUtil* fu, bool simd, bool has_freq,
                     const orc_term_state& ts, bool want_freq) {  // :410-458
        doc_in = file;
        for_util = fu;
        use_simd = simd;
        index_has_freq = has_freq;
        std::memset(doc_delta_buffer, 0, sizeof(doc_delta_buffer));
        std::memset(freq_buffer, 0, sizeof(freq_buffer));
        reset(ts, want_freq);
    }
    void reset(const orc_term_state& ts, bool want_freq) {  // :460-499
        doc_freq = ts.doc_freq;
        total_term_freq = index_has_freq ? ts.total_term_freq : (int64_t)doc_freq;
        doc_term_start_fp = ts.doc_start_fp;
        skip_offset = ts.skip_offset;
        singleton_doc_id = ts.singleton_doc_id;
        if (doc_freq > 1) doc_in.seek(doc_term_start_fp);
        doc = -1;
        needs_freq = want_freq;
        if (!index_has_freq || !needs_freq)
            for (int i = 0; i < MAX_DATA_SIZE; i++) freq_buffer[i] = 1;
        accum = 0;
        doc_upto = 0;
        next_skip_doc = BLOCK_SIZE - 1;
        doc_buffer_upto = BLOCK_SIZE;
        skipped = false;
        encode_type = PF;  // :491-496
        has_ef_decoder = false;
        ef_base_doc = -1;
        doc_bits.clear_all();
        bits_index = 0;
    }
    // ForUtil::read_other_encode_block, for_util.rs:337-372
    void read_other_encode_block() {
        if (encode_type == EF) {
            int64_t upper_bound = doc_in.read_vlong();
            ef_encoder.rebuild(BLOCK_SIZE, upper_bound);
            ef_encoder.deserialize2(doc_in);
            ef_decoder.refresh(&ef_encoder);
            has_ef_decoder = true;
        } else if (encode_type == BITSET) {
            bits_min_doc = doc_in.read_vint();
            size_t num_longs = doc_in.read_byte();
            doc_bits.resize(num_longs << 6);
            EliasFanoEncoder::read_data2(doc_bits.bits, doc_in);
        }
    }
    void read_vint_block(int num) {  // :308-333
        if (index_has_freq) {
            for (int i = 0; i < num; i++) {
                uint32_t code = (uint32_t)doc_in.read_vint();
                doc_delta_buffer[i] = (int32_t)(code >> 1);
                if (code & 1) freq_buffer[i] = 1;
                else freq_buffer[i] = doc_in.read_vint();
            }
        } else {
            for (int i = 0; i < num; i++) doc_delta_buffer[i] = doc_in.read_vint();
        }
    }
    void refill_docs() {  // :501-561
        if (accum > 0) ef_base_doc = accum;  // "EF & PF compatible"
        ef_base_total = doc_upto;
        encode_type = PF;
        bits_index = 0;
        int left = doc_freq - doc_upto;
        if (left >= BLOCK_SIZE) {
            for_util->read_block(doc_in, encoded, doc_delta_buffer, &encode_type, use_simd);
            if (encode_type == FULL) throw Error("EncodeType::FULL is unimplemented in the reference too (:637-639)");
            read_other_encode_block();
            if (index_has_freq) {
                if (needs_freq) for_util->read_block(doc_in, encoded, freq_buffer, nullptr, use_simd);
                else for_util->skip_block(doc_in);
            }
        } else if (doc_freq == 1) {
            doc_delta_buffer[0] = singleton_doc_id;
            freq_buffer[0] = (int32_t)total_term_freq;
        } else {
            read_vint_block(left);
        }
        doc_buffer_upto = 0;
    }
    int32_t next() {  // :612-647
        if (doc_upto == doc_freq) return doc = NO_MORE_DOCS;
        if (doc_buffer_upto == BLOCK_SIZE) refill_docs();
        if (encode_type == PF) {
            doc = accum + doc_delta_buffer[doc_buffer_upto];
        } else if (encode_type == EF) {  // :624-626
            ef_decoder.e = &ef_encoder;  // (self-pointer: stays valid if the iterator object was moved)
            doc = (int32_t)ef_decoder.next_value() + 1 + ef_base_doc;
        } else {  // BITSET :628-633
            bits_index = doc_bits.next_set_bit((size_t)bits_index);
            doc = bits_min_doc + bits_index;
            bits_index += 1;
        }
        accum = doc;
        doc_upto++;
        freq = freq_buffer[doc_buffer_upto];
        doc_buffer_upto++;
        return doc;
    }
    int32_t advance(int32_t target) {  // :649-789
        if (target == NO_MORE_DOCS) return doc = NO_MORE_DOCS;
        if (doc_freq > BLOCK_SIZE && target > next_skip_doc) {
            if (!skipper) skipper.reset(new SkipReader(doc_in));
            if (!skipped) {
                skipper->init(doc_term_start_fp + skip_offset, doc_term_start_fp, doc_freq);
                skipped = true;
            }
            int32_t new_doc_upto = skipper->skip_to(target) + 1;
            if (new_doc_upto > doc_upto) {
                doc_upto = new_doc_upto;
                doc_buffer_upto = BLOCK_SIZE;
                accum = skipper->doc();
                doc_in.seek(skipper->doc_ptr());
            }
            next_skip_doc = skipper->next_skip_doc();
        }
        if (doc_upto == doc_freq) return doc = NO_MORE_DOCS;
        if (doc_buffer_upto == BLOCK_SIZE) refill_docs();
        if (encode_type == PF) {
            for (;;) {
                if (doc_buffer_upto >= MAX_DATA_SIZE) throw Error("index out of bounds in advance scan");
                accum += doc_delta_buffer[doc_buffer_upto];
                doc_upto++;
                if (accum >= target) break;
                doc_buffer_upto++;
                if (doc_upto == doc_freq) return doc = NO_MORE_DOCS;
            }
        } else if (encode_type == EF) {  // :733-744
            ef_decoder.e = &ef_encoder;
            int64_t v = ef_decoder.advance_to_value((int64_t)(target - 1 - ef_base_doc));
            if (v == NO_MORE_VALUES) return doc = NO_MORE_DOCS;
            doc_buffer_upto = (int)ef_decoder.current_index();
            doc_upto = ef_base_total + doc_buffer_upto + 1;
            accum = (int32_t)v + 1 + ef_base_doc;
        } else {  // BITSET :746-778
            if (target < bits_min_doc) {
                accum = bits_min_doc;
                bits_index = 1;
                doc_buffer_upto = 0;
            } else {
                int32_t index = target - bits_min_doc;
                if (index >= (int32_t)doc_bits.num_bits) return doc = NO_MORE_DOCS;
                bool find = doc_bits.get((size_t)index);
                if (find) {
                    accum = target;
                } else {
                    index = doc_bits.next_set_bit((size_t)index);
                    if (index == NO_MORE_DOCS) return doc = NO_MORE_DOCS;
                    accum = bits_min_doc + index;
                }
                doc_buffer_upto = (int)doc_bits.count_ones_before_index2(doc_buffer_upto, (size_t)bits_index, (size_t)index);
                bits_index = index + 1;
            }
            doc_upto = ef_base_total + doc_buffer_upto + 1;
        }
        doc = accum;
        freq = freq_buffer[doc_buffer_upto];
        doc_buffer_upto++;
        return doc;
    }
    size_t cost() const { return (size_t)doc_freq; }
};

// ---------------------------------------------------------------------------
// util/small_float.rs:16-36, search/similarity/bm25_similarity.rs
// ---------------------------------------------------------------------------
static uint8_t float_to_byte315(float f) {
    int32_t bits;
    std::memcpy(&bits, &f, 4);
    int32_t small = bits >> (24 - 3);
    if (small <= ((63 - 15) << 3)) return bits <= 0 ? 0 : 1;
    if (small >= ((63 - 15) << 3) + 0x100) return 255;
    return (uint8_t)(small - ((63 - 15) << 3));
}
static float byte315_to_float(uint8_t b) {
    if (b == 0) return 0.f;
    uint32_t bits = (uint32_t)b << (24 - 3);
    bits += (63 - 15) << 24;
    float f;
    std::memcpy(&f, &bits, 4);
    return f;
}
struct NormTable {  // bm25_similarity.rs:33-43
    float t[256];
    NormTable() {
        t[0] = 0.f;
        for (int i = 1; i < 256; i++) {
            float f = byte315_to_float((uint8_t)i);
            t[i] = 1.0f / (f * f);
        }
        t[0] = 1.0f / t[255];
    }
};
static const NormTable NORM_TABLE;

static float bm25_avgdl(int64_t sum_ttf, int64_t doc_count, int64_t max_doc) {  // :72-83
    if (sum_ttf <= 0) return 1.0f;
    if (doc_count == -1) doc_count = max_doc;
    return (float)((double)sum_ttf / (double)doc_count);
}
static float bm25_idf(int64_t doc_freq, int64_t doc_count) {  // :99-114 (single term)
    float idf = 0.0f;
    idf += (float)std::log(1.0 + ((double)doc_count - (double)doc_freq + 0.5) / ((double)doc_freq + 0.5));
    return idf;
}
static void bm25_cache(float k1, float b, float avgdl, float* cache) {  // :161-165
    for (int i = 0; i < 256; i++) cache[i] = k1 * ((1.0f - b) + b * (NORM_TABLE.t[i] / avgdl));
}
static inline float bm25_score(float weight, float k1, float freq, float norm) {  // :203-212
    return weight * (k1 + 1.0f) * freq / (freq + norm);
}

struct SimWeight {  // BM25SimWeight :238-263,363-366
    float k1, b, idf, avgdl, boost, weight;
    float cache[256];
};

// ---------------------------------------------------------------------------
// Index model: what LeafReader exposes to the hot path
// (index/reader/leaf_reader.rs:62-182: postings(), norm_values(), live_docs())
// ---------------------------------------------------------------------------
struct SegmentData {
    const uint8_t* file = nullptr;
    int64_t file_len = 0;
    int version = 0;
    bool use_simd = false;
    ForUtil for_util;
    int32_t max_doc = 0;
    int32_t doc_base = 0;
    const uint8_t* norms = nullptr;
    const uint64_t* live_docs = nullptr;
    std::vector<orc_term_state> terms;
    int64_t doc_count = 0, sum_ttf = 0, sum_df = 0;
    bool live(int32_t doc) const {
        return !live_docs || ((live_docs[doc >> 6] >> (doc & 63)) & 1);
    }
};

// codec/codec_util.rs:46-57,75-124 — check_index_header for "Lucene50PostingsWriterDoc"
static void open_doc_file(SegmentData& seg) {
    Input in(seg.file, seg.file_len);
    if (in.read_int() != 0x3FD76C17) throw Error("codec header mismatch");
    int slen = in.read_vint();
    static const char* codec = "Lucene50PostingsWriterDoc";
    if (slen != (int)std::strlen(codec) || std::memcmp(in.get_and_advance((size_t)slen), codec, (size_t)slen) != 0)
        throw Error("codec name mismatch");
    int version = in.read_int();
    if (version < 0 || version > 1) throw Error("unsupported .doc version");  // posting_reader.rs:57-58
    in.get_and_advance(16);  // segment id
    int suffix = in.read_byte();
    in.get_and_advance((size_t)suffix);
    seg.version = version;
    seg.use_simd = version > 0;  // posting_reader.rs:103-107 (SSE3 always present on x86-64 hosts here)
    seg.for_util.with_input(in);
}

// search/scorer/term_scorer.rs:21-67
struct TermScorer : Scorer {
    BlockDocIterator it;
    const SimWeight* w;
    const uint8_t* norms;
    TermScorer(const SegmentData& seg, const orc_term_state& ts, const SimWeight* sw)
        : it(Input(seg.file, seg.file_len), &seg.for_util, seg.use_simd, true, ts, true),
          w(sw), norms(seg.norms) {}
    int32_t doc_id() const override { return it.doc; }
    int32_t next() override { return it.next(); }
    int32_t advance(int32_t t) override { return it.advance(t); }
    size_t cost() const override { return it.cost(); }
    float score() override {
        float norm = norms ? w->cache[norms[it.doc] & 0xFF] : w->k1;
        return bm25_score(w->weight, w->k1, (float)it.freq, norm);
    }
};

// A FILTER clause: BooleanQuery::create_weight builds its weight with needs_scores = false
// (query/boolean_query.rs:108-110), so TermQuery::create_weight picks NonScoringSimilarity
// (searcher.rs:724-730) whose scorer returns 0f32 (:192-197) and the postings are opened with
// PostingIteratorFlags::NONE (term_query.rs:145-150): same docids, the freq blocks are skipped.
struct FilterTermScorer : Scorer {
    BlockDocIterator it;
    FilterTermScorer(const SegmentData& seg, const orc_term_state& ts)
        : it(Input(seg.file, seg.file_len), &seg.for_util, seg.use_simd, true, ts, false) {}
    int32_t doc_id() const override { return it.doc; }
    int32_t next() override { return it.next(); }
    int32_t advance(int32_t t) override { return it.advance(t); }
    size_t cost() const override { return it.cost(); }
    float score() override { return 0.0f; }
};

// MatchAllDocsQuery (query/match_all_query.rs:28-116): ConstantScoreScorer { score: weight = 0f32 (the
// default; normalisation is commented out, searcher.rs:709-722), iterator: AllDocsIterator (:118-158) }
struct AllDocsScorer : Scorer {
    int32_t doc = -1, max_doc;
    explicit AllDocsScorer(int32_t md) : max_doc(md) {}
    int32_t doc_id() const override { return doc; }
    int32_t next() override { return advance(doc + 1); }
    int32_t advance(int32_t target) override { return doc = target >= max_doc ? NO_MORE_DOCS : target; }
    size_t cost() const override { return (size_t)std::max(1, max_doc); }
    float score() override { return 0.0f; }
};

// search/mod.rs:209-367 — MockDocIterator / MockSimpleScorer (score = doc id)
struct MockScorer : Scorer {
    std::vector<int32_t> docs;
    size_t idx = 0;
    int32_t cur = -1;
    explicit MockScorer(std::vector<int32_t> d) : docs(std::move(d)) {}
    int32_t doc_id() const override { return cur; }
    int32_t next() override {
        if (idx >= docs.size()) return cur = NO_MORE_DOCS;
        return cur = docs[idx++];
    }
    int32_t advance(int32_t target) override {
        int32_t d;
        do d = next();
        while (d < target);
        return d;
    }
    size_t cost() const override { return docs.size(); }
    float score() override { return (float)cur; }
};

// search/scorer/conjunction_scorer.rs:20-128
struct ConjunctionScorer : Scorer {
    ScorerPtr lead1, lead2;
    std::vector<ScorerPtr> others;
    explicit ConjunctionScorer(std::vector<ScorerPtr> children) {
        std::stable_sort(children.begin(), children.end(),
                         [](const ScorerPtr& a, const ScorerPtr& b) { return a->cost() < b->cost(); });
        lead1 = std::move(children[0]);
        lead2 = std::move(children[1]);
        for (size_t i = 2; i < children.size(); i++) others.push_back(std::move(children[i]));
    }
    int32_t skip_to_approx(int32_t target) {  // :44-83
        int32_t doc = target;
        for (;;) {
        advance_head:
            int32_t next2 = lead2->advance(doc);
            if (next2 != doc) {
                doc = lead1->advance(next2);
                if (next2 != doc) continue;
            }
            if (doc == NO_MORE_DOCS) return doc;
            for (auto& other : others) {
                if (other->doc_id() < doc) {
                    int32_t next = other->advance(doc);
                    if (next > doc) {
                        doc = lead1->advance(next);
                        goto advance_head;
                    }
                }
            }
            return doc;
        }
    }
    int32_t doc_id() const override { return lead1->doc_id(); }
    int32_t next() override { return skip_to_approx(lead1->next()); }
    int32_t advance(int32_t t) override { return skip_to_approx(lead1->advance(t)); }
    size_t cost() const override { return lead1->cost(); }
    float score() override {  // :87-95
        float s = lead1->score();
        s += lead2->score();
        for (auto& o : others) s += o->score();
        return s;
    }
};

// search/scorer/disjunction_scorer.rs:24-104,187-376 — SimpleQueue variant (<10 children)
// util/disi.rs:135-336 — DisiPriorityQueue: a binary min-heap of the sub-scorers on their current docid
// (push = up_heap, PeekMut drop = update_top = down_heap from the root) and top_list(): the sub-scorers that sit
// on the top docid, collected by walking the heap from the root and PREPENDING each hit, so score_sum /
// score_max (search/scorer/disjunction_scorer.rs:226-240,264-286) add the scores in the reverse of that walk.
// The heap layout depends on the whole history of next() calls, and with it the f32 summation order.
struct DisiQueue {
    struct W {
        Scorer* s;
        W* next;
    };
    std::vector<W> buffer;
    std::vector<W*> heap;
    size_t size = 0;
    explicit DisiQueue(std::vector<ScorerPtr>& children) {  // :163-181
        buffer.reserve(children.size());
        for (auto& c : children) buffer.push_back(W{c.get(), nullptr});
        heap.assign(children.size(), nullptr);
        for (W& w : buffer) {  // do_push :239-245
            heap[size] = &w;
            up_heap(size);
            size++;
        }
    }
    W* top() const { return heap[0]; }
    void up_heap(size_t i) {  // :296-309
        W* node = heap[i];
        const int32_t node_doc = node->s->doc_id();
        while (i > 0) {
            const size_t j = ((i + 1) >> 1) - 1;
            if (node_doc >= heap[j]->s->doc_id()) break;
            heap[i] = heap[j];
            i = j;
        }
        heap[i] = node;
    }
    void update_top() {  // down_heap(size) :311-336
        size_t i = 0;
        W* node = heap[0];
        size_t j = ((i + 1) << 1) - 1;
        if (j < size) {
            size_t k = j + 1;
            if (k < size && heap[k]->s->doc_id() < heap[j]->s->doc_id()) j = k;
            if (heap[j]->s->doc_id() < node->s->doc_id()) {
                for (;;) {
                    heap[i] = heap[j];
                    i = j;
                    j = ((i + 1) << 1) - 1;
                    k = j + 1;
                    if (k < size && heap[k]->s->doc_id() < heap[j]->s->doc_id()) j = k;
                    if (j >= size || heap[j]->s->doc_id() >= node->s->doc_id()) break;
                }
                heap[i] = node;
            }
        }
    }
    W* top_list_to(W* list, size_t i) {  // :213-231
        W* w = heap[i];
        if (w->s->doc_id() == list->s->doc_id()) {
            w->next = list;
            list = w;
            const size_t left = ((i + 1) << 1) - 1, right = left + 1;
            if (right < size) {
                list = top_list_to(list, left);
                list = top_list_to(list, right);
            } else if (left < size && heap[left]->s->doc_id() == list->s->doc_id()) {
                heap[left]->next = list;
                list = heap[left];
            }
        }
        return list;
    }
    W* top_list() {  // :190-206
        W* list = heap[0];
        list->next = nullptr;
        if (size >= 3) {
            list = top_list_to(list, 1);
            list = top_list_to(list, 2);
        } else if (size == 2 && heap[1]->s->doc_id() == list->s->doc_id()) {
            heap[1]->next = list;
            list = heap[1];
        }
        return list;
    }
    int32_t next_doc() {  // SubScorers::approximate_next, DPQ arm (disjunction_scorer.rs:334-347)
        const int32_t doc = top()->s->doc_id();
        for (;;) {
            top()->s->next();
            update_top();
            if (top()->s->doc_id() != doc) break;
        }
        return top()->s->doc_id();
    }
    int32_t advance(int32_t target) {  // :364-374
        for (;;) {
            top()->s->advance(target);
            update_top();
            if (top()->s->doc_id() >= target) break;
        }
        return top()->s->doc_id();
    }
};

struct DisjunctionSumScorer : Scorer {
    std::vector<ScorerPtr> scorers;
    int32_t curr_doc;
    bool needs_scores;
    int32_t min_should_match;
    size_t cost_;
    std::unique_ptr<DisiQueue> dpq;  // >= 10 children and min_should_match <= 1 (:41-45)
    DisjunctionSumScorer(std::vector<ScorerPtr> children, bool needs, int32_t msm)
        : scorers(std::move(children)), needs_scores(needs), min_should_match(msm) {
        if (!(scorers.size() < 10 || msm > 1)) dpq.reset(new DisiQueue(scorers));
        cost_ = 0;
        curr_doc = NO_MORE_DOCS;
        for (auto& s : scorers) {
            cost_ += s->cost();
            curr_doc = std::min(curr_doc, s->doc_id());
        }
    }
    int32_t doc_id() const override { return dpq ? dpq->top()->s->doc_id() : curr_doc; }
    int32_t next() override {  // :295-333
        if (dpq) return dpq->next_doc();
        int32_t msm = min_should_match > 1 ? min_should_match : 1;
        for (;;) {
            if (curr_doc == NO_MORE_DOCS) return curr_doc;
            int32_t cd = curr_doc;
            int32_t min_doc = NO_MORE_DOCS;
            for (auto& s : scorers) {
                if (s->doc_id() == cd) s->next();
                min_doc = std::min(min_doc, s->doc_id());
            }
            curr_doc = min_doc;
            if (msm > 1) {
                int count = 0;
                for (auto& s : scorers)
                    if (s->doc_id() == min_doc) count++;
                if (count < msm) continue;
            }
            return curr_doc;
        }
    }
    int32_t advance(int32_t target) override {  // :350-363
        if (dpq) return dpq->advance(target);
        int32_t min_doc = NO_MORE_DOCS;
        for (auto& s : scorers) {
            if (s->doc_id() < target) s->advance(target);
            min_doc = std::min(min_doc, s->doc_id());
        }
        return curr_doc = min_doc;
    }
    size_t cost() const override { return cost_; }
    float score() override {  // :57-64,211-240
        if (!needs_scores) return 0.0f;
        float score = 0.0f;
        if (dpq) {
            for (DisiQueue::W* w = dpq->top_list(); w; w = w->next) score += w->s->score();
            return score;
        }
        for (auto& s : scorers)
            if (s->doc_id() == curr_doc) score += s->score();
        return score;
    }
};

// search/scorer/disjunction_scorer.rs:106-186,241-263 — DisjunctionMaxScorer, SimpleQueue variant
// (<10 children): the union like DisjunctionSumScorer without min_should_match; score =
// max + (sum - max) * tie_breaker_multiplier, sum in child order from 0.0f, max from -inf.
struct DisjunctionMaxScorer : Scorer {
    std::vector<ScorerPtr> scorers;
    int32_t curr_doc;
    float tie_breaker_multiplier;
    size_t cost_;
    std::unique_ptr<DisiQueue> dpq;  // >= 10 disjuncts (:118-139)
    DisjunctionMaxScorer(std::vector<ScorerPtr> children, float tie) : scorers(std::move(children)), tie_breaker_multiplier(tie) {
        if (scorers.size() >= 10) dpq.reset(new DisiQueue(scorers));
        cost_ = 0;
        curr_doc = NO_MORE_DOCS;
        for (auto& s : scorers) {
            cost_ += s->cost();
            curr_doc = std::min(curr_doc, s->doc_id());
        }
    }
    int32_t doc_id() const override { return dpq ? dpq->top()->s->doc_id() : curr_doc; }
    int32_t next() override {  // approximate_next(None) :295-333 with DEFAULT_MIN_SHOULD_MATCH
        if (dpq) return dpq->next_doc();
        if (curr_doc == NO_MORE_DOCS) return curr_doc;
        int32_t cd = curr_doc, min_doc = NO_MORE_DOCS;
        for (auto& s : scorers) {
            if (s->doc_id() == cd) s->next();
            min_doc = std::min(min_doc, s->doc_id());
        }
        return curr_doc = min_doc;
    }
    int32_t advance(int32_t target) override {  // :350-374
        if (dpq) return dpq->advance(target);
        int32_t min_doc = NO_MORE_DOCS;
        for (auto& s : scorers) {
            if (s->doc_id() < target) s->advance(target);
            min_doc = std::min(min_doc, s->doc_id());
        }
        return curr_doc = min_doc;
    }
    size_t cost() const override { return cost_; }
    float score() override {  // score_max :241-286
        if (dpq) {
            float score_sum = 0.0f, score_max = -INFINITY;
            for (DisiQueue::W* w = dpq->top_list(); w; w = w->next) {
                const float sub = w->s->score();
                score_sum += sub;
                if (sub > score_max) score_max = sub;
            }
            return score_max + (score_sum - score_max) * tie_breaker_multiplier;
        }
        float score_sum = 0.0f, score_max = -INFINITY;
        for (auto& s : scorers)
            if (s->doc_id() == curr_doc) {
                float sub = s->score();
                score_sum += sub;
                score_max = std::fmax(score_max, sub);
            }
        return score_max + (score_sum - score_max) * tie_breaker_multiplier;
    }
};

// search/scorer/req_opt_scorer.rs:19-105
struct ReqOptScorer : Scorer {
    ScorerPtr req, opt;
    float scores_sum = 0.f;
    size_t scores_num = 0;
    ReqOptScorer(ScorerPtr r, ScorerPtr o) : req(std::move(r)), opt(std::move(o)) {}
    int32_t doc_id() const override { return req->doc_id(); }
    int32_t next() override { return req->next(); }
    int32_t advance(int32_t t) override { return req->advance(t); }
    size_t cost() const override { return req->cost(); }
    float score() override {
        int32_t current = req->doc_id();
        float score = req->score();
        if (scores_num > 100) {
            if (2.0f * score < scores_sum / (float)scores_num) return score;
        }
        scores_sum += score;
        scores_num += 1;
        int32_t opt_doc = opt->doc_id();
        if (opt_doc < current) opt_doc = opt->advance(current);
        if (opt_doc == current) score += opt->score();
        return score;
    }
};

// search/scorer/req_not_scorer.rs:21-119
struct ReqNotScorer : Scorer {
    ScorerPtr req, nots;
    ReqNotScorer(ScorerPtr r, ScorerPtr n) : req(std::move(r)), nots(std::move(n)) {}
    int32_t doc_id() const override { return req->doc_id(); }
    int32_t next() override {
        for (;;) {
            int32_t doc = req->next();
            if (doc == NO_MORE_DOCS) break;
            if (doc == nots->doc_id()) continue;
            if (doc < nots->doc_id()) return doc;
            int32_t not_doc = nots->advance(doc);
            if (doc < not_doc) return doc;
        }
        return NO_MORE_DOCS;
    }
    int32_t advance(int32_t target) override {
        int32_t doc = req->advance(target);
        if (doc < NO_MORE_DOCS) {
            for (;;) {
                if (doc == nots->doc_id()) return next();
                if (doc < nots->doc_id()) return doc;
                nots->advance(doc);
            }
        }
        return NO_MORE_DOCS;
    }
    size_t cost() const override { return req->cost(); }
    float score() override { return req->score(); }
};

// ---------------------------------------------------------------------------
// search/collector/top_docs.rs:28-95 + std BinaryHeap (util/external/binary_heap.rs:121-210)
// with ScoreDoc's reversed PartialOrd (sort_field/collapse_top_docs.rs:48-60)
// ---------------------------------------------------------------------------
struct TopDocsHeap {
    std::vector<orc_hit> data;
    size_t k;
    uint64_t total_hits = 0;
    explicit TopDocsHeap(size_t kk) : k(kk) { data.reserve(kk); }
    // a <= b under reversed PartialOrd  <=>  a.score >= b.score
    static bool le(const orc_hit& a, const orc_hit& b) { return a.score >= b.score; }
    static bool ge(const orc_hit& a, const orc_hit& b) { return a.score <= b.score; }
    size_t sift_up(size_t start, size_t pos) {
        orc_hit e = data[pos];
        while (pos > start) {
            size_t parent = (pos - 1) / 2;
            if (le(e, data[parent])) break;
            data[pos] = data[parent];
            pos = parent;
        }
        data[pos] = e;
        return pos;
    }
    void sift_down_range(size_t pos, size_t end) {
        orc_hit e = data[pos];
        size_t child = 2 * pos + 1;
        while (child < end) {
            size_t right = child + 1;
            if (right < end && le(data[child], data[right])) child = right;
            if (ge(e, data[child])) break;
            data[pos] = data[child];
            pos = child;
            child = 2 * pos + 1;
        }
        data[pos] = e;
    }
    void sift_down_to_bottom(size_t pos) {
        size_t end = data.size();
        size_t start = pos;
        orc_hit e = data[pos];
        size_t child = 2 * pos + 1;
        while (child < end) {
            size_t right = child + 1;
            if (right < end && le(data[child], data[right])) child = right;
            data[pos] = data[child];
            pos = child;
            child = 2 * pos + 1;
        }
        data[pos] = e;
        sift_up(start, pos);
    }
    void push(orc_hit h) {
        data.push_back(h);
        sift_up(0, data.size() - 1);
    }
    orc_hit pop() {
        orc_hit item = data.back();
        data.pop_back();
        if (!data.empty()) {
            std::swap(item, data[0]);
            sift_down_to_bottom(0);
        }
        return item;
    }
    void add_doc(int32_t doc, float score) {  // top_docs.rs:67-76
        if (data.size() < k) {
            push(orc_hit{doc, score});
        } else if (!data.empty()) {
            if (data[0].score < score) {
                data[0] = orc_hit{doc, score};
                sift_down_range(0, data.size());  // PeekMut drop
            }
        }
    }
    void collect(int32_t global_doc, float score) {  // :84-95
        add_doc(global_doc, score);
        total_hits++;
    }
    std::vector<orc_hit> top_docs() {  // :55-65
        size_t size = (size_t)std::min<uint64_t>(total_hits, data.size());
        std::vector<orc_hit> out;
        out.reserve(size);
        for (size_t i = 0; i < size; i++) out.push_back(pop());
        std::reverse(out.begin(), out.end());
        return out;
    }
};

// search/scorer/bulk_scorer.rs:57-72,89-122 — non-two-phase branch with accept_docs
template <class Collect>
static void bulk_score(Scorer& scorer, const SegmentData* seg, Collect&& collect) {
    int32_t doc = scorer.next();
    while (doc < NO_MORE_DOCS) {
        if (!seg || seg->live(doc)) collect(doc, scorer);
        doc = scorer.next();
    }
}

}  // namespace orc

// ---------------------------------------------------------------------------
// Index + searcher (search/searcher.rs:306-363,487-525,732-771;
// query/term_query.rs:58-95,145-163; query/boolean_query.rs:40-87,196-279)
// ---------------------------------------------------------------------------
struct orc_index {
    float k1, b;
    std::vector<orc::SegmentData> segs;
    int stats_seg = -1;  // largest max_doc, first on ties (stable sort desc, searcher.rs:311-312)
    int64_t total_max_doc = 0;
};

namespace orc {

static void make_weight(const orc_index& ix, uint32_t term_id, float boost, SimWeight& w) {
    // searcher.rs:732-767 term_statistics: doc_freq from the stats segment only;
    // :311-351 collection statistics of that segment with max_doc = reader.max_doc().
    const SegmentData& ss = ix.segs[(size_t)ix.stats_seg];
    int64_t df = term_id < ss.terms.size() ? ss.terms[term_id].doc_freq : 0;
    int64_t doc_count = ss.doc_count == -1 ? ix.total_max_doc : ss.doc_count;
    w.k1 = ix.k1;
    w.b = ix.b;
    w.avgdl = bm25_avgdl(ss.sum_ttf, ss.doc_count, ix.total_max_doc);
    w.idf = bm25_idf(df, doc_count);
    bm25_cache(ix.k1, ix.b, w.avgdl, w.cache);
    w.boost = boost;
    w.weight = w.idf * boost;  // do_normalize :363-366
}

struct Plan {
    std::vector<SimWeight> weights;  // one per clause
};

// BooleanWeight::create_scorer (boolean_query.rs:196-279) / TermWeight::create_scorer
static ScorerPtr create_scorer(const orc_index& ix, const SegmentData& seg, const orc_query& q,
                               const orc_clause* clauses, const Plan& plan) {
    auto term_scorer = [&](uint32_t ci) -> ScorerPtr {
        const orc_clause& c = clauses[q.clause_begin + ci];
        if (c.term_id >= seg.terms.size() || seg.terms[c.term_id].doc_freq <= 0) return nullptr;
        if (c.occur == ORC_FILTER) return ScorerPtr(new FilterTermScorer(seg, seg.terms[c.term_id]));
        return ScorerPtr(new TermScorer(seg, seg.terms[c.term_id], &plan.weights[ci]));
    };
    if (!q.is_boolean) return term_scorer(0);
    if (q.is_boolean == 2) {
        // DisjunctionMaxQuery::build (search/query/disjunction_max_query.rs:51-68): one disjunct is the
        // disjunct itself; DisjunctionMaxWeight::create_scorer (:135-155): 0 scorers -> None, 1 -> it
        if (q.n_clauses == 0) throw Error("DisjunctionMaxQuery: sub query should not be empty!");
        if (q.n_clauses == 1) return term_scorer(0);
        float tie;
        std::memcpy(&tie, &q.min_should_match, 4);
        std::vector<ScorerPtr> v;
        for (uint32_t i = 0; i < q.n_clauses; i++) {
            ScorerPtr sc = term_scorer(i);
            if (sc) v.push_back(std::move(sc));
        }
        if (v.empty()) return nullptr;
        if (v.size() == 1) return std::move(v[0]);
        return ScorerPtr(new DisjunctionMaxScorer(std::move(v), tie));
    }

    // BooleanQuery::build (:40-87)
    int32_t msm = q.min_should_match;
    std::vector<uint32_t> musts, shoulds, filters, must_nots;
    for (uint32_t i = 0; i < q.n_clauses; i++) {
        int occ = clauses[q.clause_begin + i].occur;
        (occ == ORC_MUST ? musts : occ == ORC_SHOULD ? shoulds : occ == ORC_FILTER ? filters : must_nots).push_back(i);
    }
    if (msm <= 0) msm = musts.empty() ? 1 : 0;
    if (musts.size() + shoulds.size() + filters.size() + must_nots.size() == 0)
        throw Error("boolean query should at least contain one inner query!");
    // one positive clause and nothing else: the clause itself — a lone filter becomes
    // ConstantScoreQuery::with_boost(filter, 0f32) (:66-75), i.e. its docs with score 0
    if (must_nots.empty() && musts.size() + shoulds.size() + filters.size() == 1)
        return term_scorer(musts.size() == 1 ? musts[0] : shoulds.size() == 1 ? shoulds[0] : filters[0]);
    const bool match_all = musts.size() + shoulds.size() + filters.size() == 0;  // :76-79 musts.push(MatchAllDocsQuery)
    // create_weight (:96-125): must_weights = musts, then filters (needs_scores = false)
    musts.insert(musts.end(), filters.begin(), filters.end());

    ScorerPtr must_scorer, should_scorer, must_not_scorer;
    if (match_all) must_scorer.reset(new AllDocsScorer(seg.max_doc));
    if (!musts.empty()) {
        std::vector<ScorerPtr> v;
        for (uint32_t ci : musts) {
            ScorerPtr s = term_scorer(ci);
            if (!s) return nullptr;
            v.push_back(std::move(s));
        }
        if (v.size() > 1) must_scorer.reset(new ConjunctionScorer(std::move(v)));
        else must_scorer = std::move(v[0]);
    }
    {
        std::vector<ScorerPtr> v;
        for (uint32_t ci : shoulds) {
            ScorerPtr s = term_scorer(ci);
            if (s) v.push_back(std::move(s));
        }
        if (!v.empty()) should_scorer.reset(new DisjunctionSumScorer(std::move(v), true, msm));
    }
    {
        std::vector<ScorerPtr> v;
        for (uint32_t ci : must_nots) {
            ScorerPtr s = term_scorer(ci);
            if (s) v.push_back(std::move(s));
        }
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

static void search_one(const orc_index& ix, const orc_query& q, const orc_clause* clauses,
                       uint32_t k, int parallel_mode, orc_hit* out, uint32_t* out_count,
                       uint64_t* out_total) {
    Plan plan;
    plan.weights.resize(q.n_clauses);
    for (uint32_t i = 0; i < q.n_clauses; i++)
        make_weight(ix, clauses[q.clause_begin + i].term_id, clauses[q.clause_begin + i].boost,
                    plan.weights[i]);
    TopDocsHeap main(k);
    for (const SegmentData& seg : ix.segs) {  // searcher.rs:493
        ScorerPtr scorer = create_scorer(ix, seg, q, clauses, plan);
        if (!scorer) continue;
        if (parallel_mode == 0) {
            bulk_score(*scorer, &seg, [&](int32_t doc, Scorer& s) { main.collect(doc + seg.doc_base, s.score()); });
        } else {  // searcher.rs:527-630 + top_docs.rs:145-213, leaves merged in leaf order
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

template <class F>
static void parallel_for(uint32_t n, int n_threads, F&& f) {
    if (n_threads <= 1 || n <= 1) {
        for (uint32_t i = 0; i < n; i++) f(i);
        return;
    }
    std::atomic<uint32_t> next{0};
    std::atomic<bool> failed{false};
    std::string err;
    std::vector<std::thread> ts;
    int nt = (int)std::min<uint32_t>((uint32_t)n_threads, n);
    for (int t = 0; t < nt; t++)
        ts.emplace_back([&] {
            try {
                for (;;) {
                    uint32_t i = next.fetch_add(1);
                    if (i >= n || failed.load()) break;
                    f(i);
                }
            } catch (const std::exception& e) {
                if (!failed.exchange(true)) err = e.what();
            }
        });
    for (auto& t : ts) t.join();
    if (failed.load()) throw Error(err);
}

}  // namespace orc

using namespace orc;

#define ORC_TRY try {
#define ORC_CATCH(ret)                 \
    }                                  \
    catch (const std::exception& e) {  \
        g_err = e.what();              \
        return ret;                    \
    }

extern "C" {

const char* orc_last_error(void) { return g_err.c_str(); }

orc_index* orc_index_create(float k1, float b) {
    orc_index* ix = new orc_index();
    ix->k1 = k1;
    ix->b = b;
    return ix;
}
void orc_index_destroy(orc_index* ix) { delete ix; }

int orc_index_add_segment(orc_index* ix, const uint8_t* doc_file, size_t doc_len, int32_t max_doc,
                          const uint8_t* norms, const uint64_t* live_docs,
                          const orc_term_state* terms, uint32_t n_terms, int64_t field_doc_count,
                          int64_t sum_total_term_freq, int64_t sum_doc_freq) {
    ORC_TRY
    SegmentData seg;
    seg.file = doc_file;
    seg.file_len = (int64_t)doc_len;
    open_doc_file(seg);
    seg.max_doc = max_doc;
    seg.doc_base = (int32_t)ix->total_max_doc;
    seg.norms = norms;
    seg.live_docs = live_docs;
    seg.terms.assign(terms, terms + n_terms);
    seg.doc_count = field_doc_count;
    seg.sum_ttf = sum_total_term_freq;
    seg.sum_df = sum_doc_freq;
    ix->segs.push_back(std::move(seg));
    ix->total_max_doc += max_doc;
    ix->stats_seg = 0;
    for (size_t i = 1; i < ix->segs.size(); i++)
        if (ix->segs[i].max_doc > ix->segs[(size_t)ix->stats_seg].max_doc) ix->stats_seg = (int)i;
    return 0;
    ORC_CATCH(-1)
}

int orc_search_batch(orc_index* ix, const orc_query* queries, uint32_t n_queries,
                     const orc_clause* clauses, uint32_t k, int parallel_mode, int n_threads,
                     orc_hit* out_hits, uint32_t* out_counts, uint64_t* out_total) {
    ORC_TRY
    if (ix->segs.empty()) throw Error("index has no segments");
    parallel_for(n_queries, n_threads, [&](uint32_t i) {
        search_one(*ix, queries[i], clauses, k, parallel_mode, out_hits + (size_t)i * k,
                   out_counts + i, out_total + i);
    });
    return 0;
    ORC_CATCH(-1)
}

// Per-leaf TopDocsLeafCollector result of ONE segment in the engine's leaf-record layout
// {u32 n; u32 pad; u64 total_hits; orc_hit heap[k]} (heap-array order == into_vec(),
// top_docs.rs:203-213).  Weights come from the index-wide statistics segment as usual.
int orc_search_leaf_records(orc_index* ix, uint32_t seg_i, const orc_query* queries, uint32_t n_queries,
                            const orc_clause* clauses, uint32_t k, int n_threads, uint8_t* out_records) {
    ORC_TRY
    const SegmentData& seg = ix->segs.at(seg_i);
    const size_t rb = 16 + (size_t)k * sizeof(orc_hit);
    std::memset(out_records, 0, rb * n_queries);
    parallel_for(n_queries, n_threads, [&](uint32_t qi) {
        const orc_query& q = queries[qi];
        Plan plan;
        plan.weights.resize(q.n_clauses);
        for (uint32_t i = 0; i < q.n_clauses; i++)
            make_weight(*ix, clauses[q.clause_begin + i].term_id, clauses[q.clause_begin + i].boost, plan.weights[i]);
        TopDocsHeap leaf(k);
        ScorerPtr scorer = create_scorer(*ix, seg, q, clauses, plan);
        if (scorer)
            bulk_score(*scorer, &seg, [&](int32_t doc, Scorer& s) { leaf.collect(doc + seg.doc_base, s.score()); });
        uint8_t* rec = out_records + rb * qi;
        uint32_t n = (uint32_t)leaf.data.size();
        uint64_t total = leaf.total_hits;
        std::memcpy(rec, &n, 4);
        std::memcpy(rec + 8, &total, 8);
        if (n) std::memcpy(rec + 16, leaf.data.data(), n * sizeof(orc_hit));
    });
    return 0;
    ORC_CATCH(-1)
}

int orc_term_weight(orc_index* ix, uint32_t term_id, float boost, float* out_weight,
                    float* out_idf, float* out_avgdl, float out_cache[256]) {
    ORC_TRY
    SimWeight w;
    make_weight(*ix, term_id, boost, w);
    *out_weight = w.weight;
    *out_idf = w.idf;
    *out_avgdl = w.avgdl;
    std::memcpy(out_cache, w.cache, sizeof(w.cache));
    return 0;
    ORC_CATCH(-1)
}

int64_t orc_postings(orc_index* ix, uint32_t seg_i, uint32_t term_id, int32_t* docs,
                     int32_t* freqs, int64_t cap) {
    ORC_TRY
    const SegmentData& seg = ix->segs.at(seg_i);
    if (term_id >= seg.terms.size() || seg.terms[term_id].doc_freq <= 0) return 0;
    BlockDocIterator it(Input(seg.file, seg.file_len), &seg.for_util, seg.use_simd, true,
                        seg.terms[term_id], true);
    int64_t n = 0;
    while (n < cap) {
        int32_t d = it.next();
        if (d == NO_MORE_DOCS) break;
        docs[n] = d;
        freqs[n] = it.freq;
        n++;
    }
    return n;
    ORC_CATCH(-1)
}

int orc_advance_seq(orc_index* ix, uint32_t seg_i, uint32_t term_id, const int32_t* targets,
                    uint32_t n, int32_t* out_docs, int32_t* out_freqs) {
    ORC_TRY
    const SegmentData& seg = ix->segs.at(seg_i);
    if (term_id >= seg.terms.size() || seg.terms[term_id].doc_freq <= 0) throw Error("term absent");
    BlockDocIterator it(Input(seg.file, seg.file_len), &seg.for_util, seg.use_simd, true,
                        seg.terms[term_id], true);
    for (uint32_t i = 0; i < n; i++) {
        out_docs[i] = targets[i] < 0 ? it.next() : it.advance(targets[i]);  // target -1: next()
        out_freqs[i] = out_docs[i] == NO_MORE_DOCS ? 0 : it.freq;
    }
    return 0;
    ORC_CATCH(-1)
}

int orc_forutil_decode(const uint8_t* stream, size_t len, const uint64_t* offsets,
                       uint32_t n_blocks, int doc_version, const int32_t forutil_table[32],
                       int32_t* out, int n_threads) {
    ORC_TRY
    ForUtil fu;
    fu.init_from_codes(forutil_table);
    bool by_simd = doc_version > 0;
    const uint32_t chunk = 4096;
    uint32_t n_chunks = (n_blocks + chunk - 1) / chunk;
    parallel_for(n_chunks, n_threads, [&](uint32_t c) {
        uint8_t encoded[MAX_ENCODED_SIZE + 64];
        int32_t decoded[MAX_DATA_SIZE];
        uint32_t end = std::min(n_blocks, (c + 1) * chunk);
        for (uint32_t i = c * chunk; i < end; i++) {
            Input in(stream, (int64_t)len, (int64_t)offsets[i]);
            fu.read_block(in, encoded, decoded, nullptr, by_simd);
            std::memcpy(out + (size_t)i * 128, decoded, 512);
        }
    });
    return 0;
    ORC_CATCH(-1)
}

void orc_simd_pack(const uint32_t* d, uint8_t* e, int bits) { simd_pack<false>(d, e, bits, nullptr); }
void orc_simd_unpack(const uint8_t* e, uint32_t* d, int bits) { simd_unpack<false>(e, d, bits, nullptr); }
void orc_simd_delta_pack(const uint32_t* d, uint8_t* e, uint32_t base, int bits) {
    DeltaState st{base};
    simd_pack<true>(d, e, bits, &st);
}
void orc_simd_delta_unpack(const uint8_t* e, uint32_t* d, uint32_t base, int bits) {
    DeltaState st{base};
    simd_unpack<true>(e, d, bits, &st);
}
int orc_simd_max_bits(const uint32_t* d) { return simd_max_bits(d); }

int orc_packed_decode(int format_id, int bpv, const uint8_t* blocks, size_t n_bytes,
                      int32_t* values, int iterations) {
    ORC_TRY
    BulkOp op = BulkOp::make(format_id, bpv);
    if ((size_t)iterations * (size_t)op.bytes_per_iteration() > n_bytes) throw Error("short input");
    return op.decode(blocks, values, iterations);
    ORC_CATCH(-1)
}
int orc_packed_encode(int format_id, int bpv, const int32_t* values, uint8_t* blocks,
                      int iterations) {
    ORC_TRY
    BulkOp op = BulkOp::make(format_id, bpv);
    return op.encode(values, blocks, iterations);
    ORC_CATCH(-1)
}
int orc_packed_iterations(int format_id, int bpv) {
    ORC_TRY
    return compute_iterations(BulkOp::make(format_id, bpv));
    ORC_CATCH(-1)
}
int orc_packed_encoded_size(int format_id, int bpv) {
    return (int)format_byte_count(format_id, BLOCK_SIZE, bpv);
}
int orc_max_data_size(void) {
    ORC_TRY
    return max_data_size();
    ORC_CATCH(-1)
}
int orc_fastest_format(int bpv, float overhead, int* out_bpv) {
    int f, b;
    fastest_format(BLOCK_SIZE, bpv, overhead, &f, &b);
    *out_bpv = b;
    return f;
}
int orc_block_advance(const int32_t* sorted128, int32_t target) {
    // SIMDBlockDecoder::advance counts values < target (simd_block_decoder.rs:100-128)
    int n = 0;
    for (int i = 0; i < 128; i++) n += sorted128[i] < target;
    return n;
}

static std::vector<ScorerPtr> mock_children(const int32_t* lists, const uint32_t* lens, uint32_t n) {
    std::vector<ScorerPtr> v;
    size_t off = 0;
    for (uint32_t i = 0; i < n; i++) {
        v.emplace_back(new MockScorer(std::vector<int32_t>(lists + off, lists + off + lens[i])));
        off += lens[i];
    }
    return v;
}
static int drain(Scorer& s, int32_t* out_docs, float* out_scores, uint32_t cap) {
    uint32_t n = 0;
    for (;;) {
        int32_t d = s.next();
        if (d == NO_MORE_DOCS) break;
        if (n >= cap) throw Error("output capacity exceeded");
        out_docs[n] = d;
        out_scores[n] = s.score();
        n++;
    }
    return (int)n;
}
int orc_mock_conjunction(const int32_t* lists, const uint32_t* lens, uint32_t n_lists,
                         int32_t* out_docs, float* out_scores, uint32_t cap) {
    ORC_TRY
    if (n_lists < 2) throw Error("conjunction needs >= 2 children");
    ConjunctionScorer c(mock_children(lists, lens, n_lists));
    return drain(c, out_docs, out_scores, cap);
    ORC_CATCH(-1)
}
int orc_mock_disjunction(const int32_t* lists, const uint32_t* lens, uint32_t n_lists,
                         int32_t msm, int32_t* out_docs, float* out_scores, uint32_t cap) {
    ORC_TRY
    DisjunctionSumScorer d(mock_children(lists, lens, n_lists), true, msm);
    return drain(d, out_docs, out_scores, cap);
    ORC_CATCH(-1)
}
int orc_mock_req_opt(const int32_t* req, uint32_t n_req, const int32_t* opt, uint32_t n_opt,
                     int32_t* out_docs, float* out_scores, uint32_t cap) {
    ORC_TRY
    ReqOptScorer s(ScorerPtr(new MockScorer(std::vector<int32_t>(req, req + n_req))),
                   ScorerPtr(new MockScorer(std::vector<int32_t>(opt, opt + n_opt))));
    return drain(s, out_docs, out_scores, cap);
    ORC_CATCH(-1)
}
int orc_mock_req_not(const int32_t* req, uint32_t n_req, const int32_t* nots, uint32_t n_not,
                     int32_t* out_docs, float* out_scores, uint32_t cap) {
    ORC_TRY
    ReqNotScorer s(ScorerPtr(new MockScorer(std::vector<int32_t>(req, req + n_req))),
                   ScorerPtr(new MockScorer(std::vector<int32_t>(nots, nots + n_not))));
    return drain(s, out_docs, out_scores, cap);
    ORC_CATCH(-1)
}


// Generic mock scorer tree (prefix-coded) for the reference's scorer unit tests:
//   [0,n,doc...] leaf (MockSimpleScorer) | [1,c,child...] Conjunction | [2,msm,c,child...]
//   DisjunctionSum | [3,req,opt] ReqOpt | [4,req,not] ReqNot
static ScorerPtr parse_mock(const int32_t* spec, uint32_t n, uint32_t& pos) {
    if (pos >= n) throw Error("mock spec truncated");
    int32_t kind = spec[pos++];
    if (kind == 0) {
        uint32_t len = (uint32_t)spec[pos++];
        if (pos + len > n) throw Error("mock spec truncated");
        std::vector<int32_t> docs(spec + pos, spec + pos + len);
        pos += len;
        return ScorerPtr(new MockScorer(std::move(docs)));
    }
    if (kind == 1 || kind == 2) {
        int32_t msm = kind == 2 ? spec[pos++] : 0;
        uint32_t c = (uint32_t)spec[pos++];
        std::vector<ScorerPtr> ch;
        for (uint32_t i = 0; i < c; i++) ch.push_back(parse_mock(spec, n, pos));
        if (kind == 1) return ScorerPtr(new ConjunctionScorer(std::move(ch)));
        return ScorerPtr(new DisjunctionSumScorer(std::move(ch), true, msm));
    }
    if (kind == 3 || kind == 4) {
        ScorerPtr a = parse_mock(spec, n, pos);
        ScorerPtr b = parse_mock(spec, n, pos);
        if (kind == 3) return ScorerPtr(new ReqOptScorer(std::move(a), std::move(b)));
        return ScorerPtr(new ReqNotScorer(std::move(a), std::move(b)));
    }
    throw Error("bad mock spec");
}
// ops: pairs (op, target); op 0 = next(), 1 = advance(target), 2 = score() only. out_docs[i] =
// doc_id() after the op, out_scores[i] = score() (NaN when unpositioned/exhausted and op != 2).
int orc_mock_run(const int32_t* spec, uint32_t n_spec, const int32_t* ops, uint32_t n_ops,
                 int32_t* out_docs, float* out_scores) {
    ORC_TRY
    uint32_t pos = 0;
    ScorerPtr s = parse_mock(spec, n_spec, pos);
    for (uint32_t i = 0; i < n_ops; i++) {
        int32_t op = ops[2 * i], target = ops[2 * i + 1];
        if (op == 0) s->next();
        else if (op == 1) s->advance(target);
        out_docs[i] = s->doc_id();
        bool positioned = out_docs[i] != -1 && out_docs[i] != NO_MORE_DOCS;
        out_scores[i] = (positioned || op == 2) ? s->score() : NAN;
    }
    return 0;
    ORC_CATCH(-1)
}

int orc_topk_stream(const int32_t* docs, const float* scores, uint64_t n, uint32_t k,
                    orc_hit* out_sorted, orc_hit* out_heap_order, uint32_t* out_count) {
    ORC_TRY
    TopDocsHeap h(k);
    for (uint64_t i = 0; i < n; i++) h.collect(docs[i], scores[i]);
    if (out_heap_order)
        for (size_t i = 0; i < h.data.size(); i++) out_heap_order[i] = h.data[i];
    std::vector<orc_hit> hits = h.top_docs();
    *out_count = (uint32_t)hits.size();
    for (size_t i = 0; i < hits.size(); i++) out_sorted[i] = hits[i];
    return 0;
    ORC_CATCH(-1)
}
int orc_topk_merge(const orc_hit* leaf_hits, const uint32_t* leaf_counts, uint32_t n_leaves,
                   uint32_t k, orc_hit* out_sorted, uint32_t* out_count) {
    ORC_TRY
    TopDocsHeap h(k);
    size_t off = 0;
    for (uint32_t l = 0; l < n_leaves; l++) {
        for (uint32_t i = 0; i < leaf_counts[l]; i++) h.add_doc(leaf_hits[off + i].doc, leaf_hits[off + i].score);
        h.total_hits += leaf_counts[l];
        off += leaf_counts[l];
    }
    std::vector<orc_hit> hits = h.top_docs();
    *out_count = (uint32_t)hits.size();
    for (size_t i = 0; i < hits.size(); i++) out_sorted[i] = hits[i];
    return 0;
    ORC_CATCH(-1)
}

uint8_t orc_float_to_byte315(float f) { return float_to_byte315(f); }
float orc_byte315_to_float(uint8_t b) { return byte315_to_float(b); }
float orc_norm_table(int i) { return NORM_TABLE.t[i & 255]; }
float orc_bm25_idf(int64_t df, int64_t dc) { return bm25_idf(df, dc); }
float orc_bm25_avgdl(int64_t s, int64_t dc, int64_t md) { return bm25_avgdl(s, dc, md); }
float orc_bm25_score(float w, float k1, float freq, float norm) { return bm25_score(w, k1, freq, norm); }
void orc_bm25_cache(float k1, float b, float avgdl, float out_cache[256]) { bm25_cache(k1, b, avgdl, out_cache); }
uint8_t orc_encode_norm(float boost, int32_t field_length) {  // bm25_similarity.rs:90-92
    return float_to_byte315(boost / std::sqrt((float)field_length));
}
int orc_hardware_threads(void) { return (int)std::thread::hardware_concurrency(); }

}  // extern "C"
