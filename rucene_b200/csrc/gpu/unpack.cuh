// unpack.cuh — ForUtil block decode on the device (pure integer work, no tensor cores).
//
// One warp decodes one 128-value block; lane q produces values n = 4q .. 4q+3, so the decoded
// block leaves the warp as one coalesced 512-byte store (or stays in registers for the fused
// query kernels).  Payload parts are 16-byte aligned in the HBM image (common.cuh), which makes
// every load a 128-bit (SIMD128 layout) or aligned 32-bit (big-endian layouts) access.
//
// Reference semantics (paths relative to src/core/ of zhihu/rucene):
//   SIMD128 (".doc" version 1): util/packed/packed_simd.rs:126-163 unpack_bits!
//       value n -> lane l = n%4, lane-stream slot q = n/4; v = (W[j][l] >> s | W[j+1][l] << (32-s))
//       & mask with j = q*b/32, s = q*b%32 over little-endian words.
//   Packed (version 0): util/packed/packed_misc.rs:2655-2680 — one MSB-first big-endian stream,
//       value n at bit n*b.
//   PackedSingleBlock (version 0, b in {1,2,4} under COMPACT): packed_misc.rs:2829-2841,
//       2739-2755 — 64/b values per big-endian long, value i of a long at bits [i*b, i*b+b).
//   all-equal (code 0): codec/postings/for_util.rs:210-221.
#pragma once
#include "common.cuh"

namespace rg {

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// ---- SIMD128 ----------------------------------------------------------------------------
__device__ __forceinline__ int4 unpack4_simd128(const uint4* __restrict__ part, int b, int q) {
    if (b == 32) {
        uint4 v = ldg16(part + q);
        return make_int4((int)v.x, (int)v.y, (int)v.z, (int)v.w);
    }
    const int bit = q * b;
    const int j = bit >> 5, s = bit & 31;
    const int j2 = min(j + 1, b - 1);  // stays inside the payload; masked out when unused
    const uint4 A = ldg16(part + j);
    const uint4 B = ldg16(part + j2);
    const uint32_t mask = (1u << b) - 1u;
    int4 r;
    r.x = (int)(__funnelshift_r(A.x, B.x, s) & mask);
    r.y = (int)(__funnelshift_r(A.y, B.y, s) & mask);
    r.z = (int)(__funnelshift_r(A.z, B.z, s) & mask);
    r.w = (int)(__funnelshift_r(A.w, B.w, s) & mask);
    return r;
}
// one value (random access inside a block, used for lazy freq lookups)
__device__ __forceinline__ int extract_simd128(const uint4* __restrict__ part, int b, int n) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(part);
    const int lane = n & 3, q = n >> 2;
    if (b == 32) return (int)__ldg(w + q * 4 + lane);
    const int bit = q * b;
    const int j = bit >> 5, s = bit & 31;
    const int j2 = min(j + 1, b - 1);
    const uint32_t lo = __ldg(w + j * 4 + lane), hi = __ldg(w + j2 * 4 + lane);
    return (int)(__funnelshift_r(lo, hi, s) & ((1u << b) - 1u));
}

// ---- Packed (big-endian bit stream) ------------------------------------------------------
__device__ __forceinline__ int extract_packed_be(const uint32_t* __restrict__ w, int b, int n) {
    const int bit = n * b;
    const int wi = bit >> 5, s = bit & 31;
    const int wi2 = min(wi + 1, 4 * b - 1);
    const uint32_t hi = bswap32(__ldg(w + wi)), lo = bswap32(__ldg(w + wi2));
    return (int)(__funnelshift_l(lo, hi, s) >> (32 - b));
}
// ---- PackedSingleBlock -------------------------------------------------------------------
__device__ __forceinline__ int extract_single_block(const uint32_t* __restrict__ w, int b, int n) {
    const int per = 64 / b;
    const int L = n / per, i = n - L * per;
    const uint32_t hi = bswap32(__ldg(w + 2 * L)), lo = bswap32(__ldg(w + 2 * L + 1));
    const int sh = i * b;
    const uint32_t mask = b == 32 ? 0xffffffffu : ((1u << b) - 1u);
    const uint32_t v = sh < 32 ? __funnelshift_r(lo, hi, sh) : (hi >> (sh - 32));
    return (int)(v & mask);
}

// ---- generic entry points -----------------------------------------------------------------
// `part`: 16-byte aligned block part; b: num_bits from the block header (0 = all equal).
__device__ __forceinline__ int4 unpack4(const uint4* __restrict__ part, int b, int q, int version,
                                        uint32_t sb_mask) {
    if (b == 0) {
        const int v = (int)__ldg(reinterpret_cast<const uint32_t*>(part));
        return make_int4(v, v, v, v);
    }
    if (version > 0) return unpack4_simd128(part, b, q);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(part);
    int4 r;
    if ((sb_mask >> (b - 1)) & 1u) {
        r.x = extract_single_block(w, b, 4 * q);
        r.y = extract_single_block(w, b, 4 * q + 1);
        r.z = extract_single_block(w, b, 4 * q + 2);
        r.w = extract_single_block(w, b, 4 * q + 3);
    } else {
        r.x = extract_packed_be(w, b, 4 * q);
        r.y = extract_packed_be(w, b, 4 * q + 1);
        r.z = extract_packed_be(w, b, 4 * q + 2);
        r.w = extract_packed_be(w, b, 4 * q + 3);
    }
    return r;
}
__device__ __forceinline__ int extract1(const uint4* __restrict__ part, int b, int n, int version,
                                        uint32_t sb_mask) {
    if (b == 0) return (int)__ldg(reinterpret_cast<const uint32_t*>(part));
    if (version > 0) return extract_simd128(part, b, n);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(part);
    return ((sb_mask >> (b - 1)) & 1u) ? extract_single_block(w, b, n) : extract_packed_be(w, b, n);
}

// Doc-delta block -> absolute docids: the reference accumulates one delta per next()
// (codec/postings/posting_reader.rs:622-640); here a warp-wide inclusive scan, base = last doc
// of the previous block (0 for a term's first block).
__device__ __forceinline__ int4 deltas_to_docs(int4 d, int base) {
    int4 p;
    p.x = d.x;
    p.y = p.x + d.y;
    p.z = p.y + d.z;
    p.w = p.z + d.w;
    int tot = p.w;
    const int lane = lane_id();
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, tot, o);
        if (lane >= o) tot += t;
    }
    const int excl = tot - p.w + base;
    p.x += excl;
    p.y += excl;
    p.z += excl;
    p.w += excl;
    return p;
}

// ---- the reference's other doc-block encodings --------------------------------------------
// EncodeType::EF (Elias-Fano) and EncodeType::BITSET doc blocks (codec/postings/for_util.rs:337-372,
// read side posting_reader.rs:624-633): a block is its 128 docids, not 128 deltas.  Staged layout
// (engine.cu): one 16-byte header, then the raw little-endian longs of the file.
//   BITSET header {min_doc, num_words}: docid = min_doc + position of each set bit (bit_set.rs:351-376)
//   EF     header {num_low_bits L, n_upper, n_lower}: the i-th set bit of the upper array sits at
//          position high_i + i; docid_i = ef_base_doc + 1 + ((high_i << L) | low_i), low_i = the
//          i-th L-bit field of the lower array (elias_fano_decoder.rs:79-108,122-160)
// Warp-cooperative select: 32-bit words, one per lane per round; popcounts are prefix-summed across
// the warp so every set bit knows its rank and scatters its docid to out[rank] (shared memory).
__device__ __forceinline__ void decode_other_docs(const uint4* __restrict__ part, uint32_t enc, int ef_base_doc,
                                                  int32_t* out, int lane) {
    const uint4 hdr = ldg16(part);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(part + 1);
    const bool ef = enc == 1u;
    const uint32_t n32 = 2u * hdr.y;           // upper array (EF) / bitmap (BITSET), in 32-bit words
    const uint32_t L = ef ? hdr.x : 0u;
    const uint32_t* lower = w + n32;
    const uint32_t n_lower32 = ef ? 2u * hdr.z : 0u;
    const uint32_t lmask = L ? ((1u << L) - 1u) : 0u;
    uint32_t rank0 = 0;
    for (uint32_t base = 0; base < n32 && rank0 < (uint32_t)kBlock; base += 32) {
        const uint32_t wi = base + lane;
        uint32_t x = wi < n32 ? __ldg(w + wi) : 0u;
        const uint32_t c = __popc(x);
        uint32_t incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        uint32_t r = rank0 + incl - c;
        while (x) {
            const uint32_t bit = __ffs(x) - 1;
            x &= x - 1;
            if (r < (uint32_t)kBlock) {
                const uint32_t pos = wi * 32u + bit;
                int doc;
                if (ef) {
                    uint32_t low = 0;
                    if (L) {
                        const uint32_t bp = r * L, j = bp >> 5, sh = bp & 31u;
                        const uint32_t lo = __ldg(lower + j);
                        const uint32_t hi = j + 1 < n_lower32 ? __ldg(lower + j + 1) : 0u;
                        low = __funnelshift_r(lo, hi, sh) & lmask;
                    }
                    doc = ef_base_doc + 1 + (int)(((pos - r) << L) | low);
                } else {
                    doc = (int)hdr.x + (int)pos;
                }
                out[r] = doc;
            }
            r++;
        }
        rank0 += __shfl_sync(0xffffffffu, incl, 31);
    }
    __syncwarp();
}

// out-of-line copy for k_eval_and, whose register budget (occupancy) the inlined body would raise
static __device__ __noinline__ void decode_other_docs_call(const uint4* __restrict__ part, uint32_t enc,
                                                           int ef_base_doc, int32_t* out, int lane) {
    decode_other_docs(part, enc, ef_base_doc, out, lane);
}

// vint / vlong readers over a byte pointer (store/io/data_input.rs:78-111)
__device__ __forceinline__ int read_vint(const uint8_t* __restrict__ p, uint32_t& pos) {
    uint32_t b = p[pos++];
    uint32_t v = b & 0x7f;
    int shift = 7;
    while (b & 0x80) {
        b = p[pos++];
        v |= (b & 0x7f) << shift;
        shift += 7;
    }
    return (int)v;
}

}  // namespace rg
