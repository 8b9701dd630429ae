"""The oracle pinned against every known-answer vector the reference's own tests hold for the
hot path (SURVEY.md §4 / §8c).  Each test names the reference test it transcribes
(paths relative to src/core/ of zhihu/rucene).  CPU only."""
import math

import numpy as np
import pytest

import oracle_binding as ob

NO_MORE = ob.NO_MORE_DOCS


# ---- codec/postings/for_util.rs:53-56 test_max_data_size -------------------------------
def test_max_data_size():
    assert ob.lib().orc_max_data_size() == 147


# ---- util/packed/packed_simd.rs:470-505 test_pack_unpack_bits ---------------------------
def test_pack_unpack_bits():
    d1 = np.zeros(128, np.uint32)
    d5 = np.zeros(128, np.uint32)
    d31 = np.zeros(128, np.uint32)
    for i in range(0, 128, 5):
        d1[i] = 1
        d5[i] = 0b10000 | (i & 0b1111)
        d31[i] = 0x40000000 | i
    dec = ob.simd_unpack(ob.simd_pack(d1, 1), 1)
    assert np.array_equal(dec, d1)
    assert [int(dec[i]) for i in (0, 1, 4, 5, 6, 34, 35, 36)] == [1, 0, 0, 1, 0, 0, 1, 0]
    dec = ob.simd_unpack(ob.simd_pack(d5, 5), 5)
    assert np.array_equal(dec, d5)
    assert dec[35] == (0b10000 | (35 & 0b1111))
    dec = ob.simd_unpack(ob.simd_pack(d31, 31), 31)
    assert np.array_equal(dec, d31)
    assert dec[40] == (0x40000000 | 40)


# ---- util/packed/packed_simd.rs:507-525 test_delta_pack_unpack --------------------------
def test_delta_pack_unpack():
    data = (np.arange(1, 129, dtype=np.uint32) * 128)
    assert data[127] == 128 * 128
    assert np.array_equal(ob.simd_unpack(ob.simd_pack(data, 15), 15), data)
    enc = ob.simd_delta_pack(data, 128, 14)
    assert np.array_equal(ob.simd_delta_unpack(enc, 128, 14), data)


# ---- util/packed/packed_simd.rs:404-443 test_max_bits_num, test_direct_copy -------------
def test_max_bits_num_and_direct_copy():
    d = np.arange(128, dtype=np.uint32) * 5
    assert ob.lib().orc_simd_max_bits(d.ctypes.data) == int(d.max()).bit_length()
    d = np.zeros(128, np.uint32)
    d[:3] = [0b10101, 0b1000000111, 0b11101]
    assert ob.lib().orc_simd_max_bits(d.ctypes.data) == 10
    data = np.array([(i % 9) * (i + 1) for i in range(128)], dtype=np.uint32)
    enc = ob.simd_pack(data, 32)
    assert enc.tobytes() == data.tobytes()  # b=32 is a memcpy of the little-endian words
    dec = ob.simd_unpack(enc, 32)
    assert dec[0] == 0 and dec[1] == 2 and dec[9] == 0 and dec[10] == 11
    assert np.array_equal(dec, data)


def test_simd_layout_is_4_lane_interleaved_lsb_first():
    """SURVEY 8a-2: value n lives in lane n%4 at lane-stream index n/4, LSB first."""
    rng = np.random.default_rng(7)
    for b in range(1, 33):
        vals = rng.integers(0, 1 << b, 128, dtype=np.uint64).astype(np.uint32)
        enc = ob.simd_pack(vals, b)[: 16 * b]
        words = enc.view("<u4").reshape(b, 4)
        for n in (0, 1, 5, 31, 64, 127):
            lane, q = n % 4, n // 4
            j, s = (q * b) // 32, (q * b) % 32
            v = int(words[j, lane]) >> s
            if s + b > 32:
                v |= int(words[j + 1, lane]) << (32 - s)
            assert v & ((1 << b) - 1) == int(vals[n])
        assert np.array_equal(ob.simd_unpack(enc, b), vals)


# ---- codec/postings/partial_block_decoder.rs:128-181 test_get / test_next ---------------
def test_packed_golden_bytes():
    # Packed (big-endian MSB-first stream), b=4: FF FF 00 FF -> F F F F 0 0 F F
    got = ob.packed_decode(0, 4, np.array([0xFF, 0xFF, 0x00, 0xFF], np.uint8), 4)
    assert got.tolist() == [0xF, 0xF, 0xF, 0xF, 0, 0, 0xF, 0xF]
    # PackedSingleBlock b=6: two big-endian longs, 10 values each, LSB-first inside the long
    data = np.array([0xFF, 0xF, 0, 0, 0, 0, 0xFF, 0, 0x8F, 0xFF, 0x8F, 0x8F, 0x8F, 0x8F, 0x8F, 0x8F],
                    np.uint8)
    got = ob.packed_decode(1, 6, data, 2)
    assert len(got) == 20
    assert got[0] == 0 and got[1] == 0x3C and got[2] == 0xF and got[3] == 0
    assert got[9] == 0x3C and got[10] == 0xF and got[11] == 0x3E


def test_compact_format_table():
    """FormatAndBits::fastest(128, b, COMPACT): PackedSingleBlock for b in {1,2,4} only
    (packed_misc.rs:474-531), identical encoded size 16*b for every layout."""
    import ctypes as C
    for b in range(1, 33):
        out = C.c_int()
        fmt = ob.lib().orc_fastest_format(b, 0.0, C.byref(out))
        assert out.value == b
        assert fmt == (1 if b in (1, 2, 4) else 0)
        assert ob.lib().orc_packed_encoded_size(fmt, b) == 16 * b


@pytest.mark.parametrize("fmt", [0, 1])
def test_packed_round_trip_all_widths(fmt):
    rng = np.random.default_rng(11 + fmt)
    widths = range(1, 33) if fmt == 0 else (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 16, 21, 32)
    for b in widths:
        it = ob.lib().orc_packed_iterations(fmt, b)
        vals = rng.integers(0, 1 << b, 160, dtype=np.uint64).astype(np.uint32).astype(np.int32)
        enc = ob.packed_encode(fmt, b, vals, it)
        dec = ob.packed_decode(fmt, b, enc, it)
        assert len(dec) >= 128
        assert np.array_equal(dec[:128], vals[:128])


# ---- codec/postings/simd_block_decoder.rs:168-196 ----------------------------------------
def test_block_advance():
    data = (np.arange(1, 129, dtype=np.int32) * 128)
    f = lambda t: int(data[ob.lib().orc_block_advance(data.ctypes.data, t)])
    assert f(1) == 128 and f(129) == 256 and f(130) == 256 and f(255) == 256
    assert f(256) == 256 and f(257) == 384 and f(16283) == 16384
    idx = lambda t: ob.lib().orc_block_advance(data.ctypes.data, t)
    assert (idx(1), idx(129), idx(512)) == (0, 1, 3)


# ---- search/scorer/conjunction_scorer.rs:163-220 -----------------------------------------
CONJ = ob.conj(ob.leaf([1, 2, 3, 4, 5]), ob.leaf([2, 5]), ob.leaf([2, 3, 4, 5]))


def test_conjunction_iterator_next_and_scorer():
    docs, scores = ob.mock_run(CONJ, [(2, 0), (0, 0), (0, 0), (0, 0)])
    assert docs.tolist() == [-1, 2, 5, NO_MORE]
    assert scores[0] == -3.0 and scores[1] == 6.0 and scores[2] == 15.0


def test_conjunction_iterator_advance():
    docs, _ = ob.mock_run(CONJ, [(1, 1)])
    assert docs.tolist() == [2]
    docs, _ = ob.mock_run(CONJ, [(1, 2), (1, 5), (1, 7)])
    assert docs.tolist() == [2, 5, NO_MORE]


# ---- search/scorer/req_not_scorer.rs:128-167 ----------------------------------------------
REQNOT = ob.req_not(ob.conj(ob.leaf([1, 2, 3, 4, 5, 6, 7, 8, 9]), ob.leaf([2, 3, 5, 7, 9, 10])),
                    ob.disj(0, ob.leaf([2, 5]), ob.leaf([1, 4, 5])))


def test_req_not_next_and_advance():
    docs, _ = ob.mock_run(REQNOT, [(2, 0), (0, 0), (0, 0), (0, 0), (0, 0)])
    assert docs.tolist() == [-1, 3, 7, 9, NO_MORE]
    docs, _ = ob.mock_run(REQNOT, [(1, 1), (1, 4), (1, 8), (1, 10)])
    assert docs.tolist() == [3, 7, 9, NO_MORE]


# ---- search/scorer/req_opt_scorer.rs:106-130 ----------------------------------------------
def test_req_opt_score():
    spec = ob.req_opt(ob.conj(ob.leaf([1, 2, 3, 4, 5]), ob.leaf([2, 3, 5])),
                      ob.disj(0, ob.leaf([2, 5]), ob.leaf([3, 4, 5])))
    docs, scores = ob.mock_run(spec, [(0, 0), (0, 0), (0, 0), (0, 0)])
    assert docs.tolist() == [2, 3, 5, NO_MORE]
    assert scores[:3].tolist() == [6.0, 9.0, 20.0]


# ---- search/scorer/bulk_scorer.rs:167-200, search/collector/top_docs.rs:235-264 -----------
def test_bulk_scorer_and_collect():
    docs = np.array([1, 2, 3, 4, 5], np.int32)
    hits, _ = ob.topk_stream(docs, docs.astype(np.float32), 3)
    assert hits["doc"].tolist() == [5, 4, 3]
    docs = np.array([1, 2, 3, 3, 5], np.int32)
    hits, _ = ob.topk_stream(docs, docs.astype(np.float32), 3)
    assert hits["doc"].tolist() == [5, 3, 3]


def test_topk_tie_semantics_appendix_b():
    """SURVEY Appendix B (emulated std BinaryHeap with the reversed PartialOrd): tie survival and
    tie order follow the heap layout, not the docid."""
    hits, _ = ob.topk_stream([0, 1, 2], [1.0, 1.0, 2.0], 2)
    assert list(zip(hits["doc"].tolist(), hits["score"].tolist())) == [(2, 2.0), (1, 1.0)]
    hits, _ = ob.topk_stream(list(range(6)), [1.0] * 6, 4)
    assert hits["doc"].tolist() == [3, 1, 2, 0]
    hits, _ = ob.topk_stream(list(range(8)), [1, 1, 1, 1, 2, 1, 3, 1], 4)
    assert list(zip(hits["doc"].tolist(), hits["score"].tolist())) == [(6, 3.0), (4, 2.0), (3, 1.0), (1, 1.0)]


def test_disjunction_sum_simple_queue():
    docs, scores = ob.mock_disjunction([[1, 4, 9], [2, 4], [4, 9, 11]])
    assert docs.tolist() == [1, 2, 4, 9, 11]
    assert scores.tolist() == [1.0, 2.0, 12.0, 18.0, 11.0]
    docs, _ = ob.mock_disjunction([[1, 4, 9], [2, 4], [4, 9, 11]], min_should_match=2)
    assert docs.tolist() == [4, 9]


# ---- search/similarity/bm25_similarity.rs:400-465 ----------------------------------------
def test_sane_norm_values():
    t = [ob.lib().orc_norm_table(i) for i in range(256)]
    for i in range(256):
        assert t[i] >= 0 and math.isfinite(t[i])
        if i > 0:
            assert t[i] < t[i - 1]


def test_idf_and_avg_field_length():
    L = ob.lib()
    assert L.orc_bm25_idf(1, 11) == np.float32(math.log(8.0))
    assert L.orc_bm25_idf(1, 32) == np.float32(math.log(22.0))
    assert L.orc_bm25_avgdl(0, 5, 11) == 1.0
    assert L.orc_bm25_avgdl(8, 2, 3) == 4.0
    assert L.orc_bm25_avgdl(9, -1, 3) == 3.0


def test_bm25_similarity():
    L = ob.lib()
    idf = np.float32(L.orc_bm25_idf(1, 32))
    assert abs(float(idf * idf) - 9.5545435) < 1e-6  # get_value_for_normalization = weight^2
    avgdl = L.orc_bm25_avgdl(120, 32, 32)
    cache = np.zeros(256, np.float32)
    L.orc_bm25_cache(1.2, 0.75, avgdl, cache.ctypes.data)
    # MockLeafReader norms: doc 1 = field length 120, doc 2 = length 1000 (index/mod.rs:31-345)
    n1, n2 = L.orc_encode_norm(1.0, 120), L.orc_encode_norm(1.0, 1000)
    s = lambda freq, nb: L.orc_bm25_score(idf, 1.2, freq, cache[nb])
    assert s(100.0, n1) > s(20.0, n1)
    assert s(10.0, n1) > s(10.0, n2)


# ---- util/small_float.rs:76-115 -----------------------------------------------------------
def _origin_float_to_byte(f):
    if f < 0:
        return 0
    bits = int(np.float32(f).view(np.int32))
    mantissa = (bits & 0xFFFFFF) >> 21
    exponent = (((bits >> 24) & 0x7F) - 63) + 15
    if exponent > 31:
        exponent, mantissa = 31, 7
    if exponent < 0 or (exponent == 0 and mantissa == 0):
        exponent, mantissa = 0, 1
    return (exponent << 3) | mantissa


def _origin_byte_to_float(b):
    if b == 0:
        return 0.0
    bits = (((b >> 3) & 31) + 48) << 24 | (b & 7) << 21
    return float(np.uint32(bits).view(np.float32))


def test_small_float():
    L = ob.lib()
    assert L.orc_float_to_byte315(np.float32(5.8123817e-10)) == 1
    assert L.orc_float_to_byte315(0.0) == 0
    assert L.orc_float_to_byte315(np.float32(1.4e-45)) == 1
    assert L.orc_float_to_byte315(np.float32(3.4028235e38)) == 255
    assert L.orc_float_to_byte315(float("inf")) == 255
    assert L.orc_float_to_byte315(-1.4e-45) == 0
    assert L.orc_float_to_byte315(-3.4028235e38) == 0
    assert L.orc_float_to_byte315(float("-inf")) == 0
    rng = np.random.default_rng(3)
    for m in rng.integers(0, 1 << 32, 100000, dtype=np.uint64):
        f = np.uint32(m).view(np.float32)
        if np.isnan(f):
            continue
        if f == 0 and np.signbit(f):
            continue  # -0.0: `f < 0` is false in the origin variant but bits<=0 in the fast one
        assert L.orc_float_to_byte315(f) == _origin_float_to_byte(f), f
    for i in range(256):
        assert L.orc_byte315_to_float(i) == _origin_byte_to_float(i)
