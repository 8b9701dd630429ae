"""PointRangeQuery in the oracle (tests/cpp/orc_points.cpp) against an independent numpy model: the sortable encodings,
the doc sets of PointRangeWeight::create_scorer and ranges inside BooleanQuerys."""
import struct

import numpy as np
import pytest

import oracle_binding as ob
import points_fixtures as pf
import points_oracle as po


def test_int_long_encodings_sort_as_values():
    ints = [-(1 << 31), -5, -1, 0, 1, 7, (1 << 31) - 1]
    longs = [-(1 << 63), -(1 << 40), -1, 0, 1, 1 << 40, (1 << 63) - 1]
    assert [po.int_pack(v) for v in ints] == sorted(po.int_pack(v) for v in ints)
    assert [po.long_pack(v) for v in longs] == sorted(po.long_pack(v) for v in longs)
    assert po.int_pack(0) == b"\x80\x00\x00\x00" and po.long_pack(-1) == b"\x7f" + b"\xff" * 7
    assert np.array_equal(pf.packed_of(4, ints), np.frombuffer(b"".join(po.int_pack(v) for v in ints), np.uint8).reshape(-1, 4))
    assert np.array_equal(pf.packed_of(8, longs), np.frombuffer(b"".join(po.long_pack(v) for v in longs), np.uint8).reshape(-1, 8))


def test_float_double_encodings():
    # numpy model: sortable bits = bits ^ ((bits >> 31) & 0x7fffffff) on the signed view, then the sign flip of pack
    f = np.array([-np.inf, -1.5, -0.0, 0.0, 1e-45, 2.0, np.inf], np.float32)
    b = f.view(np.int32)
    s = (b ^ ((b >> 31) & 0x7FFFFFFF)).view(np.uint32) ^ np.uint32(1 << 31)
    model = s.astype(">u4").view(np.uint8).reshape(-1, 4)
    got = np.frombuffer(b"".join(po.float_pack(float(x)) for x in f), np.uint8).reshape(-1, 4)
    assert np.array_equal(got, model)
    assert [bytes(r) for r in got] == sorted(bytes(r) for r in got)  # -0.0 < +0.0, -inf first
    # NaN bit patterns sort beyond the infinities: positive NaNs last, negative NaNs first
    assert po.float_bits_pack(0x7FC00000) > po.float_pack(float("inf"))
    assert po.float_bits_pack(0xFFC00000) < po.float_pack(float("-inf"))
    d = [float("-inf"), -2.5, -0.0, 0.0, 5e-324, 3.0, float("inf")]
    dp = [po.double_pack(x) for x in d]
    assert dp == sorted(dp)
    bits = struct.unpack("<q", struct.pack("<d", -2.5))[0]
    assert dp[1] == struct.pack(">Q", ((bits ^ ((bits >> 63) & 0x7FFFFFFFFFFFFFFF)) & (2 ** 64 - 1)) ^ (1 << 63))


@pytest.fixture(scope="module")
def fx():
    segs, points = pf.build(3, sizes=(40001, 31007))
    ix = po.PointsIndex(segs)
    for si, leaf in enumerate(points):
        for f, (nb, d, p, _) in leaf.items():
            ix.add_points(si, f, nb, d, p)
    return segs, points, ix


def _ranges(points):
    ts = points[0][pf.TS][3]
    out = [po.make_range(pf.TS, 8, po.long_pack(int(np.percentile(ts, a))), po.long_pack(int(np.percentile(ts, b))))
           for a, b in [(0, 1), (10, 20), (40, 90)]]
    v = int(points[0][pf.TS][3][5])
    out.append(po.make_range(pf.TS, 8, po.long_pack(v), po.long_pack(v)))          # exact query, inclusive bounds
    out.append(po.make_range(pf.TS, 8, po.long_pack(v), po.long_pack(v - 1)))      # lower > upper: nothing
    out.append(po.make_range(pf.UNI, 4, po.int_pack(-(1 << 31)), po.int_pack((1 << 31) - 1)))  # all_docs_match
    out.append(po.make_range(pf.UNI, 4, po.int_pack(-1000), po.int_pack(1 << 30)))
    out.append(po.make_range(pf.PART, 8, po.long_pack(-(1 << 63)), po.long_pack(0)))  # field only in leaf 0
    out.append(po.make_range(pf.TS, 8, po.long_pack(-(1 << 63)), po.long_pack((1 << 63) - 1)))  # TS: docs w/o value
    return out


def test_range_doc_sets_match_the_model(fx):
    segs, points, ix = fx
    for r in _ranges(points):
        for si, seg in enumerate(segs):
            want = pf.model_docs(points[si], r)
            got = ix.range_docs(si, r)
            if want is None:
                assert got is None
            else:
                assert np.array_equal(got, want), (si, r)
    # the shortcut returns every doc; the model agrees because every doc has a value there
    assert len(ix.range_docs(0, _ranges(points)[5])) == segs[0].max_doc


def test_boolean_queries_with_ranges_match_the_model(fx):
    """Conjunctions of one term and one range: docs = term postings & model set, minus deleted docs, scored by the
    term alone (the range adds +0.0f); total_hits from the model."""
    segs, points, ix = fx
    ranges = np.array(_ranges(points), po.RANGE_DTYPE)
    oq, oc = ob.make_queries([("bool", [(ob.MUST, 2), (ob.FILTER | po.RANGE, ri)], 0) for ri in range(len(ranges))])
    hits, counts, total = ix.search_batch(oq, oc, ranges, 10)
    base = ob.Index()
    for s in segs:
        base.add_segment(s)
    for ri in range(len(ranges)):
        want_total = 0
        for si, seg in enumerate(segs):
            d = pf.model_docs(points[si], ranges[ri])
            if d is None:
                continue
            post = base.postings(si, 2, 1 << 20)[0]
            live = np.ones(seg.max_doc, bool) if seg.live_docs is None else \
                ((seg.live_docs[np.arange(seg.max_doc) >> 6] >> (np.arange(seg.max_doc) & 63).astype(np.uint64)) & 1).astype(bool)
            m = np.intersect1d(post, d)
            want_total += int(live[m].sum())
        assert int(total[ri]) == want_total, ri


def test_deleted_docs_are_not_collected(fx):
    segs, points, ix = fx
    r = np.array([po.make_range(pf.UNI, 4, po.int_pack(-(1 << 31)), po.int_pack((1 << 31) - 1))], po.RANGE_DTYPE)
    oq, oc = ob.make_queries([("bool", [(ob.MUST | po.RANGE, 0)], 0)])
    hits, counts, total = ix.search_batch(oq, oc, r, 5)
    n_live1 = sum(bin(int(w)).count("1") for w in segs[1].live_docs)
    assert int(total[0]) == segs[0].max_doc + n_live1
    assert np.all(hits[0]["score"].view(np.uint32) == 0)
