"""PointRangeQuery through the C++ host mirror (rucene_b200/csrc/host/searcher.hpp): tests/cpp/points_mirror_example.cpp
compiled with g++ and run on the GPU, its TopDocs compared with the oracle's."""
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import points_oracle as po
from rucene_b200 import codec, search

R = po.RANGE


def test_cpp_points_example_builds():
    po.build_mirror_example()


@pytest.mark.gpu
def test_cpp_points_mirror_matches_oracle():
    exe = po.build_mirror_example()
    out = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    seg = codec.synth_segment(0x5EED0001, 50000, 500, doc_version=1, n_threads=2)
    d = np.arange(seg.max_doc)
    ts_docs = np.concatenate([d[d % 7 != 0], d[d % 5 == 0]])
    ts_vals = np.concatenate([d[d % 7 != 0] * 10, d[d % 5 == 0] * 10 + 3])
    fv = ((d % 201 - 100) / 4.0).astype(np.float32)
    fv[d % 402 == 100] = np.float32(-0.0)
    ix = po.PointsIndex([seg])
    ix.add_points(0, 0, 8, ts_docs, np.frombuffer(b"".join(search.LongPoint.pack(int(v)) for v in ts_vals), np.uint8))
    ix.add_points(0, 1, 4, d, np.frombuffer(b"".join(search.FloatPoint.pack(float(v)) for v in fv), np.uint8))
    L, F = search.LongPoint.pack, search.FloatPoint.pack
    ranges = np.array([po.make_range(0, 8, L(1000), L(200003)), po.make_range(0, 8, L(50000), L(400000)),
                       po.make_range(1, 4, F(-0.0), F(5.0)), po.make_range(0, 8, L(1000), L(1000)),
                       po.make_range(1, 4, F(0.0), F(25.0)), po.make_range(1, 4, F(-0.0), F(-0.0))], po.RANGE_DTYPE)
    specs = [("bare", 0), ("bool", [(ob.MUST, 2), (ob.FILTER | R, 1)]),
             ("bool", [(ob.MUST, 1), (ob.MUST | R, 2), (ob.MUST_NOT | R, 3)]),
             ("bool", [(ob.SHOULD, 1), (ob.SHOULD, 7), (ob.FILTER | R, 4)]), ("bool", [(ob.FILTER | R, 5)])]
    qs, cs = [], []
    for s in specs:
        if s[0] == "bare":
            qs.append((len(cs), 1, 0, 0))
            cs.append((ob.SHOULD | R, s[1], 0.0))
        else:
            qs.append((len(cs), len(s[1]), 0, 1))
            cs += [(o, t, 0.0 if o & R else 1.0) for o, t in s[1]]
    hits, counts, total = ix.search_batch(np.array(qs, ob.QUERY_DTYPE), np.array(cs, ob.CLAUSE_DTYPE), ranges, 20)
    assert len(lines) == len(specs)
    for i, line in enumerate(lines):
        parts = line.split()
        assert int(parts[0]) == int(total[i]), i
        got = [tuple(int(x) for x in p.split(":")) for p in parts[1:]]
        assert got == [(int(h["doc"]), int(np.float32(h["score"]).view(np.uint32))) for h in hits[i][:counts[i]]], i
