"""Nested BooleanQuerys through the C++ host mirror (rucene_b200/csrc/host/searcher.hpp):
tests/cpp/nested_mirror_example.cpp compiled with g++ and run on the GPU, its TopDocs compared with the oracle's."""
import subprocess

import numpy as np
import pytest

import nested_oracle as no
import oracle_binding as ob
from rucene_b200 import codec

M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER


def test_cpp_nested_example_builds():
    no.build_mirror_example()


@pytest.mark.gpu
def test_cpp_nested_mirror_matches_oracle():
    exe = no.build_mirror_example()
    out = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    seg = codec.synth_segment(0x5EED0001, 50000, 500, doc_version=1, n_threads=2)
    ix = no.NestedIndex([seg])
    specs = [("bool", [(M, [(1,), (2,)]), (M, [(3,), (4,)])], 0),
             ("bool", [(M, 5), (M, [(6,), (7,)]), (N, 8)], 0),
             ("bool", [(M, [(1,), (2,)]), (S, 3)], 0),
             ("bool", [(F, [(2,), (9,)]), (N, 1)], 0),
             ("bool", [(M, 1), (N, [(2,), (3,)])], 0)]
    oq, oc, og = no.to_arrays(specs)
    hits, counts, total = ix.search_batch(oq, oc, og, 20)
    assert len(lines) == len(specs)
    for i, line in enumerate(lines):
        parts = line.split()
        assert int(parts[0]) == int(total[i]), i
        got = [tuple(int(x) for x in p.split(":")) for p in parts[1:]]
        assert got == [(int(h["doc"]), int(np.float32(h["score"]).view(np.uint32))) for h in hits[i][:counts[i]]], i
