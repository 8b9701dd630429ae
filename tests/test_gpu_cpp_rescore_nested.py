"""Rescoring with nested groups through the C++ host mirror (rucene_b200/csrc/host/searcher.hpp):
tests/cpp/rescore_nested_mirror_example.cpp compiled with g++ and run on the GPU, its rescored TopDocs compared with
the oracle's rescorer."""
import subprocess

import numpy as np
import pytest

import nested_oracle as no
import oracle_binding as ob
import rescore_nested_oracle as rno
from rucene_b200 import codec

M, S, N, F = ob.MUST, ob.SHOULD, ob.MUST_NOT, ob.FILTER


def test_cpp_rescore_nested_example_builds():
    rno.build_mirror_example()


@pytest.mark.gpu
def test_cpp_rescore_nested_mirror_matches_oracle():
    exe = rno.build_mirror_example()
    out = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    seg = codec.synth_segment(0x5EED0001, 50000, 500, doc_version=1, n_threads=2)
    ix, rx = no.NestedIndex([seg]), rno.RescoreNestedIndex([seg])
    fq, fc, fg = no.to_arrays([("bool", [(S, 1), (S, 2), (S, 3), (S, 5), (S, 9)], 0)])
    requests = [(("bool", [(M, [(1,), (2,)]), (M, [(3,), (4,)])], 0), 1.0, 2.0, rno.TOTAL, 15),
                (("bool", [(M, 5), (N, [(6,), (7,)])], 0), 0.5, 1.0, rno.MULTIPLY, 40),
                (("bool", [(M, [(1,), (2,)]), (S, 3), (S, [(9,), (8,)])], 0), 1.0, 1.0, rno.AVG, 20)]
    assert len(lines) == len(requests)
    for i, (spec, qw, rw, mode, window) in enumerate(requests):
        hits, counts, total = ix.search_batch(fq, fc, fg, 20)
        oq, oc, og = no.to_arrays([spec])
        want = rx.rescore(oq, oc, og, hits, counts, total, window, qw, rw, mode)
        parts = lines[i].split()
        assert int(parts[0]) == int(total[0]), i
        got = [tuple(int(x) for x in p.split(":")) for p in parts[1:]]
        assert got == [(int(h["doc"]), int(np.float32(h["score"]).view(np.uint32))) for h in want[0][:counts[0]]], i
