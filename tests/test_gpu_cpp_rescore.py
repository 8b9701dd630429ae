"""QueryRescorer through the C++ host mirror (rucene_b200/csrc/host/searcher.hpp): tests/cpp/rescore_mirror_example.cpp
compiled with g++ and run on the GPU, its rows compared with the oracle's rescorer."""
import os
import subprocess

import numpy as np
import pytest

import helpers
import oracle_binding as ob
import rescore_oracle as ro
from rucene_b200 import _build, codec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build_example():
    exe = os.path.join(ROOT, "tests", "cpp", "rescore_mirror_example")
    src = os.path.join(ROOT, "tests", "cpp", "rescore_mirror_example.cpp")
    lib = os.path.dirname(_build.build_gpu())
    _build.build_codec()
    deps = [src, os.path.join(ROOT, "rucene_b200", "csrc", "host", "searcher.hpp"),
            os.path.join(ROOT, "include", "rucene_gpu.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"),
                               src, "-o", exe, "-L" + lib, "-lrucene_gpu", "-lrucene_codec",
                               "-Wl,-rpath," + lib])
    return exe


def test_cpp_rescore_example_builds():
    _build_example()


@pytest.mark.gpu
def test_cpp_rescore_mirror_matches_oracle():
    exe = _build_example()
    out = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    seg = codec.synth_segment(0x5EED0001, 50000, 500, doc_version=1, n_threads=2)
    ix = helpers.oracle_index([seg])
    q, c = ob.make_queries([("bool", [(ob.SHOULD, 1), (ob.SHOULD, 7), (ob.SHOULD, 30)], 0)])
    hits, counts, total = ix.search_batch(q, c, 20)
    oracle = ro.RescoreIndex([seg])
    requests = [(("bool", [(ob.MUST, 2), (ob.SHOULD, 9), (ob.SHOULD, 30)], 0), 15, 1.0, 2.0, ro.TOTAL),
                (("bool", [(ob.MUST, 1), (ob.MUST, 7), (ob.MUST_NOT, 4)], 0), 40, 0.5, 1.0, ro.MULTIPLY)]
    assert len(lines) == len(requests)
    for line, (spec, window, qw, rw, mode) in zip(lines, requests):
        rq, rc = ob.make_queries([spec])
        want = oracle.rescore(rq, rc, hits, counts, total, window, qw, rw, mode)
        parts = line.split()
        assert int(parts[0]) == total[0]
        got = [tuple(int(x) for x in p.split(":")) for p in parts[1:]]
        assert got == [(int(h["doc"]), int(np.float32(h["score"]).view(np.uint32))) for h in want[0][:counts[0]]]
