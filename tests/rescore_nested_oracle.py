"""ctypes binding of tests/cpp/orc_rescore_nested.cpp — TEST INFRASTRUCTURE: QueryRescorer::rescore with rescoring
queries that hold pure-SHOULD groups and point ranges, over orc_nested.cpp's recursive scorer trees (which include
oracle/oracle.cpp unchanged): the parity reference of the device's nested and range rescoring and the timed CPU
rescorer of scripts/rescore_nested_bench.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import nested_oracle as no
import oracle_binding as ob
import points_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "orc_rescore_nested.cpp")
SO = os.path.join(ROOT, "tests", "cpp", "liborc_rescore_nested.so")
AVG, MAX, MIN, TOTAL, MULTIPLY = 0, 1, 2, 3, 4

_lib = None


def build():
    deps = [SRC, no.SRC, po.SRC, os.path.join(ROOT, "oracle", "oracle.cpp"), os.path.join(ROOT, "oracle", "oracle.h")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        cmd = ["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-pthread", "-shared",
               "-Wl,-Bsymbolic", "-o", SO, SRC]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            raise RuntimeError("orc_rescore_nested build failed:\n" + p.stdout)
    return SO


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp = C.c_void_p
        L.orc_last_error.restype = C.c_char_p
        L.orc_index_create.restype = vp
        L.orc_index_create.argtypes = [C.c_float, C.c_float]
        L.orc_index_destroy.argtypes = [vp]
        L.orc_index_add_segment.argtypes = [vp, vp, C.c_size_t, C.c_int32, vp, vp, vp, C.c_uint32,
                                            C.c_int64, C.c_int64, C.c_int64]
        L.orc_term_weight.argtypes = [vp, C.c_uint32, C.c_float, vp, vp, vp, vp]
        L.orc_points_create.restype = vp
        L.orc_points_destroy.argtypes = [vp]
        L.orc_index_add_points.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, C.c_size_t]
        L.orc_rescore_nested.argtypes = [vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_float,
                                         C.c_float, C.c_int, C.c_uint32, vp, vp, vp, C.c_int]
        _lib = L
    return _lib


class RescoreNestedIndex(no.NestedIndex):
    """nested_oracle.NestedIndex (same index and points) in this library, with orc_rescore_nested."""

    def __init__(self, segs, k1=1.2, b=0.75):
        self.h = lib().orc_index_create(k1, b)
        self.p = lib().orc_points_create()
        self._keep = []
        for seg in segs:
            terms = np.ascontiguousarray(seg.terms).astype(ob.TERM_STATE_DTYPE, copy=False)
            doc_file = np.ascontiguousarray(seg.doc_file)
            norms = None if seg.norms is None else np.ascontiguousarray(seg.norms)
            live = None if seg.live_docs is None else np.ascontiguousarray(seg.live_docs, dtype=np.uint64)
            self._keep += [terms, doc_file, norms, live, seg]
            rc = lib().orc_index_add_segment(self.h, ob._p(doc_file), doc_file.size, seg.max_doc, ob._p(norms),
                                             ob._p(live), ob._p(terms), len(terms), seg.doc_count,
                                             seg.sum_total_term_freq, seg.sum_doc_freq)
            if rc != 0:
                raise ob.OracleError(lib().orc_last_error().decode())

    def add_points(self, seg, field, nbytes, docs, packed):
        d = np.ascontiguousarray(docs, dtype=np.int32)
        v = np.ascontiguousarray(packed, dtype=np.uint8).reshape(-1)
        if lib().orc_index_add_points(self.p, seg, field, nbytes, ob._p(d), ob._p(v), d.size) != 0:
            raise ob.OracleError(lib().orc_last_error().decode())

    def term_weight(self, term_id, boost=1.0):
        w, idf, avgdl = C.c_float(), C.c_float(), C.c_float()
        cache = np.zeros(256, dtype=np.float32)
        lib().orc_term_weight(self.h, term_id, boost, C.byref(w), C.byref(idf), C.byref(avgdl), ob._p(cache))
        return np.float32(w.value)

    def search_batch(self, *a, **kw):
        raise NotImplementedError("search with nested_oracle.NestedIndex")

    def rescore(self, queries, clauses, groups, hits, counts, total, window, query_weight=1.0, rescore_weight=1.0,
                mode=TOTAL, ranges=None, n_threads=1):
        """queries / clauses / groups: nested_oracle.to_arrays; hits [n, k] (doc, score); returns the rescored copy."""
        q = np.ascontiguousarray(queries, dtype=ob.QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=ob.CLAUSE_DTYPE)
        g = np.ascontiguousarray(groups, dtype=ob.QUERY_DTYPE)
        r = np.ascontiguousarray(np.zeros(1, po.RANGE_DTYPE) if ranges is None else ranges, dtype=po.RANGE_DTYPE)
        h = np.array(hits, copy=True, order="C").astype(ob.HIT_DTYPE, copy=False).reshape(len(q), -1)
        n = np.ascontiguousarray(counts, dtype=np.uint32)
        t = np.ascontiguousarray(total, dtype=np.uint64)
        rc = lib().orc_rescore_nested(self.h, self.p, ob._p(q), len(q), ob._p(c), ob._p(r), ob._p(g), len(g),
                                      min(int(window), 0xFFFFFFFF), query_weight, rescore_weight, mode, h.shape[1],
                                      ob._p(h), ob._p(n), ob._p(t), n_threads)
        if rc != 0:
            raise ob.OracleError(lib().orc_last_error().decode())
        return h

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_index_destroy(self.h)
            lib().orc_points_destroy(self.p)
            self.h = None


def build_mirror_example():
    """tests/cpp/rescore_nested_mirror_example.cpp against the C++ host mirror (searcher.hpp) and librucene_gpu.so"""
    from rucene_b200 import _build
    exe = os.path.join(ROOT, "tests", "cpp", "rescore_nested_mirror_example")
    src = os.path.join(ROOT, "tests", "cpp", "rescore_nested_mirror_example.cpp")
    lib_dir = os.path.dirname(_build.build_gpu())
    _build.build_codec()
    deps = [src, os.path.join(ROOT, "rucene_b200", "csrc", "host", "searcher.hpp"),
            os.path.join(ROOT, "include", "rucene_gpu.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"),
                               src, "-o", exe, "-L" + lib_dir, "-lrucene_gpu", "-lrucene_codec",
                               "-Wl,-rpath," + lib_dir])
    return exe
