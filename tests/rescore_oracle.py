"""ctypes binding of tests/cpp/orc_rescore.cpp — TEST INFRASTRUCTURE: QueryRescorer::rescore over the oracle's own
scorer trees (that file includes oracle/oracle.cpp unchanged), the parity reference of the device's rescoring and the
timed CPU rescorer of scripts/rescore_bench.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "orc_rescore.cpp")
SO = os.path.join(ROOT, "tests", "cpp", "liborc_rescore.so")
AVG, MAX, MIN, TOTAL, MULTIPLY = 0, 1, 2, 3, 4

_lib = None


def build():
    deps = [SRC, os.path.join(ROOT, "oracle", "oracle.cpp"), os.path.join(ROOT, "oracle", "oracle.h")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        # the oracle's own flags; -Bsymbolic: this library's orc_* calls stay inside it next to liboracle.so
        cmd = ["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-pthread", "-shared",
               "-Wl,-Bsymbolic", "-o", SO, SRC]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            raise RuntimeError("orc_rescore build failed:\n" + p.stdout)
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
        L.orc_rescore.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.c_float, C.c_float, C.c_int, C.c_uint32, vp,
                                  vp, vp, C.c_int]
        _lib = L
    return _lib


class RescoreIndex:
    """The oracle's index over `segs` (leaf order, doc_base = running max_doc) with orc_rescore."""

    def __init__(self, segs, k1=1.2, b=0.75):
        self.h = lib().orc_index_create(k1, b)
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

    def rescore(self, queries, clauses, hits, counts, total, window, query_weight=1.0, rescore_weight=1.0,
                mode=TOTAL, n_threads=1):
        """queries / clauses: oracle_binding.make_queries arrays; hits [n, k] (doc, score); returns the rescored copy."""
        q = np.ascontiguousarray(queries, dtype=ob.QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=ob.CLAUSE_DTYPE)
        h = np.array(hits, copy=True, order="C").astype(ob.HIT_DTYPE, copy=False).reshape(len(q), -1)
        n = np.ascontiguousarray(counts, dtype=np.uint32)
        t = np.ascontiguousarray(total, dtype=np.uint64)
        rc = lib().orc_rescore(self.h, ob._p(q), len(q), ob._p(c), min(int(window), 0xFFFFFFFF), query_weight,
                               rescore_weight, mode, h.shape[1], ob._p(h), ob._p(n), ob._p(t), n_threads)
        if rc != 0:
            raise ob.OracleError(lib().orc_last_error().decode())
        return h

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_index_destroy(self.h)
            self.h = None
