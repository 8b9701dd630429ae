"""ctypes binding of tests/cpp/orc_nested.cpp — TEST INFRASTRUCTURE: pure-SHOULD groups of TermQuerys as clauses of
the oracle's BooleanQuery, beside terms and point ranges (that file includes orc_points.cpp and so oracle/oracle.cpp
unchanged), the parity reference of the device's group clauses."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_binding as ob
import points_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "orc_nested.cpp")
SO = os.path.join(ROOT, "tests", "cpp", "liborc_nested.so")
GROUP = 0x200  # clause occur bit: a group, term_id indexes the group array

_lib = None


def build():
    deps = [SRC, po.SRC, os.path.join(ROOT, "oracle", "oracle.cpp"), os.path.join(ROOT, "oracle", "oracle.h")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        cmd = ["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-pthread", "-shared",
               "-Wl,-Bsymbolic", "-o", SO, SRC]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            raise RuntimeError("orc_nested build failed:\n" + p.stdout)
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
        L.orc_search_batch_nested.argtypes = [vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_int,
                                              C.c_int, vp, vp, vp]
        _lib = L
    return _lib


class NestedIndex:
    """The oracle's index over `segs` plus point fields, searched with group clauses."""

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

    def search_batch(self, queries, clauses, groups, k, ranges=None, parallel_mode=0, n_threads=1):
        q = np.ascontiguousarray(queries, dtype=ob.QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=ob.CLAUSE_DTYPE)
        g = np.ascontiguousarray(groups, dtype=ob.QUERY_DTYPE)
        r = np.ascontiguousarray(np.zeros(1, po.RANGE_DTYPE) if ranges is None else ranges, dtype=po.RANGE_DTYPE)
        hits = np.zeros((len(q), k), ob.HIT_DTYPE)
        counts = np.zeros(len(q), np.uint32)
        total = np.zeros(len(q), np.uint64)
        rc = lib().orc_search_batch_nested(self.h, self.p, ob._p(q), len(q), ob._p(c), ob._p(r), ob._p(g), len(g), k,
                                           parallel_mode, n_threads, ob._p(hits), ob._p(counts), ob._p(total))
        if rc != 0:
            raise ob.OracleError(lib().orc_last_error().decode())
        return hits, counts, total

    def engine_clauses(self, clauses):
        """rg_clause rows: a term's weight = idf * boost, a range's its boost, a group clause's 0; norm cache 0."""
        from rucene_b200 import engine
        out = np.zeros(len(clauses), engine.CLAUSE_DTYPE)
        for i, c in enumerate(clauses):
            out[i]["occur"], out[i]["term_id"] = c["occur"], c["term_id"]
            special = int(c["occur"]) & (po.RANGE | GROUP)
            out[i]["weight"] = c["boost"] if special else self.term_weight(int(c["term_id"]), float(c["boost"]))
        return out

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_index_destroy(self.h)
            lib().orc_points_destroy(self.p)
            self.h = None


def to_arrays(specs):
    """specs: ("bool", [clause...], msm) where a clause is (occur, term_id[, boost]), (occur | RANGE, range_id) or
    (occur, [(term_id[, boost])...][, group_msm]) for a group.  Group members follow all the queries' own clauses.
    Returns (queries, clauses, groups) as oracle arrays."""
    qs, cs, gs, members = [], [], [], []
    for s in specs:
        qs.append((len(cs), len(s[1]), s[2], 1))
        for cl in s[1]:
            if isinstance(cl[1], list):
                cs.append((cl[0] | GROUP, len(gs), 0.0))
                gs.append((cl[1], cl[2] if len(cl) > 2 else 0))
            else:
                cs.append((cl[0], cl[1], cl[2] if len(cl) > 2 else (0.0 if cl[0] & po.RANGE else 1.0)))
    groups = []
    for mem, msm in gs:
        groups.append((len(cs), len(mem), msm, 1))
        for m in mem:
            cs.append((ob.SHOULD, m[0], m[1] if len(m) > 1 else 1.0))
    return (np.array(qs, ob.QUERY_DTYPE), np.array(cs, ob.CLAUSE_DTYPE),
            np.array(groups, ob.QUERY_DTYPE).reshape(-1))


def engine_queries(oq):
    from rucene_b200 import engine
    q = np.zeros(len(oq), engine.QUERY_DTYPE)
    for f in ("clause_begin", "n_clauses", "min_should_match"):
        q[f] = oq[f]
    q["flags"] = np.where(oq["is_boolean"] == 1, engine.Q_BOOLEAN, 0)
    return q


def build_mirror_example():
    """tests/cpp/nested_mirror_example.cpp against the C++ host mirror (searcher.hpp) and librucene_gpu.so"""
    from rucene_b200 import _build
    exe = os.path.join(ROOT, "tests", "cpp", "nested_mirror_example")
    src = os.path.join(ROOT, "tests", "cpp", "nested_mirror_example.cpp")
    lib = os.path.dirname(_build.build_gpu())
    _build.build_codec()
    deps = [src, os.path.join(ROOT, "rucene_b200", "csrc", "host", "searcher.hpp"),
            os.path.join(ROOT, "include", "rucene_gpu.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"),
                               src, "-o", exe, "-L" + lib, "-lrucene_gpu", "-lrucene_codec", "-Wl,-rpath," + lib])
    return exe
