"""ctypes binding of tests/cpp/orc_points.cpp — TEST INFRASTRUCTURE: PointRangeQuery clauses in the oracle's
BooleanQuery (that file includes oracle/oracle.cpp unchanged), the parity reference of the device's range clauses.
Also the point encodings (util/numeric.rs, point_range_query.rs: IntPoint / LongPoint / FloatPoint / DoublePoint
pack) used by the tests."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np

import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "orc_points.cpp")
SO = os.path.join(ROOT, "tests", "cpp", "liborc_points.so")
RANGE = 0x100  # clause occur bit: a range clause, term_id indexes the range array
RANGE_DTYPE = np.dtype([("field", "<u4"), ("bytes_per_dim", "<u4"), ("lower", "u1", 8), ("upper", "u1", 8)])

_lib = None


def build():
    deps = [SRC, os.path.join(ROOT, "oracle", "oracle.cpp"), os.path.join(ROOT, "oracle", "oracle.h")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        cmd = ["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-pthread", "-shared",
               "-Wl,-Bsymbolic", "-o", SO, SRC]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            raise RuntimeError("orc_points build failed:\n" + p.stdout)
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
        L.orc_range_docs.restype = C.c_int64
        L.orc_range_docs.argtypes = [vp, vp, C.c_uint32, vp, vp, C.c_int64]
        L.orc_search_batch_ranges.argtypes = [vp, vp, vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint32, C.c_int,
                                              C.c_int, vp, vp, vp]
        _lib = L
    return _lib


# ---- sortable encodings (util/numeric.rs:163-220) ----
def int_pack(v):
    return struct.pack(">I", (int(v) & 0xFFFFFFFF) ^ 0x80000000)


def long_pack(v):
    return struct.pack(">Q", (int(v) & 0xFFFFFFFFFFFFFFFF) ^ 0x8000000000000000)


def sortable_float_bits(bits):  # i32 bits -> i32: bits ^ ((bits >> 31) & 0x7fffffff)
    b = bits - (1 << 32) if bits & 0x80000000 else bits
    return (b ^ ((b >> 31) & 0x7FFFFFFF)) & 0xFFFFFFFF


def sortable_double_bits(bits):
    b = bits - (1 << 64) if bits & (1 << 63) else bits
    return (b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)) & 0xFFFFFFFFFFFFFFFF


def float_pack(f):
    return float_bits_pack(struct.unpack("<I", struct.pack("<f", f))[0])


def double_pack(f):
    bits = struct.unpack("<Q", struct.pack("<d", f))[0]
    s = sortable_double_bits(bits)
    return long_pack(s - (1 << 64) if s & (1 << 63) else s)


def float_bits_pack(bits):
    """FloatPoint::pack of the f32 with these raw bits (NaN payloads included)."""
    s = sortable_float_bits(bits)
    return int_pack(s - (1 << 32) if s & 0x80000000 else s)


def make_range(field, nbytes, lower, upper):
    r = np.zeros(1, RANGE_DTYPE)[0]
    r["field"], r["bytes_per_dim"] = field, nbytes
    r["lower"][:nbytes] = np.frombuffer(lower, np.uint8)
    r["upper"][:nbytes] = np.frombuffer(upper, np.uint8)
    return r


class PointsIndex:
    """The oracle's index over `segs` plus point fields: add_points(seg, field, nbytes, docs, packed [n, nbytes])."""

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

    def range_docs(self, seg, rng):
        """PointRangeWeight::create_scorer's doc set in leaf seg (None: no scorer)."""
        r = np.ascontiguousarray(np.array([rng], RANGE_DTYPE))
        n = lib().orc_range_docs(self.h, self.p, seg, ob._p(r), None, 0)
        if n == -2:
            raise ob.OracleError(lib().orc_last_error().decode())
        if n < 0:
            return None
        out = np.zeros(max(1, n), np.int32)
        lib().orc_range_docs(self.h, self.p, seg, ob._p(r), ob._p(out), n)
        return out[:n]

    def term_weight(self, term_id, boost=1.0):
        w, idf, avgdl = C.c_float(), C.c_float(), C.c_float()
        cache = np.zeros(256, dtype=np.float32)
        lib().orc_term_weight(self.h, term_id, boost, C.byref(w), C.byref(idf), C.byref(avgdl), ob._p(cache))
        return np.float32(w.value)

    def search_batch(self, queries, clauses, ranges, k, parallel_mode=0, n_threads=1):
        q = np.ascontiguousarray(queries, dtype=ob.QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=ob.CLAUSE_DTYPE)
        r = np.ascontiguousarray(ranges, dtype=RANGE_DTYPE)
        hits = np.zeros((len(q), k), ob.HIT_DTYPE)
        counts = np.zeros(len(q), np.uint32)
        total = np.zeros(len(q), np.uint64)
        rc = lib().orc_search_batch_ranges(self.h, self.p, ob._p(q), len(q), ob._p(c), ob._p(r), len(r), k,
                                           parallel_mode, n_threads, ob._p(hits), ob._p(counts), ob._p(total))
        if rc != 0:
            raise ob.OracleError(lib().orc_last_error().decode())
        return hits, counts, total

    def engine_clauses(self, clauses):
        """The oracle's clause array as rg_clause rows: weight = idf * boost (a range: its boost), norm cache 0."""
        from rucene_b200 import engine
        out = np.zeros(len(clauses), engine.CLAUSE_DTYPE)
        for i, c in enumerate(clauses):
            out[i]["occur"], out[i]["term_id"] = c["occur"], c["term_id"]
            rng = int(c["occur"]) & RANGE
            out[i]["weight"] = c["boost"] if rng else self.term_weight(int(c["term_id"]), float(c["boost"]))
        return out

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_index_destroy(self.h)
            lib().orc_points_destroy(self.p)
            self.h = None


def build_mirror_example():
    """tests/cpp/points_mirror_example.cpp against the C++ host mirror (searcher.hpp) and librucene_gpu.so"""
    from rucene_b200 import _build
    exe = os.path.join(ROOT, "tests", "cpp", "points_mirror_example")
    src = os.path.join(ROOT, "tests", "cpp", "points_mirror_example.cpp")
    lib = os.path.dirname(_build.build_gpu())
    _build.build_codec()
    deps = [src, os.path.join(ROOT, "rucene_b200", "csrc", "host", "searcher.hpp"),
            os.path.join(ROOT, "include", "rucene_gpu.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"),
                               src, "-o", exe, "-L" + lib, "-lrucene_gpu", "-lrucene_codec", "-Wl,-rpath," + lib])
    return exe
