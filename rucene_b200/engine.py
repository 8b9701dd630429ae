"""ctypes binding of librucene_gpu.so (include/rucene_gpu.h).

There is no CPU fallback anywhere in this module: if the CUDA library cannot be built/loaded or
no device is present, every entry point raises.
"""
import ctypes as C
import os

import numpy as np

from . import _build

RG_OK, RG_EINVAL, RG_ENODEVICE, RG_ECUDA, RG_EUNSUPPORTED, RG_ENOMEM = 0, -1, -2, -3, -4, -5
MUST, SHOULD, MUST_NOT, FILTER = 0, 1, 2, 3
Q_BOOLEAN = 1
Q_DISMAX = 2    # rg_query.flags: DisjunctionMaxQuery; min_should_match = bits of the f32 tie breaker
MODE_SEARCH, MODE_SEARCH_PARALLEL = 0, 1
CFG_NO_COLUMNS, CFG_EAGER_COLUMNS, CFG_NO_BITMAPS, CFG_MAXSCORE, CFG_STATS, CFG_TFPLANES, CFG_NO_LISTS = 1, 2, 4, 8, 16, 32, 64   # rg_config.flags (include/rucene_gpu.h)
NO_MORE_DOCS = 0x7FFFFFFF
RESCORE_AVG, RESCORE_MAX, RESCORE_MIN, RESCORE_TOTAL, RESCORE_MULTIPLY = 0, 1, 2, 3, 4   # RescoreMode (rg_rescore_params.mode)

TERM_STATE_DTYPE = np.dtype([("doc_freq", "<i4"), ("singleton_doc_id", "<i4"),
                             ("total_term_freq", "<i8"), ("doc_start_fp", "<i8"),
                             ("skip_offset", "<i8")])
CLAUSE_DTYPE = np.dtype([("occur", "<i4"), ("term_id", "<u4"), ("weight", "<f4"),
                         ("cache_id", "<u4")])
QUERY_DTYPE = np.dtype([("clause_begin", "<u4"), ("n_clauses", "<u4"),
                        ("min_should_match", "<i4"), ("flags", "<u4")])
HIT_DTYPE = np.dtype([("doc", "<i4"), ("score", "<f4")])
CLAUSE_GROUP = 0x200   # rg_clause.occur bit: a pure-SHOULD group of terms, term_id indexes the group array (*_nested)
CLAUSE_RANGE = 0x100   # rg_clause.occur bit: a point-range clause, term_id indexes the range array (*_ranges calls)
RANGE_DTYPE = np.dtype([("field", "<u4"), ("bytes_per_dim", "<u4"), ("lower", "u1", 8), ("upper", "u1", 8)])


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("cand_arena_bytes", C.c_uint64),
                ("range_postings", C.c_uint32), ("flags", C.c_uint32)]


class SearchParams(C.Structure):
    _fields_ = [("k", C.c_uint32), ("k1", C.c_float), ("mode", C.c_uint32),
                ("reserved", C.c_uint32)]


class RescoreParams(C.Structure):
    _fields_ = [("window_size", C.c_uint32), ("query_weight", C.c_float), ("rescore_weight", C.c_float),
                ("mode", C.c_uint32), ("k1", C.c_float), ("reserved", C.c_uint32)]


class EngineError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("rucene_gpu error %d: %s" % (code, msg))
        self.code = code


class Unsupported(EngineError):
    """Plan shape outside the accelerated path (RG_EUNSUPPORTED)."""


_lib = None


def lib():
    """Load (building if stale) librucene_gpu.so; raises if it cannot be built."""
    global _lib
    if _lib is not None:
        return _lib
    # RUCENE_B200_GPU_LIB: load an alternative build of the same library (kernel A/B measurements)
    L = C.CDLL(os.environ.get("RUCENE_B200_GPU_LIB") or _build.build_gpu())
    vp = C.c_void_p
    L.rg_last_error.restype = C.c_char_p
    L.rg_last_error.argtypes = [vp]
    L.rg_engine_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.rg_engine_destroy.argtypes = [vp]
    L.rg_engine_destroy.restype = None
    L.rg_engine_set_stream.argtypes = [vp, vp]
    L.rg_engine_set_flags.argtypes = [vp, C.c_uint32]
    L.rg_engine_column_stats.argtypes = [vp, vp]
    L.rg_engine_list_stats.argtypes = [vp, vp]
    L.rg_engine_launch_count.restype = C.c_uint64
    L.rg_engine_launch_count.argtypes = [vp]
    L.rg_engine_last_kernel_ms.restype = C.c_float
    L.rg_engine_last_kernel_ms.argtypes = [vp, C.c_char_p]
    L.rg_engine_index_bytes.restype = C.c_uint64
    L.rg_engine_index_bytes.argtypes = [vp]
    L.rg_segment_upload.argtypes = [vp, C.c_uint32, C.c_int32, C.c_int32, vp, C.c_size_t, vp, vp,
                                    vp, C.c_uint32]
    L.rg_norm_cache_set.argtypes = [vp, C.c_uint32, vp]
    L.rg_terms_upload.argtypes = [vp, C.c_uint32, vp, vp, vp, C.c_uint32]
    L.rg_terms_lookup.argtypes = [vp, vp, vp, C.c_uint32, vp, vp]
    L.rg_search_batch.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(SearchParams), vp,
                                  vp, vp]
    L.rg_batch_prepare.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(SearchParams),
                                   C.POINTER(vp)]
    L.rg_points_upload.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, C.c_size_t]
    L.rg_batch_prepare_ranges.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(SearchParams), vp,
                                          C.c_uint32, C.POINTER(vp)]
    L.rg_search_batch_ranges.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(SearchParams), vp,
                                         C.c_uint32, vp, vp, vp]
    L.rg_batch_range_stats.argtypes = [vp, vp, vp]
    L.rg_batch_prepare_nested.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(SearchParams), vp,
                                          C.c_uint32, vp, C.c_uint32, C.POINTER(vp)]
    L.rg_search_batch_nested.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(SearchParams), vp,
                                         C.c_uint32, vp, C.c_uint32, vp, vp, vp]
    L.rg_batch_group_stats.argtypes = [vp, vp, vp]
    L.rg_batch_run.argtypes = [vp, vp]
    L.rg_batch_fetch.argtypes = [vp, vp, vp, vp, vp]
    L.rg_batch_destroy.argtypes = [vp, vp]
    L.rg_batch_destroy.restype = None
    L.rg_batch_stats.argtypes = [vp, vp, vp]
    L.rg_batch_debug.argtypes = [vp, vp, vp]
    L.rg_batch_columns.argtypes = [vp, vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    L.rg_batch_leaf_records.argtypes = [vp, vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.rg_batch_run_sharded.argtypes = [vp, vp, vp, C.c_uint32, vp, vp, vp]
    L.rg_merge_leaf_records_device.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32]
    L.rg_merge_fetch.argtypes = [vp, vp, vp, vp]
    L.rg_merge_leaf_records.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp]
    L.rg_batch_rescore.argtypes = [vp, vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(RescoreParams)]
    L.rg_rescore_hits.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(RescoreParams), C.c_uint32, vp, vp,
                                  vp]
    L.rg_batch_rescore_nested.argtypes = [vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32,
                                          C.POINTER(RescoreParams)]
    L.rg_rescore_hits_nested.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32,
                                         C.POINTER(RescoreParams), C.c_uint32, vp, vp, vp]
    L.rg_segment_decode.argtypes = [vp, C.c_uint32, C.c_uint64, C.c_uint64, vp, vp]
    L.rg_forutil_decode.argtypes = [vp, vp, C.c_size_t, vp, C.c_uint32, C.c_int, vp, vp]
    L.rg_blockset_stage.argtypes = [vp, vp, C.c_size_t, vp, C.c_uint32, C.c_int, vp, C.POINTER(vp)]
    L.rg_blockset_decode.argtypes = [vp, vp]
    L.rg_blockset_fetch.argtypes = [vp, vp, vp]
    L.rg_blockset_stats.argtypes = [vp, vp, vp]
    L.rg_blockset_destroy.argtypes = [vp, vp]
    L.rg_blockset_destroy.restype = None
    _lib = L
    return L


def _check(rc, h=None):
    if rc != RG_OK:
        msg = lib().rg_last_error(h).decode(errors="replace")
        raise (Unsupported if rc == RG_EUNSUPPORTED else EngineError)(rc, msg)


def _p(a):
    return None if a is None else a.ctypes.data


class Batch:
    def __init__(self, engine, h, n_queries, k):
        self.engine, self.h, self.n_queries, self.k = engine, h, n_queries, k

    def run(self):
        _check(lib().rg_batch_run(self.engine.h, self.h), self.engine.h)

    def fetch(self):
        hits = np.zeros((self.n_queries, self.k), HIT_DTYPE)
        counts = np.zeros(self.n_queries, np.uint32)
        total = np.zeros(self.n_queries, np.uint64)
        _check(lib().rg_batch_fetch(self.engine.h, self.h, _p(hits), _p(counts), _p(total)),
               self.engine.h)
        return hits, counts, total

    def group_stats(self):
        """Group leads of the last run: items a group led, member postings merged, postings that became holes."""
        out = np.zeros(3, np.uint64)
        _check(lib().rg_batch_group_stats(self.engine.h, self.h, _p(out)), self.engine.h)
        return {"items": int(out[0]), "merged": int(out[1]), "holes": int(out[2])}

    def range_stats(self):
        """Range-lead 128-doc blocks of the last run: skipped, taken whole, scanned."""
        out = np.zeros(3, np.uint64)
        _check(lib().rg_batch_range_stats(self.engine.h, self.h, _p(out)), self.engine.h)
        return {"skipped": int(out[0]), "whole": int(out[1]), "scanned": int(out[2])}

    def stats(self):
        out = np.zeros(8, np.uint64)
        _check(lib().rg_batch_stats(self.engine.h, self.h, _p(out)), self.engine.h)
        return {"items": int(out[0]), "postings": int(out[1]), "algorithmic_bytes": int(out[2]),
                "candidate_slots": int(out[3]), "kernels_per_run": int(out[4]),
                "h2d_bytes": int(out[5]), "or_items": int(out[6]), "and_items": int(out[7])}

    def debug(self):
        """RG_CFG_STATS event counters of the last run (include/rucene_gpu.h: rg_batch_debug)"""
        out = np.zeros(16, np.uint64)
        _check(lib().rg_batch_debug(self.engine.h, self.h, _p(out)), self.engine.h)
        names = ["items", "windows", "windows_scanned_with_bound", "windows_before_theta", "docids_only_counted",
                 "stream_postings", "column_gathers", "refills", "candidates", "steps_scanned", "windows_cut",
                 "windows_scored", "docs_scored"]
        d = {n: int(out[i]) for i, n in enumerate(names)}
        d["column_windows_from_bitmaps"] = int(out[13]) & 0xffffffff   # decode-free k_eval_or: no column cell read
        d["column_windows_swept"] = int(out[13]) >> 32                 # ... every column cell of the window read
        d["decode_free_items"] = int(out[14])   # the planner's routing (no RG_CFG_STATS needed)
        d["and_touched_bytes"] = int(out[15])   # always counted by k_eval_and (no RG_CFG_STATS needed)
        return d

    def columns(self):
        """(number of score columns chosen for this batch, their bytes in HBM)"""
        n, nbytes = C.c_uint32(), C.c_uint64()
        _check(lib().rg_batch_columns(self.engine.h, self.h, C.byref(n), C.byref(nbytes)), self.engine.h)
        return n.value, nbytes.value

    def run_sharded(self, nccl_comm, n_ranks):
        """rg_batch_run_sharded: run + ncclAllGather of the leaf records over the caller's ncclComm_t + leaf-order
        merge, entirely inside the C library."""
        hits = np.zeros((self.n_queries, self.k), HIT_DTYPE)
        counts = np.zeros(self.n_queries, np.uint32)
        total = np.zeros(self.n_queries, np.uint64)
        _check(lib().rg_batch_run_sharded(self.engine.h, self.h, nccl_comm, n_ranks, _p(hits), _p(counts), _p(total)),
               self.engine.h)
        return hits, counts, total

    def leaf_records(self):
        ptr, nbytes = C.c_void_p(), C.c_size_t()
        _check(lib().rg_batch_leaf_records(self.engine.h, self.h, C.byref(ptr), C.byref(nbytes)),
               self.engine.h)
        return ptr.value, nbytes.value

    def close(self):
        if self.h:
            lib().rg_batch_destroy(self.engine.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BlockSet:
    def __init__(self, engine, h, n_blocks):
        self.engine, self.h, self.n_blocks = engine, h, n_blocks

    def decode(self):
        _check(lib().rg_blockset_decode(self.engine.h, self.h), self.engine.h)

    def fetch(self):
        out = np.zeros((self.n_blocks, 128), np.int32)
        _check(lib().rg_blockset_fetch(self.engine.h, self.h, _p(out)), self.engine.h)
        return out

    def stats(self):
        out = np.zeros(4, np.uint64)
        _check(lib().rg_blockset_stats(self.engine.h, self.h, _p(out)), self.engine.h)
        return {"encoded_bytes": int(out[0]), "decoded_bytes": int(out[1]), "blocks": int(out[2]),
                "device_bytes": int(out[3])}

    def close(self):
        if self.h:
            lib().rg_blockset_destroy(self.engine.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """rg_engine handle: one per process / GPU."""

    def __init__(self, device=-1, cand_arena_bytes=0, range_postings=0, flags=0):
        self.h = None
        cfg = Config(device, cand_arena_bytes, range_postings, flags)
        h = C.c_void_p()
        _check(lib().rg_engine_create(C.byref(cfg), C.byref(h)))
        self.h = h.value
        self.n_segments = 0

    def close(self):
        if self.h:
            lib().rg_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream):
        _check(lib().rg_engine_set_stream(self.h, cuda_stream), self.h)

    def set_flags(self, flags):
        _check(lib().rg_engine_set_flags(self.h, flags), self.h)

    def column_stats(self):
        out = np.zeros(4, np.uint64)
        _check(lib().rg_engine_column_stats(self.h, _p(out)), self.h)
        return {"cached": int(out[0]), "bytes": int(out[1]), "built": int(out[2]), "hits": int(out[3])}

    def list_stats(self):
        """persistent scored posting lists (RG_CFG_NO_LISTS turns them off)"""
        out = np.zeros(4, np.uint64)
        _check(lib().rg_engine_list_stats(self.h, _p(out)), self.h)
        return {"cached": int(out[0]), "bytes": int(out[1]), "built": int(out[2]), "hits": int(out[3])}

    def launch_count(self):
        return int(lib().rg_engine_launch_count(self.h))

    def last_kernel_ms(self, which):
        return float(lib().rg_engine_last_kernel_ms(self.h, which.encode()))

    def index_bytes(self):
        return int(lib().rg_engine_index_bytes(self.h))

    def upload_segment(self, seg, doc_base=None):
        """seg: codec.Segment-like.  Segments go up in leaf order; doc_base defaults to the
        running sum of max_doc (IndexReader::leaves())."""
        if doc_base is None:
            doc_base = getattr(self, "_next_base", 0)
        terms = np.ascontiguousarray(seg.terms).astype(TERM_STATE_DTYPE, copy=False)
        doc_file = np.ascontiguousarray(seg.doc_file)
        norms = None if seg.norms is None else np.ascontiguousarray(seg.norms, dtype=np.uint8)
        live = None if seg.live_docs is None else np.ascontiguousarray(seg.live_docs, dtype=np.uint64)
        _check(lib().rg_segment_upload(self.h, self.n_segments, doc_base, seg.max_doc, _p(doc_file),
                                       doc_file.size, _p(norms), _p(live), _p(terms), len(terms)),
               self.h)
        self.n_segments += 1
        self._next_base = doc_base + seg.max_doc

    @staticmethod
    def _pack_terms(terms):
        blob = b"".join(terms)
        off = np.zeros(len(terms) + 1, np.uint64)
        if terms:
            off[1:] = np.cumsum([len(t) for t in terms])
        return np.frombuffer(blob, np.uint8) if blob else np.zeros(1, np.uint8), off

    def upload_terms(self, seg_ord, terms, term_ids=None):
        """terms: list of bytes in dictionary order (sorted, unique); term_ids: engine-wide id per entry."""
        blob, off = self._pack_terms(list(terms))
        ids = None if term_ids is None else np.ascontiguousarray(term_ids, dtype=np.uint32)
        _check(lib().rg_terms_upload(self.h, seg_ord, _p(blob), _p(off), _p(ids), len(terms)), self.h)

    def lookup_terms(self, terms):
        """-> (engine-wide term ids, doc_freq[n_segments][n]) resolved on the device."""
        terms = list(terms)
        blob, off = self._pack_terms(terms)
        ids = np.zeros(len(terms), np.uint32)
        df = np.zeros((max(1, self.n_segments), len(terms)), np.int32)
        _check(lib().rg_terms_lookup(self.h, _p(blob), _p(off), len(terms), _p(ids), _p(df)), self.h)
        return ids, df

    def set_norm_cache(self, cache_id, cache):
        c = np.ascontiguousarray(cache, dtype=np.float32)
        assert c.shape == (256,)
        _check(lib().rg_norm_cache_set(self.h, cache_id, _p(c)), self.h)

    @staticmethod
    def _params(k, k1, mode):
        return SearchParams(k, k1, mode, 0)

    def search_batch(self, queries, clauses, k, k1=1.2, mode=MODE_SEARCH):
        q = np.ascontiguousarray(queries, dtype=QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=CLAUSE_DTYPE)
        hits = np.zeros((len(q), k), HIT_DTYPE)
        counts = np.zeros(len(q), np.uint32)
        total = np.zeros(len(q), np.uint64)
        p = self._params(k, k1, mode)
        _check(lib().rg_search_batch(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), _p(hits),
                                     _p(counts), _p(total)), self.h)
        return hits, counts, total

    def prepare(self, queries, clauses, k, k1=1.2, mode=MODE_SEARCH, ranges=None, groups=None):
        """ranges (RANGE_DTYPE array, may be empty): clauses with CLAUSE_RANGE in occur are point ranges.
        groups (QUERY_DTYPE array, may be empty): clauses with CLAUSE_GROUP in occur are pure-SHOULD groups."""
        q = np.ascontiguousarray(queries, dtype=QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=CLAUSE_DTYPE)
        p = self._params(k, k1, mode)
        h = C.c_void_p()
        if groups is not None:
            g = np.ascontiguousarray(groups, dtype=QUERY_DTYPE)
            r = None if ranges is None else np.ascontiguousarray(ranges, dtype=RANGE_DTYPE)
            _check(lib().rg_batch_prepare_nested(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), _p(r),
                                                 0 if r is None else len(r), _p(g), len(g), C.byref(h)), self.h)
        elif ranges is None:
            _check(lib().rg_batch_prepare(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), C.byref(h)),
                   self.h)
        else:
            r = np.ascontiguousarray(ranges, dtype=RANGE_DTYPE)
            _check(lib().rg_batch_prepare_ranges(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), _p(r), len(r),
                                                 C.byref(h)), self.h)
        return Batch(self, h.value, len(q), k)

    def search_batch_ranges(self, queries, clauses, ranges, k, k1=1.2, mode=MODE_SEARCH):
        q = np.ascontiguousarray(queries, dtype=QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=CLAUSE_DTYPE)
        r = np.ascontiguousarray(ranges, dtype=RANGE_DTYPE)
        hits = np.zeros((len(q), k), HIT_DTYPE)
        counts = np.zeros(len(q), np.uint32)
        total = np.zeros(len(q), np.uint64)
        p = self._params(k, k1, mode)
        _check(lib().rg_search_batch_ranges(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), _p(r), len(r),
                                            _p(hits), _p(counts), _p(total)), self.h)
        return hits, counts, total

    def search_batch_nested(self, queries, clauses, groups, k, k1=1.2, mode=MODE_SEARCH, ranges=None):
        """groups (QUERY_DTYPE): the pure-SHOULD groups that CLAUSE_GROUP clauses name; ranges may be None."""
        q = np.ascontiguousarray(queries, dtype=QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=CLAUSE_DTYPE)
        g = np.ascontiguousarray(groups, dtype=QUERY_DTYPE)
        r = None if ranges is None else np.ascontiguousarray(ranges, dtype=RANGE_DTYPE)
        hits = np.zeros((len(q), k), HIT_DTYPE)
        counts = np.zeros(len(q), np.uint32)
        total = np.zeros(len(q), np.uint64)
        p = self._params(k, k1, mode)
        _check(lib().rg_search_batch_nested(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), _p(r),
                                            0 if r is None else len(r), _p(g), len(g), _p(hits), _p(counts),
                                            _p(total)), self.h)
        return hits, counts, total

    def upload_points(self, seg_ord, field, bytes_per_dim, docs, packed):
        """Every 1-D point of one field of leaf seg_ord: docs[i] has the packed sortable value packed[i]
        (uint8 [n, bytes_per_dim]); any order, a doc may repeat."""
        d = np.ascontiguousarray(docs, dtype=np.int32)
        v = np.ascontiguousarray(packed, dtype=np.uint8).reshape(-1)
        if v.size != d.size * bytes_per_dim:
            raise ValueError("packed must hold len(docs) * bytes_per_dim bytes")
        _check(lib().rg_points_upload(self.h, seg_ord, field, bytes_per_dim, _p(d), _p(v), d.size), self.h)

    # ---- QueryRescorer (rescorer.rs) ----
    @staticmethod
    def _rescore_params(window_size, query_weight, rescore_weight, mode, k1):
        return RescoreParams(min(int(window_size), 0xFFFFFFFF), query_weight, rescore_weight, mode, k1, 0)

    @staticmethod
    def _nested_arrays(groups, ranges):
        g = None if groups is None else np.ascontiguousarray(groups, dtype=QUERY_DTYPE)
        r = None if ranges is None else np.ascontiguousarray(ranges, dtype=RANGE_DTYPE)
        return g, r, 0 if g is None else len(g), 0 if r is None else len(r)

    def rescore_batch(self, batch, queries, clauses, window_size, query_weight=1.0, rescore_weight=1.0,
                      mode=RESCORE_TOTAL, k1=1.2, groups=None, ranges=None):
        """rg_batch_rescore: after batch.run(), before batch.fetch(); rescores the batch's rows on the device.
        groups / ranges (the rescoring queries' own arrays, either may be None): rg_batch_rescore_nested."""
        q = np.ascontiguousarray(queries, dtype=QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=CLAUSE_DTYPE)
        p = self._rescore_params(window_size, query_weight, rescore_weight, mode, k1)
        if groups is None and ranges is None:
            _check(lib().rg_batch_rescore(self.h, batch.h, _p(q), len(q), _p(c), len(c), C.byref(p)), self.h)
            return
        g, r, ng, nr = self._nested_arrays(groups, ranges)
        _check(lib().rg_batch_rescore_nested(self.h, batch.h, _p(q), len(q), _p(c), len(c), _p(r), nr, _p(g), ng,
                                             C.byref(p)), self.h)

    def rescore_hits(self, queries, clauses, hits, counts, total, window_size, query_weight=1.0, rescore_weight=1.0,
                     mode=RESCORE_TOTAL, k1=1.2, groups=None, ranges=None):
        """rg_rescore_hits over host rows (hits [n, k] of HIT_DTYPE); returns the rescored copy of hits.
        groups / ranges (either may be None): rg_rescore_hits_nested."""
        q = np.ascontiguousarray(queries, dtype=QUERY_DTYPE)
        c = np.ascontiguousarray(clauses, dtype=CLAUSE_DTYPE)
        h = np.array(hits, dtype=HIT_DTYPE, copy=True, order="C").reshape(len(q), -1)
        n = np.ascontiguousarray(counts, dtype=np.uint32)
        t = np.ascontiguousarray(total, dtype=np.uint64)
        p = self._rescore_params(window_size, query_weight, rescore_weight, mode, k1)
        if groups is None and ranges is None:
            _check(lib().rg_rescore_hits(self.h, _p(q), len(q), _p(c), len(c), C.byref(p), h.shape[1], _p(h), _p(n),
                                         _p(t)), self.h)
            return h
        g, r, ng, nr = self._nested_arrays(groups, ranges)
        _check(lib().rg_rescore_hits_nested(self.h, _p(q), len(q), _p(c), len(c), _p(r), nr, _p(g), ng, C.byref(p),
                                            h.shape[1], _p(h), _p(n), _p(t)), self.h)
        return h

    def merge_leaf_records(self, dev_ptr, n_leaves, n_queries, k):
        hits = np.zeros((n_queries, k), HIT_DTYPE)
        counts = np.zeros(n_queries, np.uint32)
        total = np.zeros(n_queries, np.uint64)
        _check(lib().rg_merge_leaf_records(self.h, dev_ptr, n_leaves, n_queries, k, _p(hits),
                                           _p(counts), _p(total)), self.h)
        return hits, counts, total

    def merge_leaf_records_device(self, dev_ptr, n_leaves, n_queries, k):
        """finish_parallel on the device; the result stays there until merge_fetch()."""
        _check(lib().rg_merge_leaf_records_device(self.h, dev_ptr, n_leaves, n_queries, k), self.h)
        self._merged = (n_queries, k)

    def merge_fetch(self):
        n_queries, k = self._merged
        hits = np.zeros((n_queries, k), HIT_DTYPE)
        counts = np.zeros(n_queries, np.uint32)
        total = np.zeros(n_queries, np.uint64)
        _check(lib().rg_merge_fetch(self.h, _p(hits), _p(counts), _p(total)), self.h)
        return hits, counts, total

    # ---- block codec ----
    def segment_decode(self, seg_ord, first_block=0, n_blocks=1 << 62, fetch=False):
        """Decode block pairs of an uploaded segment (doc deltas + freqs).  -> (stats, out or None)"""
        stats = np.zeros(4, np.uint64)
        out = None
        if fetch:
            probe = np.zeros(4, np.uint64)
            _check(lib().rg_segment_decode(self.h, seg_ord, first_block, 0, None, _p(probe)), self.h)
            n = int(min(n_blocks, int(probe[3]) - first_block))
            out = np.zeros((n, 2, 128), np.int32)
        _check(lib().rg_segment_decode(self.h, seg_ord, first_block, n_blocks, _p(out), _p(stats)), self.h)
        return {"encoded_bytes": int(stats[0]), "decoded_bytes": int(stats[1]), "blocks": int(stats[2]),
                "segment_blocks": int(stats[3])}, out

    def forutil_decode(self, stream, offsets, doc_version, table):
        stream = np.ascontiguousarray(stream, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        table = np.ascontiguousarray(table, dtype=np.int32)
        out = np.zeros((len(offsets), 128), np.int32)
        _check(lib().rg_forutil_decode(self.h, _p(stream), stream.size, _p(offsets), len(offsets),
                                       doc_version, _p(table), _p(out)), self.h)
        return out

    def stage_blocks(self, stream, offsets, doc_version, table):
        stream = np.ascontiguousarray(stream, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        table = np.ascontiguousarray(table, dtype=np.int32)
        h = C.c_void_p()
        _check(lib().rg_blockset_stage(self.h, _p(stream), stream.size, _p(offsets), len(offsets),
                                       doc_version, _p(table), C.byref(h)), self.h)
        return BlockSet(self, h.value, len(offsets))
