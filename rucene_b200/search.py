"""Python mirror of the reference's search surface for the accelerated path.

Same names and argument meaning as the Rust reference (paths relative to
src/core/ of zhihu/rucene):

    Term                 index/mod.rs Term::new(field, bytes)
    TermQuery            search/query/term_query.rs:46-49    TermQuery::new(term, boost, ctx)
    BooleanQuery.build   search/query/boolean_query.rs:40-87 build(musts, shoulds, filters, must_nots, msm)
    ConstantScoreQuery   search/query/match_all_query.rs:162-205 (what a lone FILTER clause becomes, boost 0)
    MatchAllDocsQuery    search/query/match_all_query.rs:28-116  (what build() adds to a pure MUST_NOT query)
    BM25Similarity       search/similarity/bm25_similarity.rs:45-46 (k1=1.2, b=0.75)
    TopDocsCollector     search/collector/top_docs.rs:107-124 TopDocsCollector::new(k) / top_docs()
    TopDocs / ScoreDoc   search/sort_field/collapse_top_docs.rs:22-68,288-326
    IndexSearcher.search search/searcher.rs:238-240,487-525
    RescoreMode / RescoreRequest / QueryRescorer   search/scorer/rescorer.rs:67-115,130-607
    PointRangeQuery      search/query/point_range_query.rs (1-D: IntPoint / LongPoint / FloatPoint / DoublePoint
                         pack, new_range_query, new_exact_query; sortable bytes of util/numeric.rs:163-220)

Everything that touches postings runs on the GPU through the C ABI (engine.py); this module only
does what Query::create_weight does on the host once per query: collection/term statistics from
the largest segment (searcher.rs:311-351,732-767) and the BM25 weight (bm25_similarity.rs:151-177).
"""
import enum
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import codec, engine

DEFAULT_BM25_K1 = 1.2
DEFAULT_BM25_B = 0.75


@dataclass(frozen=True)
class Term:
    field: str
    bytes: bytes

    @staticmethod
    def new(field, data):
        return Term(field, data if isinstance(data, (bytes, bytearray)) else str(data).encode())


class Query:
    pass


@dataclass
class TermQuery(Query):
    term: Term
    boost: float = 1.0
    ctx: Optional[object] = None

    @staticmethod
    def new(term, boost=1.0, ctx=None):
        return TermQuery(term, boost, ctx)


class IllegalArgument(ValueError):
    """error::ErrorKind::IllegalArgument"""


@dataclass(frozen=True)
class PointRangeQuery(Query):
    """A 1-D point range, bounds inclusive, as packed sortable bytes.  It scores 0f32 (PointRangeWeight's weight is
    only set by normalize(), which the searcher never calls), so on the device it is a docid filter."""
    field: str
    lower: bytes
    upper: bytes

    @property
    def bytes_per_dim(self):
        return len(self.lower)

    @staticmethod
    def new(field, lower_point, upper_point):
        if len(lower_point) != len(upper_point) or len(lower_point) not in (4, 8):
            raise IllegalArgument("1-D points of 4 or 8 bytes: lower and upper must have the same length")
        return PointRangeQuery(field, bytes(lower_point), bytes(upper_point))


def _sortable_int_bits(bits):   # NumericUtils::sortable_float_bits on the i32 view of an f32
    b = np.array([bits], np.uint32).view(np.int32)[0]
    return int(np.int32(b ^ ((b >> 31) & 0x7FFFFFFF)))


def _sortable_long_bits(bits):  # NumericUtils::sortable_double_bits on the i64 view of an f64
    b = np.array([bits], np.uint64).view(np.int64)[0]
    return int(np.int64(b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)))


class IntPoint:
    BYTES = 4

    @staticmethod
    def pack(value):
        """int_to_sortable_bytes: the sign bit flipped, big-endian"""
        return ((int(value) & 0xFFFFFFFF) ^ 0x80000000).to_bytes(4, "big")

    @classmethod
    def new_range_query(cls, field, lower, upper):
        return PointRangeQuery.new(field, cls.pack(lower), cls.pack(upper))

    @classmethod
    def new_exact_query(cls, field, value):
        return cls.new_range_query(field, value, value)


class LongPoint(IntPoint):
    BYTES = 8

    @staticmethod
    def pack(value):
        return ((int(value) & 0xFFFFFFFFFFFFFFFF) ^ 0x8000000000000000).to_bytes(8, "big")


class FloatPoint(IntPoint):
    @staticmethod
    def pack(value):
        """IntPoint::pack(sortable_float_bits(f.to_bits())): -0.0 < +0.0, NaNs beyond the infinities"""
        return IntPoint.pack(_sortable_int_bits(int(np.array([value], np.float32).view(np.uint32)[0])))

    @staticmethod
    def pack_bits(bits):
        """pack of the f32 with these raw bits (any NaN payload)"""
        return IntPoint.pack(_sortable_int_bits(int(bits) & 0xFFFFFFFF))


class DoublePoint(IntPoint):
    BYTES = 8

    @staticmethod
    def pack(value):
        return LongPoint.pack(_sortable_long_bits(int(np.array([value], np.float64).view(np.uint64)[0])))

    @staticmethod
    def pack_bits(bits):
        return LongPoint.pack(_sortable_long_bits(int(bits) & 0xFFFFFFFFFFFFFFFF))


@dataclass
class MatchAllDocsQuery(Query):
    """Every docid of every leaf, score 0f32 (the weight's default; normalisation is commented out in
    searcher.rs:709-722)."""


@dataclass
class ConstantScoreQuery(Query):
    """ConstantScoreQuery::with_boost(query, boost): the docs of `query` (evaluated without scores), score = boost."""
    query: Query
    boost: float = 0.0

    @staticmethod
    def with_boost(query, boost):
        return ConstantScoreQuery(query, float(boost))


@dataclass
class BooleanQuery(Query):
    must_queries: List[Query]
    should_queries: List[Query]
    filter_queries: List[Query]
    must_not_queries: List[Query]
    min_should_match: int

    @staticmethod
    def build(musts, shoulds, filters, must_nots, min_should_match=0):
        """boolean_query.rs:40-87 — note the collapse of a single positive clause."""
        musts, shoulds, filters, must_nots = list(musts), list(shoulds), list(filters), list(must_nots)
        msm = min_should_match if min_should_match > 0 else (1 if not musts else 0)
        if not (musts or shoulds or filters or must_nots):
            raise IllegalArgument("boolean query should at least contain one inner query!")
        if not must_nots and len(musts) + len(shoulds) + len(filters) == 1:
            if musts:
                return musts[0]
            if shoulds:
                return shoulds[0]
            return ConstantScoreQuery.with_boost(filters[0], 0.0)
        if not (musts or shoulds or filters):
            musts.append(MatchAllDocsQuery())  # only must_not exists (:76-79)
        return BooleanQuery(musts, shoulds, filters, must_nots, msm)


@dataclass
class DisjunctionMaxQuery(Query):
    disjuncts: List[Query]
    tie_breaker_multiplier: float

    @staticmethod
    def build(disjuncts, tie_breaker_multiplier):
        """search/query/disjunction_max_query.rs:51-68 — one disjunct is the disjunct itself."""
        disjuncts = list(disjuncts)
        if not disjuncts:
            raise IllegalArgument("DisjunctionMaxQuery: sub query should not be empty!")
        if len(disjuncts) == 1:
            return disjuncts[0]
        return DisjunctionMaxQuery(disjuncts, float(tie_breaker_multiplier))


@dataclass
class BM25Similarity:
    k1: float = DEFAULT_BM25_K1
    b: float = DEFAULT_BM25_B


@dataclass
class ScoreDoc:
    doc: int
    score: float

    def doc_id(self):
        return self.doc


@dataclass
class TopDocs:
    _total_hits: int
    _score_docs: List[ScoreDoc]

    def total_hits(self):
        return self._total_hits

    def score_docs(self):
        return self._score_docs


class RescoreMode(enum.IntEnum):
    """rescorer.rs:96-115 — how a matched hit's two scores combine (f32)."""
    Avg = engine.RESCORE_AVG
    Max = engine.RESCORE_MAX
    Min = engine.RESCORE_MIN
    Total = engine.RESCORE_TOTAL
    Multiply = engine.RESCORE_MULTIPLY


@dataclass
class RescoreRequest:
    """RescoreRequest::new (rescorer.rs:67-94); rescore_movedout is never read by the reference and is left out."""
    query: Query
    query_weight: float = 1.0
    rescore_weight: float = 1.0
    mode: RescoreMode = RescoreMode.Total
    window_size: int = 10


class QueryRescorer:
    """QueryRescorer::rescore (rescorer.rs:130-140) for score TopDocs: the first window_size hits are scored by
    request.query on the GPU (rg_rescore_hits), combined with their first-pass score and sorted again; the hits
    after the window are scaled by query_weight.  top_docs is edited in place."""

    def rescore(self, searcher, request: RescoreRequest, top_docs: TopDocs):
        docs = top_docs.score_docs()
        if top_docs.total_hits() == 0 or not docs:
            return
        q, c, ranges, groups = searcher._compile_any([request.query])
        hits = np.zeros((1, len(docs)), engine.HIT_DTYPE)
        hits[0]["doc"] = [d.doc for d in docs]
        hits[0]["score"] = np.array([d.score for d in docs], np.float32)
        out = searcher.engine.rescore_hits(q, c, hits, [len(docs)], [top_docs.total_hits()], request.window_size,
                                           request.query_weight, request.rescore_weight, int(request.mode),
                                           k1=searcher.similarity.k1, groups=groups, ranges=ranges)
        for i, h in enumerate(out[0]):
            docs[i].doc = int(h["doc"])
            docs[i].score = float(h["score"])


class TopDocsCollector:
    """TopDocsCollector::new(estimated_hits).  The GPU searcher fills it with the exact result
    the reference's collect()/add_doc()/top_docs() sequence would have produced."""

    def __init__(self, estimated_hits):
        if estimated_hits < 1:
            raise IllegalArgument("estimated_hits must be >= 1")
        self.estimated_hits = int(estimated_hits)
        self._top = TopDocs(0, [])

    @staticmethod
    def new(estimated_hits):
        return TopDocsCollector(estimated_hits)

    def needs_scores(self):
        return True

    def top_docs(self):
        return self._top


@dataclass
class IndexReader:
    """What StandardDirectoryReader exposes to the searcher: leaves in order plus a terms
    dictionary (host side; the FST/BlockTree seek itself is out of scope, SURVEY §8f-3)."""
    segments: Sequence[codec.Segment]
    term_ids: dict = field(default_factory=dict)   # (field, bytes) -> engine-wide term id
    field_name: str = "body"
    # 1-D point fields: name -> one entry per leaf, (docs int32 [n], packed uint8 [n, bytes_per_dim]) or None when the
    # leaf has no points of the field (what PointValues::intersect with an accept-all visitor yields)
    points: dict = field(default_factory=dict)

    def max_doc(self):
        return sum(s.max_doc for s in self.segments)

    def term_id(self, term: Term):
        if term.field != self.field_name:
            return None
        if self.term_ids:
            return self.term_ids.get((term.field, bytes(term.bytes)))
        try:  # synthetic indexes: the term text is its id
            return int(term.bytes)
        except ValueError:
            return None


class GpuIndexSearcher:
    """IndexSearcher<C> whose search() runs on the H100 (DefaultIndexSearcher::new(reader, None))."""

    def __init__(self, reader: IndexReader, similarity: Optional[BM25Similarity] = None,
                 device=-1, eng: Optional[engine.Engine] = None, range_postings=0,
                 cand_arena_bytes=0, flags=0, device_terms=False):
        """device_terms: upload every leaf's terms dictionary (rg_terms_upload) and resolve the Term bytes of a batch
        with one device lookup (rg_terms_lookup) instead of the host-side dict — what replaces the per-query
        SegmentTermIterator::seek_exact of the reference."""
        self.reader = reader
        self.device_terms = bool(device_terms)
        self._resolved = None
        self.similarity = similarity or BM25Similarity()
        self.engine = eng or engine.Engine(device=device, range_postings=range_postings,
                                           cand_arena_bytes=cand_arena_bytes, flags=flags)
        if not eng:
            for seg in reader.segments:
                self.engine.upload_segment(seg)
        # engine-wide point field ids: the fields in name order
        self._point_fields = {name: i for i, name in enumerate(sorted(reader.points))}
        if not eng:
            for name, fid in self._point_fields.items():
                for ord_, leaf in enumerate(reader.points[name]):
                    if leaf is not None:
                        docs, packed = leaf
                        packed = np.asarray(packed, np.uint8)
                        self.engine.upload_points(ord_, fid, packed.shape[1], docs, packed)
        self._ranges = None
        self._groups = None
        # with_similarity (searcher.rs:306-363): statistics of the largest-max_doc leaf
        # (stable sort descending -> first among equals), max_doc of the whole reader
        segs = list(reader.segments)
        self._stats_seg = max(range(len(segs)), key=lambda i: (segs[i].max_doc, -i))
        s = segs[self._stats_seg]
        self._max_doc = reader.max_doc()
        self._doc_count = s.doc_count
        self._sum_ttf = s.sum_total_term_freq
        self._avgdl = codec.bm25_avg_field_length(self._sum_ttf, self._doc_count, self._max_doc)
        self._cache = codec.bm25_norm_cache(self.similarity.k1, self.similarity.b, self._avgdl)
        self.engine.set_norm_cache(0, self._cache)
        if self.device_terms:
            if not reader.term_ids:
                raise IllegalArgument("device_terms needs IndexReader.term_ids (the dictionary)")
            entries = sorted((b, tid) for (f, b), tid in reader.term_ids.items() if f == reader.field_name)
            for ord_, seg in enumerate(segs):   # a leaf's dictionary holds the terms that occur in it
                mine = [(b, tid) for b, tid in entries if tid < len(seg.terms) and seg.terms["doc_freq"][tid] > 0]
                self.engine.upload_terms(ord_, [b for b, _ in mine], [tid for _, tid in mine])

    # TermQuery::create_weight -> BM25Similarity::compute_weight
    def term_weight(self, term_id, boost):
        s = self.reader.segments[self._stats_seg]
        df = int(s.terms["doc_freq"][term_id]) if term_id is not None and term_id < len(s.terms) else 0
        doc_count = self._max_doc if self._doc_count == -1 else self._doc_count
        idf = np.float32(codec.bm25_idf(df, doc_count))
        return np.float32(idf * np.float32(boost))

    def _compile(self, query, clauses):
        """-> (clause_begin, n_clauses, min_should_match, flags); appends to `clauses`.  A group's members (see
        _compile_one) follow the query's own clauses."""
        pending = []
        out = self._compile_one(query, clauses, pending)
        for gi, members in pending:
            begin = len(clauses)
            for q in members.should_queries:
                self._add_term(q, engine.SHOULD, clauses)
            self._groups[gi] = (begin, len(members.should_queries), members.min_should_match, engine.Q_BOOLEAN)
        return out

    def _add_term(self, q, occur, clauses):
        if not isinstance(q, TermQuery):
            raise engine.Unsupported(engine.RG_EUNSUPPORTED, "only TermQuery leaves are accelerated")
        if self._resolved is not None:   # ids and doc_freq came from the device dictionary
            tid, df = self._resolved.get((q.term.field, bytes(q.term.bytes)), (None, 0))
            doc_count = self._max_doc if self._doc_count == -1 else self._doc_count
            w = np.float32(np.float32(codec.bm25_idf(df, doc_count)) * np.float32(q.boost))
            clauses.append((occur, 0xFFFFFFFF if tid is None else tid, w, 0))
            return
        tid = self.reader.term_id(q.term)
        absent = tid is None
        clauses.append((occur, 0xFFFFFFFF if absent else tid, self.term_weight(None if absent else tid, q.boost), 0))

    def _compile_one(self, query, clauses, pending):
        begin = len(clauses)

        def add(q, occur):
            if isinstance(q, BooleanQuery) and self._groups is not None:
                # a nested BooleanQuery: a group (RG_CLAUSE_GROUP) when it is pure SHOULD over TermQuerys; its
                # members are written after the query's own clauses
                if q.must_queries or q.filter_queries or q.must_not_queries or \
                        not all(isinstance(m, TermQuery) for m in q.should_queries):
                    raise engine.Unsupported(engine.RG_EUNSUPPORTED, "only pure-SHOULD groups of TermQuerys are accelerated")
                clauses.append((occur | engine.CLAUSE_GROUP, len(self._groups), 0.0, 0))
                pending.append((len(self._groups), q))
                self._groups.append(None)
                return
            if isinstance(q, PointRangeQuery):
                if self._ranges is None:
                    raise engine.Unsupported(engine.RG_EUNSUPPORTED, "PointRangeQuery is not accelerated here")
                # a field no leaf has points of gets an id no leaf was uploaded with: no scorer anywhere
                fid = self._point_fields.get(q.field, 0xFFFFFFFF)
                r = np.zeros(1, engine.RANGE_DTYPE)[0]
                r["field"], r["bytes_per_dim"] = fid, q.bytes_per_dim
                r["lower"][:q.bytes_per_dim] = np.frombuffer(q.lower, np.uint8)
                r["upper"][:q.bytes_per_dim] = np.frombuffer(q.upper, np.uint8)
                clauses.append((occur | engine.CLAUSE_RANGE, len(self._ranges), 0.0, 0))
                self._ranges.append(r)
                return
            self._add_term(q, occur, clauses)

        if isinstance(query, (TermQuery, PointRangeQuery)):
            add(query, engine.SHOULD)
            return (begin, 1, 0, 0)
        if isinstance(query, ConstantScoreQuery):
            if query.boost != 0.0:
                raise engine.Unsupported(engine.RG_EUNSUPPORTED, "ConstantScoreQuery with a non-zero boost is not accelerated")
            add(query.query, engine.FILTER)   # the lone FILTER clause of BooleanQuery::build (:66-75)
            return (begin, 1, 0, engine.Q_BOOLEAN)
        if isinstance(query, BooleanQuery):
            musts = list(query.must_queries)
            if any(isinstance(q, MatchAllDocsQuery) for q in musts):
                # only as build() writes it: the single MUST of a query that has nothing but MUST_NOT clauses —
                # the engine reads "only MUST_NOT clauses" as exactly that
                if len(musts) != 1 or query.should_queries or query.filter_queries or not query.must_not_queries:
                    raise engine.Unsupported(engine.RG_EUNSUPPORTED, "MatchAllDocsQuery beside other positive clauses")
                musts = []
            for q in musts:
                add(q, engine.MUST)
            for q in query.filter_queries:
                add(q, engine.FILTER)
            for q in query.should_queries:
                add(q, engine.SHOULD)
            for q in query.must_not_queries:
                add(q, engine.MUST_NOT)
            return (begin, len(clauses) - begin, query.min_should_match, engine.Q_BOOLEAN)
        if isinstance(query, DisjunctionMaxQuery):
            for q in query.disjuncts:
                add(q, engine.SHOULD)
            tie_bits = int(np.array([query.tie_breaker_multiplier], np.float32).view(np.int32)[0])
            return (begin, len(clauses) - begin, tie_bits, engine.Q_DISMAX)
        raise engine.Unsupported(engine.RG_EUNSUPPORTED, "query type is not accelerated")

    def _resolve_on_device(self, queries):
        """One rg_terms_lookup for every Term of the batch -> {(field, bytes): (term id or None, df in the stats leaf)}"""
        terms = set()

        def walk(q):
            if isinstance(q, TermQuery):
                if q.term.field == self.reader.field_name:
                    terms.add(bytes(q.term.bytes))
            elif isinstance(q, ConstantScoreQuery):
                walk(q.query)
            elif isinstance(q, BooleanQuery):
                for sub in q.must_queries + q.should_queries + q.filter_queries + q.must_not_queries:
                    walk(sub)
            elif isinstance(q, DisjunctionMaxQuery):
                for sub in q.disjuncts:
                    walk(sub)
        for q in queries:
            walk(q)
        terms = sorted(terms)
        ids, df = self.engine.lookup_terms(terms)
        return {(self.reader.field_name, b): (None if ids[i] == 0xFFFFFFFF else int(ids[i]), int(df[self._stats_seg][i]))
                for i, b in enumerate(terms)}

    def compile_batch(self, queries):
        clauses, qs = [], []
        self._resolved = self._resolve_on_device(queries) if self.device_terms else None
        for q in queries:
            qs.append(self._compile(q, clauses))
        return (np.array(qs, dtype=engine.QUERY_DTYPE).reshape(-1),
                np.array(clauses, dtype=engine.CLAUSE_DTYPE).reshape(-1))

    def compile_batch_ranges(self, queries):
        """compile_batch for queries that may hold PointRangeQuerys: (queries, clauses, ranges) for the *_ranges calls"""
        self._ranges = []
        try:
            q, c = self.compile_batch(queries)
            return q, c, np.array(self._ranges, dtype=engine.RANGE_DTYPE).reshape(-1)
        finally:
            self._ranges = None

    def compile_batch_nested(self, queries):
        """compile_batch for queries with nested pure-SHOULD BooleanQuerys (and maybe PointRangeQuerys):
        (queries, clauses, ranges, groups) for the *_nested calls"""
        self._ranges, self._groups = [], []
        try:
            q, c = self.compile_batch(queries)
            return (q, c, np.array(self._ranges, dtype=engine.RANGE_DTYPE).reshape(-1),
                    np.array(self._groups, dtype=engine.QUERY_DTYPE).reshape(-1))
        finally:
            self._ranges = self._groups = None

    @staticmethod
    def _has_groups(queries):
        """a BooleanQuery below the top level (the lone FILTER of build() wraps its clause in a ConstantScoreQuery)"""
        def sub(q):
            if isinstance(q, ConstantScoreQuery):
                return isinstance(q.query, BooleanQuery)
            if isinstance(q, BooleanQuery):
                return any(isinstance(s, BooleanQuery)
                           for s in q.must_queries + q.should_queries + q.filter_queries + q.must_not_queries)
            if isinstance(q, DisjunctionMaxQuery):
                return any(isinstance(s, BooleanQuery) for s in q.disjuncts)
            return False
        return any(sub(q) for q in queries)

    @staticmethod
    def _has_ranges(queries):
        def walk(q):
            if isinstance(q, PointRangeQuery):
                return True
            if isinstance(q, ConstantScoreQuery):
                return walk(q.query)
            if isinstance(q, BooleanQuery):
                return any(walk(s) for s in q.must_queries + q.should_queries + q.filter_queries + q.must_not_queries)
            if isinstance(q, DisjunctionMaxQuery):
                return any(walk(s) for s in q.disjuncts)
            return False
        return any(walk(q) for q in queries)

    def _compile_any(self, queries):
        """(queries, clauses, ranges, groups) through the compile call the batch needs; ranges / groups None when
        the plain or the *_ranges calls take it"""
        if self._has_groups(queries):
            return self.compile_batch_nested(queries)
        if self._has_ranges(queries):
            return self.compile_batch_ranges(queries) + (None,)
        return self.compile_batch(queries) + (None, None)

    def search_batch(self, queries, k, mode=engine.MODE_SEARCH, rescore=None):
        """rescore: (rescoring queries, RescoreRequest) — one rescoring query per query, the request's weights,
        mode and window for all: QueryRescorer::rescore on every row on the device before the rows are fetched."""
        q, c, ranges, groups = self._compile_any(queries)
        if rescore is None:
            if groups is not None:
                return self.engine.search_batch_nested(q, c, groups, k, k1=self.similarity.k1, mode=mode,
                                                       ranges=ranges)
            if ranges is not None:
                return self.engine.search_batch_ranges(q, c, ranges, k, k1=self.similarity.k1, mode=mode)
            return self.engine.search_batch(q, c, k, k1=self.similarity.k1, mode=mode)
        rescore_queries, req = rescore
        rq, rc, rranges, rgroups = self._compile_any(rescore_queries)   # their own range / group arrays
        batch = self.engine.prepare(q, c, k, k1=self.similarity.k1, mode=mode, ranges=ranges, groups=groups)
        try:
            batch.run()
            self.engine.rescore_batch(batch, rq, rc, req.window_size, req.query_weight, req.rescore_weight,
                                      int(req.mode), k1=self.similarity.k1, groups=rgroups, ranges=rranges)
            return batch.fetch()
        finally:
            batch.close()

    def search(self, query, collector: TopDocsCollector):
        """IndexSearcher::search(&query, &mut collector)."""
        hits, counts, total = self.search_batch([query], collector.estimated_hits)
        n = int(counts[0])
        collector._top = TopDocs(int(total[0]), [ScoreDoc(int(h["doc"]), float(h["score"])) for h in hits[0][:n]])

    def search_parallel(self, query, collector: TopDocsCollector):
        hits, counts, total = self.search_batch([query], collector.estimated_hits,
                                                mode=engine.MODE_SEARCH_PARALLEL)
        n = int(counts[0])
        collector._top = TopDocs(int(total[0]), [ScoreDoc(int(h["doc"]), float(h["score"])) for h in hits[0][:n]])
