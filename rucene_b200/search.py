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

Everything that touches postings runs on the GPU through the C ABI (engine.py); this module only
does what Query::create_weight does on the host once per query: collection/term statistics from
the largest segment (searcher.rs:311-351,732-767) and the BM25 weight (bm25_similarity.rs:151-177).
"""
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
        """-> (clause_begin, n_clauses, min_should_match, flags); appends to `clauses`."""
        begin = len(clauses)

        def add(q, occur):
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
            clauses.append((occur, 0xFFFFFFFF if absent else tid,
                            self.term_weight(None if absent else tid, q.boost), 0))

        if isinstance(query, TermQuery):
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

    def search_batch(self, queries, k, mode=engine.MODE_SEARCH):
        q, c = self.compile_batch(queries)
        return self.engine.search_batch(q, c, k, k1=self.similarity.k1, mode=mode)

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
