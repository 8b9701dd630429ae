#!/usr/bin/env python
"""Rescoring with nested groups and point ranges on the device (rg_batch_rescore_nested, k_rescore<true>): config 3's
index (10 M docs, 100 K terms, one leaf) plus points_bench.py's timestamp LongPoint field.  The first pass is 1024
5-term SHOULD queries at k = 100; each row's first 100 hits are rescored by one of three workloads:
  (a) `+(t0|t1) +(t2|t3)`, mode Total (a query-string builder's synonym groups);
  (b) `+t_rarest (t1|t2) #timestamp:[the most recent 10 %]`, mode Multiply (a recency filter beside an optional group);
  (c) `+t0 -(t3|t4)`, mode Total (an excluded group).
Prints one JSON line: per workload the median rg_engine_last_kernel_ms("rescore") over the timed steps, its share of
a run + rescore + fetch step, the oracle's rescorer (tests/cpp/orc_rescore_nested.cpp) over the same rows on the
usable host cores in queries/s, and whether every rescored row equals the oracle's bit for bit; plus the card's name
and power limit.

usage: scripts/rescore_nested_bench.py [--steps N] [--warmup W]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (config 3's index and the query generator)
import oracle_binding as ob  # noqa: E402
import rescore_nested_oracle as rno  # noqa: E402
from points_bench import card  # noqa: E402
from rucene_b200 import codec, engine, search  # noqa: E402

TS = "timestamp"


def to_oracle(q, c, g):
    def queries(x):
        o = np.zeros(len(x), ob.QUERY_DTYPE)
        o["clause_begin"], o["n_clauses"], o["min_should_match"] = x["clause_begin"], x["n_clauses"], x["min_should_match"]
        o["is_boolean"] = (x["flags"] & engine.Q_BOOLEAN) != 0
        return o
    oc = np.zeros(len(c), ob.CLAUSE_DTYPE)
    oc["occur"], oc["term_id"] = c["occur"], c["term_id"]
    oc["boost"] = np.where(c["occur"] & engine.CLAUSE_RANGE, 0.0, 1.0)
    return queries(q), oc, queries(np.zeros(0, engine.QUERY_DTYPE) if g is None else g)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    w = bench.WORKLOADS["c3"]
    max_doc, n_terms = w["docs"], w["terms"]
    t0 = time.perf_counter()
    seg = codec.synth_segment(w["seed_index"], max_doc, n_terms, doc_version=1)
    rng = np.random.default_rng(0x5EED00F0)   # points_bench.py's timestamp field
    docs = np.arange(max_doc, dtype=np.int32)
    ts = docs.astype(np.int64) * 1000 + rng.integers(-5000, 5000, max_doc)
    packed = (ts.view(np.uint64) ^ np.uint64(1 << 63)).astype(">u8").view(np.uint8).reshape(-1, 8)
    s = search.GpuIndexSearcher(search.IndexReader([seg], points={TS: [(docs, packed)]}), device=0)
    ox = rno.RescoreNestedIndex([seg])
    ox.add_points(0, 0, 8, docs, packed)
    setup_s = time.perf_counter() - t0

    qs = bench.gen_queries("c4", n_terms, 1024, w["seed_queries"])
    df = seg.terms["doc_freq"]
    T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
    B = search.BooleanQuery.build
    G = lambda *ts_: B([], [T(t) for t in ts_], [], [])
    v = np.sort(ts)
    recent = search.LongPoint.new_range_query(TS, int(v[int(len(v) * 0.9)]), int(v[-1]))
    first = [B([], [T(t) for t in tt], [], []) for _, tt in qs]
    work = {"a_groups_total": ([B([G(tt[0], tt[1]), G(tt[2], tt[3])], [], [], []) for _, tt in qs],
                               engine.RESCORE_TOTAL)}
    b_queries = []
    for _, tt in qs:
        rare = min(tt, key=lambda t: int(df[t]))
        rest = [t for t in tt if t != rare]
        b_queries.append(B([T(rare)], [G(rest[0], rest[1])], [recent], []))
    work["b_recency_multiply"] = (b_queries, engine.RESCORE_MULTIPLY)
    work["c_excluded_group_total"] = ([B([T(tt[0])], [], [], [G(tt[3], tt[4])]) for _, tt in qs], engine.RESCORE_TOTAL)

    q, c, r, g = s._compile_any(first)
    batch = s.engine.prepare(q, c, 100, k1=s.similarity.k1, ranges=r, groups=g)
    cores = len(os.sched_getaffinity(0))
    out = {}
    try:
        batch.run()
        rows = batch.fetch()
        for name, (queries, mode) in work.items():
            rq, rc, rr, rg = s._compile_any(queries)
            res, step = [], []
            for i in range(a.warmup + a.steps):
                t1 = time.perf_counter()
                batch.run()
                s.engine.rescore_batch(batch, rq, rc, 100, 1.0, 1.0, mode, k1=s.similarity.k1, groups=rg, ranges=rr)
                got = batch.fetch()   # waits for the rescored rows
                t2 = time.perf_counter()
                if i >= a.warmup:
                    res.append(s.engine.last_kernel_ms("rescore"))
                    step.append((t2 - t1) * 1e3)
            oq, oc, og = to_oracle(rq, rc, rg)
            t1 = time.perf_counter()
            want = ox.rescore(oq, oc, og, rows[0], rows[1], rows[2], 100, 1.0, 1.0, mode, ranges=rr, n_threads=cores)
            cpu_s = time.perf_counter() - t1
            same = bool(np.array_equal(want.view(np.uint64), got[0].view(np.uint64)) and
                        np.array_equal(got[1], rows[1]) and np.array_equal(got[2], rows[2]))
            med = float(np.median(res))
            out[name] = {"k_rescore_ms_median": med, "k_rescore_ms_min": float(np.min(res)),
                         "step_ms_median": float(np.median(step)),
                         "rescore_share_of_step": med / float(np.median(step)),
                         "oracle_rescore_queries_per_s": len(qs) / cpu_s,
                         "parity": "identical" if same else "MISMATCH", "sample_queries": len(qs)}
    finally:
        batch.close()
        s.engine.close()
    name, power = card()
    print(json.dumps({"metric": "rescore_nested_bench", "device": {"name": name, "power_limit_w": power},
                      "index": {"docs": max_doc, "terms": n_terms, "point_fields": [TS], "setup_s": round(setup_s, 1)},
                      "first_pass": {"queries": len(qs), "clauses": "5 SHOULD", "k": 100}, "window": 100,
                      "steps": a.steps, "warmup": a.warmup, "oracle_threads": cores, "workloads": out}))


if __name__ == "__main__":
    main()
