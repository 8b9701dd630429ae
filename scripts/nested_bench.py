#!/usr/bin/env python
"""Nested BooleanQuerys on the device: config 3's index (10 M docs, 100 K terms, one leaf).  Prints one JSON line.

Workloads (1024 queries each, k = 10; the terms of a query are distinct, drawn as bench.py draws config 4's):
  (a) `+(a|b) +(c|d)`: two required groups (the cheaper group leads);
  (b) `+a +(b|c) -d`: a term and a required group, with a MUST_NOT term;
  (c) `+(a|b) c`: a required group and an optional term (ReqOpt).
Per workload: the median of rg_engine_last_kernel_ms("eval") and of "run" over the timed steps, queries/s from the run
median, end-to-end queries/s of GpuIndexSearcher.search_batch (compile, plan, run, fetch) on the same batch, the
group-lead counters of the last run, the oracle's queries/s on a sample (all usable host cores, one query per thread)
and a bit-for-bit parity verdict of the device against the oracle on that sample.

usage: scripts/nested_bench.py [--steps N] [--warmup W] [--sample S]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (config 3's index and the query term sampler)
import nested_oracle as no  # noqa: E402
import oracle_binding as ob  # noqa: E402
from rucene_b200 import codec, engine, search  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = float(subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                  capture_output=True, text=True, timeout=30).stdout.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        pl = None
    return name, pl


def to_oracle(q, c, g):
    """the engine arrays of a compiled batch as the oracle's (every term boost 1: the weights are idf * 1)"""
    def qs(a):
        o = np.zeros(len(a), ob.QUERY_DTYPE)
        o["clause_begin"], o["n_clauses"], o["min_should_match"] = a["clause_begin"], a["n_clauses"], a["min_should_match"]
        o["is_boolean"] = a["flags"] & engine.Q_BOOLEAN
        return o
    oc = np.zeros(len(c), ob.CLAUSE_DTYPE)
    oc["occur"], oc["term_id"], oc["boost"] = c["occur"], c["term_id"], 1.0
    return qs(q), oc, qs(g)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=256)
    a = ap.parse_args()
    w = bench.WORKLOADS["c3"]
    t0 = time.perf_counter()
    seg = codec.synth_segment(w["seed_index"], w["docs"], w["terms"], doc_version=1)
    s = search.GpuIndexSearcher(search.IndexReader([seg]), device=0)
    ix = no.NestedIndex([seg])
    setup_s = time.perf_counter() - t0

    terms = [t for _, t in bench.gen_queries("c4", w["terms"], w["batch"], w["seed_queries"])]
    T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
    B = search.BooleanQuery.build
    G = lambda *ts: B([], [T(t) for t in ts], [], [])
    workloads = {
        "a_group_and_group": [B([G(t[0], t[1]), G(t[2], t[3])], [], [], []) for t in terms],
        "b_term_group_not": [B([T(t[0]), G(t[1], t[2])], [], [], [T(t[3])]) for t in terms],
        "c_group_opt_term": [B([G(t[0], t[1])], [T(t[2])], [], []) for t in terms],
    }
    n_threads = len(os.sched_getaffinity(0))
    out = {}
    for name, queries in workloads.items():
        q, c, r, g = s.compile_batch_nested(queries)
        batch = s.engine.prepare(q, c, 10, k1=s.similarity.k1, groups=g)
        try:
            for _ in range(a.warmup):
                batch.run()
                batch.fetch()
            ev, run = [], []
            for _ in range(a.steps):
                batch.run()
                hits, counts, total = batch.fetch()
                ev.append(s.engine.last_kernel_ms("eval"))
                run.append(s.engine.last_kernel_ms("run"))
            stats = batch.group_stats()
        finally:
            batch.close()
        e2e = []
        for _ in range(max(1, a.steps // 4)):
            t1 = time.perf_counter()
            eh, ecnt, etot = s.search_batch(queries, 10)
            e2e.append(time.perf_counter() - t1)
        idx = np.random.default_rng(7).choice(len(queries), min(a.sample, len(queries)), replace=False)
        sq, sc, _, sg = s.compile_batch_nested([queries[i] for i in idx])
        t1 = time.perf_counter()
        wh, wcnt, wt = ix.search_batch(*to_oracle(sq, sc, sg), 10, n_threads=n_threads)
        oracle_s = time.perf_counter() - t1
        same = bool(np.array_equal(wt, total[idx]) and np.array_equal(wcnt, counts[idx]) and all(
            np.array_equal(hits[i][:n].view(np.uint64), wh[j][:n].view(np.uint64))
            for j, (i, n) in enumerate(zip(idx, wcnt))) and np.array_equal(eh.view(np.uint64), hits.view(np.uint64)))
        run_ms = float(np.median(run))
        out[name] = {"eval_ms_median": float(np.median(ev)), "run_ms_median": run_ms,
                     "queries_per_s": len(q) / (run_ms / 1e3),
                     "e2e_queries_per_s": len(q) / float(np.median(e2e)), "group_stats": stats,
                     "oracle_queries_per_s": len(idx) / oracle_s,
                     "parity_on_sample": "identical TopDocs" if same else "MISMATCH", "sample": int(len(idx))}
    name, power = card()
    print(json.dumps({"metric": "nested_bench", "device": {"name": name, "power_limit_w": power},
                      "index": {"docs": w["docs"], "terms": w["terms"], "setup_s": round(setup_s, 1)},
                      "batch": w["batch"], "k": 10, "steps": a.steps, "warmup": a.warmup,
                      "oracle_threads": n_threads, "workloads": out}))


if __name__ == "__main__":
    main()
