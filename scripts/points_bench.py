#!/usr/bin/env python
"""PointRangeQuery filters on the device: config 3's index (10 M docs, 100 K terms, one leaf) plus two LongPoint fields,
a timestamp that rises with docid (with noise) and a uniform random value.  Prints one JSON line.

Workloads (1024 queries each, k = 10):
  (a) config 3's 2-term MUST, without a filter and with a FILTER range of ~1 %, 10 % and 50 % on each field;
  (b) `#range t1 t2`: a FILTER range (10 %) beside two SHOULD terms (ReqOpt with a range lead, cut into docid ranges);
  (c) bare ranges (1 % of the docs each, at seeded positions).
Per workload: the median of rg_engine_last_kernel_ms("eval") and of "run" over the timed steps, queries/s from the
run median, the range-lead block counters of the last run, the oracle's queries/s on a sample (one query per host
core) and a bit-for-bit parity verdict of the device against the oracle on that sample.

usage: scripts/points_bench.py [--steps N] [--warmup W] [--sample S]
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

import bench  # noqa: E402  (config 3's index and query generator)
import oracle_binding as ob  # noqa: E402
import points_oracle as po  # noqa: E402
from rucene_b200 import codec, engine, search  # noqa: E402

TS, UNI = "timestamp", "uniform"


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
        pl = float(pl)
    except (OSError, ValueError, subprocess.SubprocessError):
        pl = None
    return name, pl


def to_oracle(q, c):
    oq = np.zeros(len(q), ob.QUERY_DTYPE)
    oq["clause_begin"], oq["n_clauses"], oq["min_should_match"] = q["clause_begin"], q["n_clauses"], q["min_should_match"]
    oq["is_boolean"] = q["flags"] & engine.Q_BOOLEAN
    oc = np.zeros(len(c), ob.CLAUSE_DTYPE)
    oc["occur"], oc["term_id"] = c["occur"], c["term_id"]
    oc["boost"] = np.where(c["occur"] & engine.CLAUSE_RANGE, 0.0, 1.0)
    return oq, oc


def sub_batch(q, c, idx):
    """queries idx of (q, c) as a self-contained batch (clauses renumbered)"""
    qs, cs = np.zeros(len(idx), q.dtype), []
    for j, i in enumerate(idx):
        b, n = int(q[i]["clause_begin"]), int(q[i]["n_clauses"])
        qs[j] = q[i]
        qs[j]["clause_begin"] = sum(len(x) for x in cs)
        cs.append(c[b:b + n])
    return qs, np.concatenate(cs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=128)
    a = ap.parse_args()
    w = bench.WORKLOADS["c3"]
    max_doc = w["docs"]
    t0 = time.perf_counter()
    seg = codec.synth_segment(w["seed_index"], max_doc, w["terms"], doc_version=1)
    rng = np.random.default_rng(0x5EED00F0)
    docs = np.arange(max_doc, dtype=np.int32)
    ts = docs.astype(np.int64) * 1000 + rng.integers(-5000, 5000, max_doc)
    uni = rng.integers(0, 1 << 40, max_doc)
    pack = lambda v: (np.asarray(v, np.int64).view(np.uint64) ^ np.uint64(1 << 63)).astype(">u8").view(np.uint8).reshape(-1, 8)
    packed = {TS: pack(ts), UNI: pack(uni)}
    reader = search.IndexReader([seg], points={TS: [(docs, packed[TS])], UNI: [(docs, packed[UNI])]})
    s = search.GpuIndexSearcher(reader, device=0)
    ix = po.PointsIndex([seg])
    for fid, name in enumerate(sorted(packed)):
        ix.add_points(0, fid, 8, docs, packed[name])
    setup_s = time.perf_counter() - t0

    terms = bench.gen_queries("c3", w["terms"], w["batch"], w["seed_queries"])
    T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
    qrng = np.random.default_rng(0x5EED00F1)
    sorted_vals = {TS: np.sort(ts), UNI: np.sort(uni)}

    def rand_range(field, frac):
        v = sorted_vals[field]
        lo = int(qrng.integers(0, int(len(v) * (1 - frac))))
        return search.LongPoint.new_range_query(field, int(v[lo]), int(v[lo + int(len(v) * frac) - 1]))

    B = search.BooleanQuery.build
    workloads = {"a_no_filter": [B([T(x) for x in tt], [], [], []) for _, tt in terms]}
    for field in (TS, UNI):
        for frac in (0.01, 0.1, 0.5):
            workloads["a_%s_%g" % (field, frac)] = [B([T(x) for x in tt], [], [rand_range(field, frac)], [])
                                                     for _, tt in terms]
    workloads["b_range_t1_t2"] = [B([], [T(x) for x in tt], [rand_range(TS, 0.1)], []) for _, tt in terms]
    workloads["c_bare_range"] = [rand_range(TS, 0.01) for _ in terms]
    n_threads = len(os.sched_getaffinity(0))
    out = {}
    for name, queries in workloads.items():
        q, c, r = s.compile_batch_ranges(queries)
        batch = s.engine.prepare(q, c, 10, k1=s.similarity.k1, ranges=r)
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
            blocks = batch.range_stats()
        finally:
            batch.close()
        idx = np.random.default_rng(7).choice(len(q), min(a.sample, len(q)), replace=False)
        sq, sc = sub_batch(q, c, idx)
        oq, oc = to_oracle(sq, sc)
        t1 = time.perf_counter()
        wh, wcnt, wt = ix.search_batch(oq, oc, r, 10, n_threads=n_threads)
        oracle_s = time.perf_counter() - t1
        same = bool(np.array_equal(wt, total[idx]) and np.array_equal(wcnt, counts[idx]) and all(
            np.array_equal(hits[i][:n].view(np.uint64), wh[j][:n].view(np.uint64))
            for j, (i, n) in enumerate(zip(idx, wcnt))))
        run_ms = float(np.median(run))
        out[name] = {"eval_ms_median": float(np.median(ev)), "run_ms_median": run_ms,
                     "queries_per_s": len(q) / (run_ms / 1e3), "blocks": blocks,
                     "oracle_queries_per_s": len(idx) / oracle_s, "parity_on_sample": "identical TopDocs" if same
                     else "MISMATCH", "sample": int(len(idx))}
    name, power = card()
    print(json.dumps({"metric": "points_bench", "device": {"name": name, "power_limit_w": power},
                      "index": {"docs": max_doc, "terms": w["terms"], "point_fields": sorted(packed),
                                "setup_s": round(setup_s, 1)},
                      "batch": w["batch"], "k": 10, "steps": a.steps, "warmup": a.warmup,
                      "oracle_threads": n_threads, "workloads": out}))


if __name__ == "__main__":
    main()
