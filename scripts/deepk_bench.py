#!/usr/bin/env python
"""Deep top-k on the device: config 4's index and batch (100 M docs, 1 M terms, one leaf, 4096 5-term SHOULD queries)
and config 3's (10 M docs, 100 K terms, 1024 2-term MUST queries), each at k = 1000, 2048, 4096 and 16384.  Prints one
JSON line.

Per (config, k): the median of rg_engine_last_kernel_ms "eval" and "replay" over the timed steps, summed over the
sub-batches a step needs (a batch whose candidates do not fit the arena is cut in halves until they do), candidates
per query (rg_batch_stats slot 3), whether the per-item score histograms that carry theta along a heap chain were kept
(they are dropped when n_items * 1 KB exceeds 2 GiB), end-to-end queries/s (prepare excluded, run + fetch included)
and a bit-for-bit parity verdict against the oracle on a sample of queries.  The card's name and power limit are read
in the same run.

usage: scripts/deepk_bench.py [--steps N] [--warmup W] [--sample S] [--configs c4,c3] [--ks 1000,2048,4096,16384]
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

import bench  # noqa: E402  (the configs' index and query generators)
import helpers  # noqa: E402
import oracle_binding as ob  # noqa: E402
from rucene_b200 import codec, engine, search  # noqa: E402


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


def chunks(n, parts):
    return [np.arange(n * i // parts, n * (i + 1) // parts) for i in range(parts)]


def sub_batch(q, c, idx):
    """queries idx of (q, c) as a self-contained batch (clauses renumbered)"""
    qs, cs = np.zeros(len(idx), q.dtype), []
    for j, i in enumerate(idx):
        b, n = int(q[i]["clause_begin"]), int(q[i]["n_clauses"])
        qs[j] = q[i]
        qs[j]["clause_begin"] = sum(len(x) for x in cs)
        cs.append(c[b:b + n])
    return qs, np.concatenate(cs)


def run_k(s, q, c, k, steps, warmup):
    """One leg: the batch at depth k, cut into as few sub-batches as the candidate arena allows."""
    parts = 1
    while True:
        subs = [sub_batch(q, c, idx) for idx in chunks(len(q), parts)]
        batches = []
        try:
            for sq, sc in subs:
                batches.append(s.engine.prepare(sq, sc, k, k1=s.similarity.k1))
            ev, rp, e2e = [], [], []
            for step in range(warmup + steps):
                e_ms = r_ms = 0.0
                t0 = time.perf_counter()
                outs = []
                for b in batches:
                    b.run()
                    outs.append(b.fetch())
                    e_ms += s.engine.last_kernel_ms("eval")
                    r_ms += s.engine.last_kernel_ms("replay")
                dt = time.perf_counter() - t0
                if step >= warmup:
                    ev.append(e_ms)
                    rp.append(r_ms)
                    e2e.append(dt)
            st = [b.stats() for b in batches]
            break
        except engine.EngineError as e:
            if e.code != engine.RG_ENOMEM or parts >= len(q):
                raise
            parts *= 2
        finally:
            for b in batches:
                b.close()
    hits = np.concatenate([o[0] for o in outs])
    counts = np.concatenate([o[1] for o in outs])
    total = np.concatenate([o[2] for o in outs])
    cand = sum(x["candidate_slots"] for x in st)
    return {"sub_batches": parts, "eval_ms_median": float(np.median(ev)), "replay_ms_median": float(np.median(rp)),
            "candidates_per_query": cand / len(q), "histograms_kept": all(x["items"] * 1024 <= (2 << 30) for x in st),
            "items": sum(x["items"] for x in st), "queries_per_s": len(q) / float(np.median(e2e))}, (hits, counts, total)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=16)
    ap.add_argument("--configs", default="c4,c3")
    ap.add_argument("--ks", default="1000,2048,4096,16384")
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",")]
    out = {}
    for cfg in a.configs.split(","):
        w = bench.WORKLOADS[cfg]
        t0 = time.perf_counter()
        seg = codec.synth_segment(w["seed_index"], w["docs"], w["terms"], doc_version=1)
        s = search.GpuIndexSearcher(search.IndexReader([seg]), device=0)
        ix = helpers.oracle_index([seg])
        setup_s = time.perf_counter() - t0
        T = lambda t: search.TermQuery.new(search.Term.new("body", str(t)))
        qs = bench.gen_queries(cfg, w["terms"], w["batch"], w["seed_queries"])
        B = search.BooleanQuery.build
        queries = [B([T(x) for x in tt], [], [], []) if occ == "must" else B([], [T(x) for x in tt], [], [])
                   for occ, tt in qs]
        q, c = s.compile_batch(queries)
        occ = ob.MUST if qs[0][0] == "must" else ob.SHOULD
        idx = np.random.default_rng(7).choice(len(qs), min(a.sample, len(qs)), replace=False)
        oq, oc = ob.make_queries([("bool", [(occ, int(t)) for t in qs[i][1]], 0) for i in idx])
        legs = {}
        for k in ks:
            leg, (hits, counts, total) = run_k(s, q, c, k, a.steps, a.warmup)
            wh, wc, wt = ix.search_batch(oq, oc, k, n_threads=len(os.sched_getaffinity(0)))
            try:
                helpers.assert_same_topdocs((hits[idx], counts[idx], total[idx]), (wh, wc, wt), "deepk")
                leg["parity_on_sample"] = "identical TopDocs"
            except AssertionError as e:
                leg["parity_on_sample"] = "MISMATCH %s" % (e,)
            leg["sample"] = int(len(idx))
            legs[str(k)] = leg
            print(cfg, k, json.dumps(leg), file=sys.stderr, flush=True)
        s.engine.close()
        del ix
        out[cfg] = {"docs": w["docs"], "terms": w["terms"], "batch": w["batch"], "setup_s": round(setup_s, 1),
                    "what": w["what"], "k": legs}
    name, power = card()
    print(json.dumps({"metric": "deepk_bench", "device": {"name": name, "power_limit_w": power},
                      "steps": a.steps, "warmup": a.warmup, "configs": out}))


if __name__ == "__main__":
    main()
