"""Rescoring on config 4: the first pass of bench.py's flagship workload (4096 x 5-term SHOULD, k = 100), then
QueryRescorer on the device (rg_batch_rescore) with two request kinds:
  (a) the query's 5 terms as an all-MUST conjunction, mode Total;
  (b) a ReqOpt of the query's rarest term (MUST) plus the other four (SHOULD), mode Multiply.
Window 100.  Prints one JSON line: k_rescore time (CUDA events, median of the timed steps), its share of a
run + rescore step, probes (window targets x clauses in the leaf) and blocks decoded on a sample, the oracle's
rescorer (orc_rescore, tests/cpp/orc_rescore.cpp) over the same windows on the usable host cores in queries/s, and
whether every rescored row equals orc_rescore's bit for bit."""
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

import bench  # noqa: E402  (its main is guarded: only the helpers are used)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=bench.WORKLOADS["c4"]["docs"])
    ap.add_argument("--terms", type=int, default=bench.WORKLOADS["c4"]["terms"])
    ap.add_argument("--batch", type=int, default=bench.WORKLOADS["c4"]["batch"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=16)
    args = ap.parse_args()
    import torch
    import helpers
    import oracle_binding as ob
    import rescore_model as rm
    import rescore_oracle as ro
    from rucene_b200 import codec, engine

    w = bench.WORKLOADS["c4"]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    seg = codec.synth_segment(w["seed_index"], args.docs, args.terms, doc_version=1)
    eng = engine.Engine(device=0)
    eng.upload_segment(seg, doc_base=0)
    df0 = seg.terms["doc_freq"]
    avgdl = codec.bm25_avg_field_length(seg.sum_total_term_freq, seg.doc_count, args.docs)
    cache = codec.bm25_norm_cache(1.2, 0.75, avgdl)
    eng.set_norm_cache(0, cache)

    def weight_of(t):
        return np.float32(codec.bm25_idf(int(df0[t]), seg.doc_count))

    qs = bench.gen_queries("c4", args.terms, args.batch, w["seed_queries"])
    q, c = bench.build_query_arrays(qs, weight_of, engine)
    k = w["k"]
    # rescoring queries, in the engine's format
    kinds = {}
    for kind in ("a", "b"):
        rq = np.zeros(len(qs), engine.QUERY_DTYPE)
        rc = np.zeros(5 * len(qs), engine.CLAUSE_DTYPE)
        for i, (_, terms) in enumerate(qs):
            ts = list(terms)
            if kind == "b":
                rare = min(ts, key=lambda t: int(df0[t]))
                ts = [rare] + [t for t in ts if t != rare]
            for j, t in enumerate(ts):
                rc[5 * i + j] = (engine.MUST if kind == "a" or j == 0 else engine.SHOULD, t, weight_of(t), 0)
            rq[i] = (5 * i, 5, 0, engine.Q_BOOLEAN)
        kinds[kind] = (rq, rc, engine.RESCORE_TOTAL if kind == "a" else engine.RESCORE_MULTIPLY)

    batch = eng.prepare(q, c, k, k1=1.2)
    batch.run()
    first = batch.fetch()
    out = {"gpu": gpu, "docs": args.docs, "terms": args.terms, "batch": args.batch, "k": k, "window": 100,
           "timed_steps": args.steps}
    ix = helpers.oracle_index([seg])
    model = rm.Model(ix, [seg], cache, 1.2)  # postings for the probe / block counts
    oracle = ro.RescoreIndex([seg])
    cores = bench.usable_cores()
    sample = np.random.default_rng(5).choice(len(qs), min(args.sample, len(qs)), replace=False)
    for kind, (rq, rc, mode) in kinds.items():
        res, step = [], []
        for i in range(args.warmup + args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batch.run()
            eng.rescore_batch(batch, rq, rc, 100, 1.0, 1.0, mode, k1=1.2)
            got = batch.fetch()
            t1 = time.perf_counter()
            if i >= args.warmup:
                res.append(eng.last_kernel_ms("rescore"))
                step.append((t1 - t0) * 1e3)
        # every row against orc_rescore over the same first-pass rows, timed on the usable host cores
        oq = np.zeros(len(qs), ob.QUERY_DTYPE)
        oq["clause_begin"], oq["n_clauses"], oq["min_should_match"] = rq["clause_begin"], rq["n_clauses"], 0
        oq["is_boolean"] = 1
        oc = np.zeros(len(rc), ob.CLAUSE_DTYPE)
        oc["occur"], oc["term_id"], oc["boost"] = rc["occur"], rc["term_id"], 1.0
        t0 = time.perf_counter()
        want = oracle.rescore(oq, oc, first[0], first[1], first[2], 100, 1.0, 1.0, mode, n_threads=cores)
        cpu_s = time.perf_counter() - t0
        ok = bool(np.array_equal(want.view(np.uint64), got[0].view(np.uint64)))
        # what the probes touch, on the sample
        probes = blocks = 0
        for i in sample:
            targets = np.sort(first[0][i][:min(int(first[1][i]), 100)]["doc"])
            for t in rc[5 * i:5 * i + 5]["term_id"]:
                p = model.postings(0, int(t))
                if p is None:
                    continue
                docs = p[0]
                pos = np.searchsorted(docs, targets)
                probes += len(targets)
                blocks += len(np.unique(pos[pos < len(docs)] // 128))
        out[kind] = {"mode": "Total" if kind == "a" else "Multiply",
                     "k_rescore_ms_median": float(np.median(res)), "k_rescore_ms_min": float(np.min(res)),
                     "step_ms_median": float(np.median(step)),
                     "rescore_share_of_step": float(np.median(res) / np.median(step)),
                     "probes_per_query_sample": probes / len(sample), "blocks_per_query_sample": blocks / len(sample),
                     "sample_queries": int(len(sample)), "rows_equal_orc_rescore": ok,
                     "orc_rescore_queries_per_s": len(qs) / cpu_s, "orc_rescore_host_cores": cores,
                     "gpu_over_cpu": (len(qs) / (np.median(res) * 1e-3)) / (len(qs) / cpu_s)}
    out["first_pass_run_ms"] = eng.last_kernel_ms("run")
    batch.close()
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
