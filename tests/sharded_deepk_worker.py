"""torchrun worker for test_gpu_deepk.py: sharded search at k = 4096 — one leaf per rank, every rank on cuda:0, the
leaf records (16 + 8 k bytes per query) all-gathered over gloo and merged on the device; rank 0 compares with the
oracle's leaf-ordered search_parallel."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import helpers  # noqa: E402
import oracle_binding as ob  # noqa: E402
from rucene_b200 import codec, engine, sharded  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
    max_doc, n_terms, k = 150000, 3000, 4096
    segs = [codec.synth_segment(0x5EED0D00 + r, max_doc, n_terms, doc_version=1) for r in range(world)]
    local = segs[rank]
    eng = engine.Engine(device=0, range_postings=20000)
    eng.upload_segment(local, doc_base=rank * max_doc)
    df0, doc_count, sum_ttf = sharded.broadcast_stats(local.terms["doc_freq"], local.doc_count,
                                                      local.sum_total_term_freq, src=0, device=None)
    avgdl = codec.bm25_avg_field_length(sum_ttf, doc_count, max_doc * world)
    eng.set_norm_cache(0, codec.bm25_norm_cache(1.2, 0.75, avgdl))
    rng = np.random.default_rng(0x5EED0D00)
    specs = [("bool", [(ob.SHOULD, 0), (ob.SHOULD, 1)], 0)]
    for i, ts in enumerate(helpers.distinct_query_terms(rng, n_terms, 30, 2, 5)):
        specs.append(("bool", [(ob.MUST if i % 2 == 0 and len(ts) <= 3 else ob.SHOULD, t) for t in ts], 0))
    oq, oc = ob.make_queries(specs)
    q = np.zeros(len(oq), engine.QUERY_DTYPE)
    q["clause_begin"], q["n_clauses"], q["flags"] = oq["clause_begin"], oq["n_clauses"], engine.Q_BOOLEAN
    c = np.zeros(len(oc), engine.CLAUSE_DTYPE)
    c["occur"], c["term_id"] = oc["occur"], oc["term_id"]
    c["weight"] = [np.float32(codec.bm25_idf(int(df0[t]), doc_count)) for t in oc["term_id"]]
    got = sharded.ShardedSearcher(eng).search_batch(q, c, k)
    torch.cuda.synchronize()
    ok = True
    if rank == 0:
        want = helpers.oracle_index(segs).search_batch(oq, oc, k, parallel_mode=1, n_threads=8)
        try:
            helpers.assert_same_topdocs(got, want, "sharded k=%d" % k)
            assert int(want[1].max()) == k
            print("SHARDED_DEEPK_OK queries=%d" % len(q))
        except AssertionError as e:
            ok = False
            print("SHARDED_DEEPK_MISMATCH", e)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
