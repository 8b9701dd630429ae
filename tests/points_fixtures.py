"""Leaves with point fields for the PointRangeQuery tests, and an independent numpy model of the range doc sets."""
import numpy as np

import helpers
import points_oracle as po

# field ids: 0 a LongPoint timestamp rising with docid (noise, some docs with two values, some with none),
# 1 an IntPoint uniform value (every doc exactly one: the all_docs_match shortcut applies), 2 a LongPoint only in leaf 0
TS, UNI, PART = 0, 1, 2
DFS = [30000, 9000, 3000, 700, 129, 100, 5000, 1500, 1]


def leaf_points(rng, max_doc, seg_i):
    """{field: (nbytes, docs, packed [n, nbytes], keys as python-comparable uint64)}"""
    out = {}
    base = np.arange(max_doc, dtype=np.int64) * 10 + rng.integers(-30, 30, max_doc)
    has = rng.random(max_doc) < 0.97
    has[256:384] = True            # a block where every doc has a value ...
    has[384:512] = True
    has[384 + 77] = False          # ... and one that misses a single doc
    docs = np.nonzero(has)[0].astype(np.int32)
    vals = base[docs]
    two = docs[rng.random(docs.size) < 0.05]
    docs = np.concatenate([docs, two]).astype(np.int32)
    vals = np.concatenate([vals, base[two] + 7])
    perm = rng.permutation(docs.size)
    docs, vals = docs[perm], vals[perm]
    out[TS] = (8, docs, vals)
    udocs = rng.permutation(max_doc).astype(np.int32)
    uvals = rng.integers(-(1 << 31), 1 << 31, max_doc)
    out[UNI] = (4, udocs, uvals)
    if seg_i == 0:
        pd = rng.choice(max_doc, max_doc // 3, replace=False).astype(np.int32)
        out[PART] = (8, pd, rng.integers(-(1 << 40), 1 << 40, pd.size))
    return out


def packed_of(nbytes, vals):
    """IntPoint / LongPoint pack, vectorised: the sign bit flipped, big-endian."""
    if nbytes == 8:
        u = np.asarray(vals, np.int64).view(np.uint64) ^ np.uint64(1 << 63)
        return u.astype(">u8").view(np.uint8).reshape(-1, 8)
    u = np.asarray(vals, np.int64).astype(np.int32).view(np.uint32) ^ np.uint32(1 << 31)
    return u.astype(">u4").view(np.uint8).reshape(-1, 4)


def build(seed, sizes=(70001, 30007), doc_version=1):
    rng = np.random.default_rng(seed)
    segs, points = [], []
    for i, md in enumerate(sizes):
        seg, _ = helpers.build_segment(rng, md, DFS, doc_version=doc_version,
                                       live_fraction=0.9 if i == 1 else None)
        segs.append(seg)
        pts = leaf_points(rng, md, i)
        points.append({f: (nb, d, packed_of(nb, v), v) for f, (nb, d, v) in pts.items()})
    return segs, points


def model_docs(points_leaf, rng_row):
    """numpy model of PointRangeWeight's doc set: None without the field, else the sorted distinct docs with a
    value v (signed, as encoded) whose packed bytes lie in [lower, upper]."""
    f = int(rng_row["field"])
    if f not in points_leaf:
        return None
    nb, docs, packed, _ = points_leaf[f]
    keys = np.zeros(len(docs), np.uint64)
    for j in range(nb):
        keys = (keys << np.uint64(8)) | packed[:, j].astype(np.uint64)
    lo = int.from_bytes(bytes(rng_row["lower"][:nb]), "big")
    hi = int.from_bytes(bytes(rng_row["upper"][:nb]), "big")
    sel = (keys >= np.uint64(lo)) & (keys <= np.uint64(hi))
    return np.unique(docs[sel]).astype(np.int32)
