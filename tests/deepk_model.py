"""Independent numpy model of the deep-k theta bound (k > 1024): the per-query score bucket map the planner picks
(deep_bucket_maps in search.cu), the bucket of a score and a bucket's lower edge (deep_key / deep_publish in
eval_shared.cuh), theta from a histogram, and TopDocsCollector's heap (top_docs.rs over std BinaryHeap) to compare
the oracle against."""
import numpy as np

B = 256


def to_ordered(s):
    """float_to_ordered: f32 -> u32, monotone in the float order (-0 just below +0, NaNs outside)."""
    u = np.asarray(s, np.float32).view(np.uint32).astype(np.uint64)
    neg = (u & 0x80000000) != 0
    return np.where(neg, (~u) & 0xffffffff, u | 0x80000000).astype(np.uint32)


def from_ordered(o):
    o = np.asarray(o, np.uint64)
    top = (o & 0x80000000) != 0
    return np.where(top, o & 0x7fffffff, (~o) & 0xffffffff).astype(np.uint32).view(np.float32)


def bucket_map(u):
    """(base, shift) for a query whose scores are bounded by u (f32): the top bucket starts at u and the 255 below
    are 1/32 octave wide; without a finite positive bound the absolute map (0, 24)."""
    u = np.float32(u)
    if u > 0 and np.isfinite(u):
        bits = int(np.array([u], np.float32).view(np.uint32)[0])
        return (bits | 0x80000000) - ((B - 1) << 18), 18
    return 0, 24


def score_bound(w1s):
    """The planner's U: the round-up f32 sum of nextafter(w1) over the clauses' weight * (k1 + 1), zero ones skipped;
    inf when a clause has no usable bound (negative weight)."""
    u = np.float32(0)
    for w1 in w1s:
        w1 = np.float32(w1)
        if w1 == 0:
            continue
        if not (w1 >= 0 and np.isfinite(w1)):
            return np.float32(np.inf)
        u = np.nextafter(np.float32(u + np.nextafter(w1, np.float32(np.inf))), np.float32(np.inf))
    return u


def key(m, s):
    base, shift = m
    o = to_ordered(s).astype(np.int64)
    return np.clip((o - base) >> shift, 0, B - 1).astype(np.int64)


def edge(m, b):
    """Lower edge of bucket b >= 1 (bucket 0: -inf)."""
    base, shift = m
    if b == 0:
        return np.float32(-np.inf)
    return from_ordered(np.array([base + (b << shift)], np.uint64))[0]


def histogram(m, scores):
    s = np.asarray(scores, np.float32)
    s = s[~np.isnan(s)]
    return np.bincount(key(m, s), minlength=B)


def theta(m, hist, k):
    """edge(b) for the largest b whose suffix count is >= k (-inf when only the floor bucket qualifies)."""
    suf = np.cumsum(np.asarray(hist)[::-1])[::-1]
    ok = np.nonzero(suf >= k)[0]
    return edge(m, int(ok[-1])) if len(ok) and ok[-1] >= 1 else np.float32(-np.inf)


def top_docs(stream, k):
    """TopDocsCollector over (doc, score) in collection order: add_doc into std's BinaryHeap with the reversed
    score-only order (top_docs.rs:67-76), then top_docs() pops min(total, len) times and reverses."""
    data = []

    def le(a, b):  # a <= b in the heap's order  <=>  a.score >= b.score
        return a[1] >= b[1]

    def sift_up(start, pos):
        e = data[pos]
        while pos > start:
            p = (pos - 1) // 2
            if le(e, data[p]):
                break
            data[pos] = data[p]
            pos = p
        data[pos] = e

    def sift_down(pos, end, to_bottom):
        start, e = pos, data[pos]
        c = 2 * pos + 1
        while c < end:
            if c + 1 < end and le(data[c], data[c + 1]):
                c += 1
            if not to_bottom and e[1] <= data[c][1]:
                break
            data[pos] = data[c]
            pos = c
            c = 2 * pos + 1
        data[pos] = e
        if to_bottom:
            sift_up(start, pos)

    total = 0
    for d, s in stream:
        total += 1
        if len(data) < k:
            data.append((d, s))
            sift_up(0, len(data) - 1)
        elif data[0][1] < s:
            data[0] = (d, s)
            sift_down(0, len(data), False)
    out = []
    for _ in range(min(total, len(data))):
        item = data.pop()
        if data:
            item, data[0] = data[0], item
            sift_down(0, len(data), True)
        out.append(item)
    return out[::-1], total
