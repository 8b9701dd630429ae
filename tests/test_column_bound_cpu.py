"""The slack of the decode-free k_eval_or's column bound (query_kernels.cu: columns_only_window), restated in numpy.

A whole window in which only score columns have postings is counted from their bitmaps when C <= theta' =
theta * (1 - 2^-17) (rounded down), C being the round-up sum of the columns' block maxima.  No doc whose f32 score
(clause order, round to nearest, from +0.0f) is above theta may hide in such a window.  Here the block maxima are the
cells themselves (the tightest the table can be) and theta the smallest float for which the bound clears."""
import numpy as np

F32 = np.float32
SLACK = 1.0 - 2.0 ** -17


def _round_up(x64):
    r = np.float32(x64)
    return r if float(r) >= x64 else np.nextafter(r, F32(np.inf))


def _round_down(x64):
    r = np.float32(x64)
    return r if float(r) <= x64 else np.nextafter(r, F32(-np.inf))


def _smallest_theta(bound):
    t = np.float32(float(bound) / SLACK)
    while _round_down(float(t) * SLACK) >= bound:
        t = np.nextafter(t, F32(0))
    while _round_down(float(t) * SLACK) < bound:
        t = np.nextafter(t, F32(np.inf))
    return t


def test_bound_never_below_the_clause_order_sum():
    rng = np.random.default_rng(0xB0B)
    for trial in range(20000):
        n = int(rng.integers(1, 10))  # k_eval_or takes at most kMaxTerms = 9 clauses
        scale = [1e-3, 1.0, 30.0][trial % 3]
        cells = (rng.random(n) * scale + scale * 1e-3).astype(F32)
        s_f = F32(0)
        for v in cells:
            s_f = F32(s_f + v)  # round to nearest, clause order
        c_ub = F32(0)
        for v in rng.permutation(cells):  # the kernel adds the columns in butterfly order, rounding up
            c_ub = _round_up(float(c_ub) + float(v))  # the f64 sum of two such f32 values is exact
        theta = _smallest_theta(c_ub)
        assert s_f <= theta, (trial, cells, s_f, c_ub, theta)
