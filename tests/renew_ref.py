"""NumPy restatement of LightGBM 3.2's leaf renewal for regression_l1, quantile and mape (regression_objective.hpp PercentileFun and
WeightedPercentileFun, SerialTreeLearner::RenewTreeOutput), as the engine runs it (renew_kernel.cuh).  It imports neither mmlspark_b200
nor oracle.

- A leaf's rows are its in-bag rows in partition order, which is ascending row index.  The residual of a row is float64(label) - score,
  under rf float64(label) - the init score.
- The residuals are sorted with a stable sort: equal residuals keep their row order, and -0.0 ties with +0.0 but keeps its own value.
- PercentileFun: fp = (cnt - 1)(1 - alpha) in double, pos = int(fp) + 1 in the descending order d[]; pos < 1 gives d[0], pos >= cnt
  gives d[cnt - 1], otherwise v1 - (v1 - v2) * (fp - (pos - 1)) with v1 = d[pos - 1], v2 = d[pos].
- WeightedPercentileFun: the cdf of the weights in ascending order, summed one by one in fp64; threshold = cdf[cnt - 1] * alpha; pos =
  upper_bound(cdf, threshold), at most cnt - 1; pos 0 or cnt - 1 gives that residual; otherwise, with v1, v2 the residuals at pos - 1
  and pos, (threshold - cdf[pos]) / step * (v2 - v1) + v1 where step = cdf[pos + 1] - cdf[pos] >= 1, else v2.
- alpha is double(float32(alpha)) for quantile (the objective keeps it as a float) and 0.5 for regression_l1 and mape.  mape's weights
  are float32 1 / max(1, |label|), times the weight if there is one.
- Data-parallel: a leaf's value is the sum of the rank-local percentiles over the ranks that have rows in it, divided by their number,
  or 0 if no rank does.
With T = float32 the same functions are the init score's label percentile (the label type is float32)."""
import math

import numpy as np


def renew_alpha(objective, alpha=0.9):
    return float(np.float32(alpha)) if objective == "quantile" else 0.5


def mape_weights(label, weight=None):
    y = np.asarray(label, np.float32)
    w = (np.float32(1.0) / np.maximum(np.float32(1.0), np.abs(y))).astype(np.float32)
    return w if weight is None else (w * np.asarray(weight, np.float32)).astype(np.float32)


def _ascending(v):
    return np.argsort(v, kind="stable")


def percentile(values, alpha, T=np.float64):
    """PercentileFun over values in partition order"""
    v = np.asarray(values, T)
    cnt = len(v)
    if cnt <= 1:
        return v[0]
    d = v[_ascending(v)][::-1]
    float_pos = (cnt - 1) * (1.0 - alpha)
    pos = int(float_pos) + 1
    if pos < 1:
        return d[0]
    if pos >= cnt:
        return d[cnt - 1]
    bias = float_pos - (pos - 1)
    v1, v2 = d[pos - 1], d[pos]
    return T(float(v1) - float(T(v1 - v2)) * bias)


def block_scan_cdf(w):
    """not upstream's order: the cdf as a 1024-thread block scan sums it (lane scans of 32, a scan of the 32 warp totals, then
    carry + (warp offset + lane sum) per 1024-row chunk).  Tests use it to show that a case tells the two orders apart."""
    w = np.asarray(w, np.float64)
    out, carry = np.empty(len(w)), 0.0
    for base in range(0, len(w), 1024):
        m = min(1024, len(w) - base)
        v = np.zeros(1024)
        v[:m] = w[base:base + m]
        incl = v.reshape(32, 32).copy()
        for o in (1, 2, 4, 8, 16):
            incl[:, o:] = incl[:, o:] + incl[:, :-o].copy()
        tot = incl[:, 31].copy()
        for o in (1, 2, 4, 8, 16):
            tot[o:] = tot[o:] + tot[:-o].copy()
        c = carry + (np.concatenate([[0.0], tot[:-1]])[:, None] + incl)
        out[base:base + m] = c.reshape(-1)[:m]
        carry = c.reshape(-1)[-1]
    return out


def weighted_cdf(values, weights, scan=np.add.accumulate):
    """(ascending order, the cdf of the weights in that order, summed one by one in fp64 unless `scan` says otherwise)"""
    order = _ascending(np.asarray(values))
    return order, scan(np.asarray(weights, np.float64)[order])


def weighted_percentile(values, weights, alpha, T=np.float64, why=None, scan=np.add.accumulate):
    """WeightedPercentileFun over values and weights in partition order; `why` (a list) gets a line when the threshold lies within
    2 ulps of a cdf value without being equal to it, where the last bits of a sum would decide the position"""
    v = np.asarray(values, T)
    cnt = len(v)
    if cnt <= 1:
        return v[0]
    order, cdf = weighted_cdf(v, weights, scan)
    threshold = cdf[cnt - 1] * alpha
    if why is not None:
        near = (cdf != threshold) & (np.abs(cdf - threshold) <= 2 * np.spacing(abs(threshold)))
        if near.any():
            why.append("threshold %r within 2 ulps of cdf value %r" % (threshold, cdf[np.nonzero(near)[0][0]]))
    pos = min(int(np.searchsorted(cdf, threshold, side="right")), cnt - 1)
    if pos == 0 or pos == cnt - 1:
        return v[order[pos]]
    v1, v2 = v[order[pos - 1]], v[order[pos]]
    step = cdf[pos + 1] - cdf[pos]
    if step >= 1.0:
        return T((threshold - cdf[pos]) / step * float(T(v2 - v1)) + float(v1))
    return v2


def leaf_value(res, alpha, w=None, why=None, scan=np.add.accumulate):
    return float(percentile(res, alpha) if w is None else weighted_percentile(res, w, alpha, why=why, scan=scan))


def renew(leaf_rows, label, score, alpha, weight=None, rank_of_row=None, R=1, why=None, scan=np.add.accumulate):
    """every leaf's renewed output: leaf_rows, each leaf's (in-bag) rows ascending; score: per row, or the rf init score; weight: the
    renewal weights (mape_weights for mape), None unweighted; rank_of_row with R > 1: the data-parallel average"""
    res = np.asarray(label, np.float32).astype(np.float64) - (np.asarray(score, np.float64) if np.ndim(score) else float(score))
    res = np.broadcast_to(res, (len(label),))
    out = []
    for rows in leaf_rows:
        rows = np.asarray(rows)
        vals = []
        for r in range(R):
            rr = rows if R == 1 else rows[rank_of_row[rows] == r]
            if len(rr):
                vals.append(leaf_value(res[rr], alpha, None if weight is None else np.asarray(weight)[rr], why, scan))
        if R == 1:
            out.append(vals[0] if vals else 0.0)
        else:
            out.append(math.fsum(vals) / len(vals) if vals else 0.0)
    return out
