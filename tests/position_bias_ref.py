"""NumPy restatement of the ranking objectives' position factors ([UPSTREAM 4.1 RankingObjective::UpdatePositionBiasFactors and
Metadata::SetPosition, from knowledge]) as the engine computes them (csrc/objective.h, kernels.cuh k_position_bias_update):

- ids: every distinct position value over every rank, sorted; a row's id is the index of its value.  Factors start at 0.
- gradients: lambdarank and rank_xendcg take a query's gradients at s_i + b[id_i] (reference_lambdarank of test_gpu_gradients.py and
  xendcg_gradients of xendcg_xentlambda_ref.py, called on the adjusted scores).
- update, after every training pass, on the weighted g and h: per id p the sums of g and h on K3's fixed-point grid (q = rint(x 2^e),
  e = 34 - ilogb(max |x|) over every rank's rows) and the row count, then in fp64, every operation rounded on its own:
      d1 = -sum_g - b_p * reg * cnt,  d2 = -sum_h - reg * cnt,  b_p += learning_rate * d1 / (|d2| + 0.001)."""
import numpy as np

from test_gpu_gradients import reference_lambdarank
from xendcg_xentlambda_ref import xendcg_gradients


def position_ids(rank_positions):
    """(values, ids per rank): the sorted union of every rank's position values and each rank's rows mapped into it"""
    values = np.unique(np.concatenate([np.asarray(p, np.int64) for p in rank_positions]))
    return values.astype(np.int32), [np.searchsorted(values, np.asarray(p, np.int64)).astype(np.int64) for p in rank_positions]


def exponent(m):
    """K3's fixed-point exponent of a float32 maximum: 34 - ilogb(m), 0 for a zero or non-finite maximum, clamped to [-1000, 1000]"""
    m = np.float32(m)
    if not (m > 0 and np.isfinite(m)):
        return 0
    return int(min(max(34 - (int(np.frexp(m)[1]) - 1), -1000), 1000))


def fixed(x, e):
    """the words rint(x 2^e) of float32 values, as int64 (d_fixed)"""
    return np.rint(np.ldexp(np.asarray(x, np.float32).astype(np.float64), e)).astype(np.int64)


def fixed_sums(ids, g, h, P, eg, eh):
    """(Q_g, Q_h, cnt) int64 [P]: the per-id sums of the words of g and h at exponents (eg, eh) and the row counts"""
    qg, qh, cnt = np.zeros(P, np.int64), np.zeros(P, np.int64), np.zeros(P, np.int64)
    np.add.at(qg, ids, fixed(g, eg))
    np.add.at(qh, ids, fixed(h, eh))
    np.add.at(cnt, ids, 1)
    return qg, qh, cnt


def newton_step(b, qg, qh, cnt, eg, eh, learning_rate, reg):
    """the factors after one update at the sums, in k_position_bias_update's order of fp64 operations"""
    b = np.asarray(b, np.float64)
    sg = qg.astype(np.float64) * np.ldexp(1.0, -eg)
    sh = qh.astype(np.float64) * np.ldexp(1.0, -eh)
    c = cnt.astype(np.float64)
    d1 = (-sg) - ((b * reg) * c)
    d2 = (-sh) - (reg * c)
    return b + (learning_rate * d1) / (np.abs(d2) + 0.001)


def update(b, ids, g, h, learning_rate, reg):
    """one update from the gradients of every rank: ids, g, h are lists with one array per rank (or single arrays for one rank)"""
    if not isinstance(ids, (list, tuple)):
        ids, g, h = [ids], [g], [h]
    g = [np.asarray(a, np.float32) for a in g]
    h = [np.asarray(a, np.float32) for a in h]
    mg = max([np.float32(np.max(np.abs(a))) if len(a) else np.float32(0) for a in g])
    mh = max([np.float32(np.max(np.abs(a))) if len(a) else np.float32(0) for a in h])
    eg, eh = exponent(mg), exponent(mh)
    P = len(b)
    qg, qh, cnt = np.zeros(P, np.int64), np.zeros(P, np.int64), np.zeros(P, np.int64)
    for i, gg, hh in zip(ids, g, h):
        a, c, d = fixed_sums(i, gg, hh, P, eg, eh)
        qg, qh, cnt = qg + a, qh + c, cnt + d
    return newton_step(b, qg, qh, cnt, eg, eh, learning_rate, reg)


def adjusted(score, ids, b):
    return np.asarray(score, np.float64) + np.asarray(b, np.float64)[ids]


def lambdarank(score, ids, b, y, w, sizes, truncation=30, norm=True, label_gain=None, sig=1.0):
    """lambdarank's (g, h) at the adjusted scores"""
    return reference_lambdarank(adjusted(score, ids, b), y, w, sizes, truncation, norm, label_gain=label_gain, sig=sig)


def xendcg(score, ids, b, y, sizes, rands, w=None):
    """rank_xendcg's (g, h, scale) at the adjusted scores; rands advance as in xendcg_gradients"""
    return xendcg_gradients(adjusted(score, ids, b), y, sizes, rands, weight=w)
