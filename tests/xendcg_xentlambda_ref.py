"""NumPy restatement of LightGBM 3.2's rank_xendcg and cross_entropy_lambda objectives and of the cross_entropy_lambda and
kullback_leibler metrics ([UPSTREAM] rank_objective.hpp RankXENDCG, xentropy_objective.hpp CrossEntropyLambda, xentropy_metric.hpp).
Independent of the product: fp64 NumPy, cast to float32 where LightGBM casts to score_t, sums taken in document order."""
import numpy as np

F32 = np.float32
K_EPSILON = 1e-15


class Lcg:
    """[UPSTREAM Random]: x <- 214013 x + 2531011 (uint32), NextFloat = ((x >> 16) & 0x7fff) / 32768"""

    def __init__(self, seed):
        self.x = seed & 0xFFFFFFFF

    def next_float(self):
        self.x = (214013 * self.x + 2531011) & 0xFFFFFFFF
        return F32(((self.x >> 16) & 0x7FFF) / 32768.0)


def _seq_sum(a):
    return float(np.add.accumulate(a)[-1])


def xendcg_query(score, label, rand):
    """(lambda, hessian, scale) float32 of one query; draws len(score) floats from `rand` unless the query has at most one document.
    scale = max(|f32 t1|, |f32 t2|, |f32 t3|), the size of the float sum that makes lambda"""
    cnt = len(score)
    if cnt <= 1:
        z = np.zeros(cnt, F32)
        return z, z.copy(), z.copy()
    score = np.asarray(score, np.float64)
    with np.errstate(all="ignore"):
        wmax = score[0]
        for v in score[1:]:
            wmax = max(v, wmax)
        e = np.exp(score - wmax)
        rho = e / _seq_sum(e)
        r = np.array([rand.next_float() for _ in range(cnt)], F32).astype(np.float64)
        params = np.ldexp(1.0, np.asarray(label).astype(np.int64)) - r
        inv = 1.0 / max(K_EPSILON, _seq_sum(params))
        t1 = -params * inv + rho
        lam = t1.astype(F32)
        p1 = t1 / (1.0 - rho)
        t2 = rho * (_seq_sum(p1) - p1)
        lam = lam + t2.astype(F32)
        p2 = t2 / (1.0 - rho)
        t3 = rho * (_seq_sum(p2) - p2)
        lam = lam + t3.astype(F32)
        hes = (rho * (1.0 - rho)).astype(F32)
        scale = np.maximum(np.maximum(np.abs(t1.astype(F32)), np.abs(t2.astype(F32))), np.abs(t3.astype(F32)))
    return lam, hes, scale


def xendcg_gradients(score, label, group_sizes, rands, weight=None):
    """whole dataset: (g, h, scale) float32; rands[q] is query q's Lcg and advances by the query's size (sizes above one)"""
    n = len(score)
    g, h, sc = np.zeros(n, F32), np.zeros(n, F32), np.zeros(n, F32)
    b = 0
    for q, cnt in enumerate(group_sizes):
        g[b:b + cnt], h[b:b + cnt], sc[b:b + cnt] = xendcg_query(score[b:b + cnt], label[b:b + cnt], rands[q])
        b += cnt
    if weight is not None:         # score_t * label_t
        with np.errstate(all="ignore"):
            g, h, sc = g * weight, h * weight, sc * weight
    return g, h, sc


def xendcg_rands(num_queries, seed=5):
    return [Lcg(seed + q) for q in range(num_queries)]


def xentlambda_gradients(s, y, w=None):
    """(g, h) float32 of cross_entropy_lambda at raw scores s"""
    s = np.asarray(s, np.float64)
    y = np.asarray(y, F32).astype(np.float64)
    with np.errstate(all="ignore"):
        if w is None:
            z = 1.0 / (1.0 + np.exp(-s))
            return (z - y).astype(F32), (z * (1.0 - z)).astype(F32)
        w = np.asarray(w, F32).astype(np.float64)
        epf = np.exp(s)
        hhat = np.log1p(epf)
        z = 1.0 - np.exp(-w * hhat)
        enf = 1.0 / epf
        g = (1.0 - y / z) * w / (1.0 + enf)
        c = 1.0 / (1.0 - z)
        d = 1.0 + epf
        a = w * epf / (d * d)
        d = c - 1.0
        b = (c / (d * d)) * (1.0 + w * epf - c)
        return g.astype(F32), (a * (1.0 + y * b)).astype(F32)


def xentlambda_init_score(y, w=None):
    y = np.asarray(y, F32).astype(np.float64)
    w = np.ones_like(y) if w is None else np.asarray(w, F32).astype(np.float64)
    return float(np.log(np.expm1((y * w).sum() / w.sum())))


def xent_loss(y, p):
    with np.errstate(all="ignore"):
        a = y * np.where(p > 1e-12, np.log(np.where(p > 1e-12, p, 1.0)), np.log(1e-12))
        q = 1.0 - p
        b = (1.0 - y) * np.where(q > 1e-12, np.log(np.where(q > 1e-12, q, 1.0)), np.log(1e-12))
    return -(a + b)


def yent_loss(y):
    """minus the entropy of the label: y log y + (1 - y) log(1 - y), each term dropped at arguments up to 1e-12"""
    q = 1.0 - y
    with np.errstate(all="ignore"):
        return np.where(y > 1e-12, y * np.log(np.where(y > 1e-12, y, 1.0)), 0.0) + np.where(q > 1e-12, q * np.log(np.where(q > 1e-12, q, 1.0)), 0.0)


def metric_xentlambda(p, y, w=None):
    """p = the objective's output transform of the raw score"""
    y = np.asarray(y, F32).astype(np.float64)
    w = np.ones_like(y) if w is None else np.asarray(w, F32).astype(np.float64)
    return float(xent_loss(y, 1.0 - np.exp(-w * p)).sum() / len(y))


def metric_kldiv(p, y, w=None):
    y = np.asarray(y, F32).astype(np.float64)
    w = np.ones_like(y) if w is None else np.asarray(w, F32).astype(np.float64)
    return float((w * yent_loss(y)).sum() / w.sum() + (w * xent_loss(y, p)).sum() / w.sum())
