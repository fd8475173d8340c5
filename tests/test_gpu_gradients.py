"""The K1/K2 gradient kernels (k_grad_* in csrc/kernels.cuh) element by element against a NumPy restatement of the LightGBM 3.2
GetGradients formulas, at scores chosen through the dataset's init_score: signed zeros, denormal-sized and huge scores where exp
overflows and sigmoids saturate, huber's |diff| == alpha, quantile's float32 delta, zero and extreme weights.  Gradients are read
with B200GBM_BoosterGetGradients before the first iteration, so the scores are exactly the init scores.

The reference is independent of the product and of the oracle: fp64 NumPy, cast to float32 where LightGBM casts to score_t.
Bar: non-finite values at the same positions with the same kind (and the same sign for infinities; the sign of a NaN made by an
invalid operation is not specified by IEEE 754 and differs between x86 and the GPU), finite values within 1 float32 ulp (the device
exp / log may differ from the host's in the last fp64 bit) and at least 99.9 % bit-equal.  Lambdarank is bit-exact without the
normalisation and within 2 ulps with it (the kernel sums sum_lambdas in another order)."""
import math
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 learning_rate=0.1 min_data_in_leaf=20 verbosity=-1 "
N = 300_001             # the grid-stride loops (num_sms * 8 blocks of 256 threads) wrap around and end on a ragged tail
GRID = np.array([0.0, -0.0, 1e-300, -1e-300, 1e-8, -1e-8, 0.5, -0.5, 5.0, -5.0, 30.0, -30.0, 37.0, -37.0, 700.0, -700.0,
                 709.7, -709.7, 710.0, -710.0, 745.0, -745.0, 800.0, -800.0])
HUBER_ALPHA = 0.75      # labels are multiples of 1/4, so label +- alpha is exact and |diff| == alpha really occurs


# ------------------------------------------------------------------------------------------------ comparison
def _ordered(a):
    """float32 -> integers in the same order, adjacent floats adjacent (-0.0 and +0.0 one apart)"""
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF) - 1, b)


def _compare(got, want, max_ulp, what):
    """asserts the bar of the module docstring; returns the number of elements that are not bit-equal"""
    got = np.asarray(got, dtype=np.float32)
    want = np.asarray(want, dtype=np.float32)
    assert got.shape == want.shape, what
    fg, fw = np.isfinite(got), np.isfinite(want)
    bad = np.nonzero(fg != fw)[0]
    assert len(bad) == 0, "%s: finite / non-finite differ at %d positions, first %d: got %r want %r" % (what, len(bad), bad[0], got[bad[0]], want[bad[0]])
    nf = ~fw
    assert np.array_equal(np.isnan(got[nf]), np.isnan(want[nf])), what + ": inf where NaN is expected or the reverse"
    inf = np.isinf(want)
    assert np.array_equal(got[inf], want[inf]), what + ": infinities of the wrong sign"
    d = np.abs(_ordered(got[fw]) - _ordered(want[fw]))
    if len(d) and d.max() > max_ulp:
        i = np.nonzero(fw)[0][np.argmax(d)]
        raise AssertionError("%s: %d ulps apart at %d: got %r want %r (%d elements over %d ulps)" % (what, d.max(), i, got[i], want[i], int((d > max_ulp).sum()), max_ulp))
    not_equal = int((got[fw].view(np.int32) != want[fw].view(np.int32)).sum())
    assert not_equal <= 0.001 * got.size, "%s: %d of %d elements are not bit-equal" % (what, not_equal, got.size)
    return not_equal


# ------------------------------------------------------------------------------------------------ inputs
def _scores(rng, n):
    s = 3.0 * rng.standard_normal(n)
    pick = rng.random(n) < 0.5
    s[pick] = GRID[rng.integers(0, len(GRID), int(pick.sum()))]
    s[:len(GRID)] = GRID
    return s


def _weights(mode, rng, n):
    if mode == "none":
        return None
    if mode == "uniform":
        return np.full(n, 0.75, dtype=np.float32)
    if mode == "zeros":
        w = (0.5 + rng.random(n)).astype(np.float32)
        w[rng.random(n) < 0.1] = 0.0
        return w
    assert mode == "wide"
    return (10.0 ** rng.uniform(-20.0, 20.0, n)).astype(np.float32)


def _labels(kind, rng, n):
    if kind == "real":          # multiples of 1/4 around 0; label 0 under the grid scores (quantile's -0.0 delta)
        y = np.round(rng.standard_normal(n) * 12.0) / 4.0
        y[:len(GRID)] = 0.0
    elif kind == "mape":        # |y| < 1 for half of the rows, where the label weight is 1
        y = np.where(rng.random(n) < 0.5, rng.uniform(-1.0, 1.0, n), np.round(rng.standard_normal(n) * 12.0) / 4.0)
        y[:len(GRID)] = 0.0
    elif kind == "count":       # poisson / gamma / tweedie: >= 0, zeros included
        y = np.where(rng.random(n) < 0.3, 0.0, rng.gamma(2.0, 1.5, n))
        y[:len(GRID)] = np.where(np.arange(len(GRID)) % 2 == 0, 0.0, 1.0)
    elif kind == "prob":        # cross_entropy: 0, 1 and fractions
        u = rng.random(n)
        y = np.where(u < 0.25, 0.0, np.where(u < 0.5, 1.0, rng.random(n)))
    else:
        raise ValueError(kind)
    return y.astype(np.float32)


# ------------------------------------------------------------------------------------------------ NumPy reference
def _class_weights(pos, neg, is_unbalance, spw):
    """[LightGBM BinaryLogloss::Init] {w_neg, w_pos}"""
    wn, wp = 1.0, 1.0
    if is_unbalance and pos > 0 and neg > 0:
        if pos > neg:
            wn = pos / neg
        else:
            wp = neg / pos
    return wn, wp * spw


def _binary(s, is_pos, sig, wn, wp, w64):
    lab = np.where(is_pos, 1.0, -1.0)
    lw = np.where(is_pos, wp, wn)
    response = -lab * sig / (1.0 + np.exp(lab * sig * s))
    ar = np.abs(response)
    g, h = response * lw, ar * (sig - ar) * lw
    if w64 is not None:
        g, h = g * w64, h * w64
    return g, h


def _sign(x):
    return (x > 0).astype(np.float64) - (x < 0).astype(np.float64)


def reference_gradients(objective, p, s, y, w):
    """(g, h) float32 class-major, as LightGBM's <Objective>::GetGradients computes them"""
    y64 = y.astype(np.float64)
    w64 = None if w is None else w.astype(np.float64)
    f32 = np.float32
    with np.errstate(all="ignore"):
        if objective in ("regression_l1", "quantile", "mape"):
            h = np.ones_like(y) if w is None else w.copy()
            if objective == "quantile":          # delta and alpha are score_t
                delta = (s - y64).astype(f32)
                a = f32(p["alpha"])
                g = np.where(delta >= 0, f32(1.0) - a, -a).astype(f32)
                if w is not None:
                    g = g * w
            else:
                sgn = _sign(s - y64)
                if objective == "regression_l1":
                    g = sgn if w is None else sgn * w64
                else:                            # label_weight = 1 / max(1, |y|) (* w) in float
                    lw = f32(1.0) / np.maximum(f32(1.0), np.abs(y))
                    if w is not None:
                        lw = lw * w
                    g = sgn * lw.astype(np.float64)
            return g.astype(f32), h.astype(f32)
        if objective == "binary":
            is_pos = y > 0
            npos = int(is_pos.sum())
            if npos == 0 or npos == len(y):
                return np.zeros(len(y), f32), np.zeros(len(y), f32)
            wn, wp = _class_weights(npos, len(y) - npos, p["is_unbalance"], p["scale_pos_weight"])
            g, h = _binary(s, is_pos, p["sigmoid"], wn, wp, w64)
            return g.astype(f32), h.astype(f32)
        if objective == "multiclassova":
            K, n = p["num_class"], len(y)
            g, h = np.zeros(K * n, f32), np.zeros(K * n, f32)
            li = y.astype(np.int64)
            for k in range(K):
                is_pos = li == k
                npos = int(is_pos.sum())
                if npos == 0 or npos == n:
                    continue
                wn, wp = _class_weights(npos, n - npos, False, 1.0)
                gk, hk = _binary(s[k * n:(k + 1) * n], is_pos, p["sigmoid"], wn, wp, w64)
                g[k * n:(k + 1) * n], h[k * n:(k + 1) * n] = gk, hk
            return g, h
        if objective == "multiclass":
            K, n = p["num_class"], len(y)
            sk = s.reshape(K, n)
            wmax = sk[0].copy()
            for k in range(1, K):
                wmax = np.maximum(wmax, sk[k])
            wsum = np.zeros(n)
            for k in range(K):
                wsum = wsum + np.exp(sk[k] - wmax)
            factor = K / (K - 1.0)
            li = y.astype(np.int64)
            g, h = np.zeros((K, n), f32), np.zeros((K, n), f32)
            for k in range(K):
                pk = np.exp(sk[k] - wmax) / wsum
                gk, hk = np.where(li == k, pk - 1.0, pk), factor * pk * (1.0 - pk)
                if w is not None:
                    gk, hk = gk * w64, hk * w64
                g[k], h[k] = gk, hk
            return g.ravel(), h.ravel()
        if objective == "regression":
            g, h = s - y64, np.ones_like(s)
        elif objective == "huber":
            diff = s - y64
            g, h = np.where(np.abs(diff) <= p["alpha"], diff, _sign(diff) * p["alpha"]), np.ones_like(s)
        elif objective == "fair":
            c, x = p["fair_c"], s - y64
            g, h = c * x / (np.abs(x) + c), c * c / ((np.abs(x) + c) * (np.abs(x) + c))
        elif objective == "poisson":
            g, h = np.exp(s) - y64, np.exp(s + p["poisson_max_delta_step"])
        elif objective == "gamma":
            g, h = 1.0 - y64 * np.exp(-s), y64 * np.exp(-s)
        elif objective == "tweedie":
            rho = p["tweedie_variance_power"]
            e1, e2 = np.exp((1 - rho) * s), np.exp((2 - rho) * s)
            g, h = -y64 * e1 + e2, -y64 * (1 - rho) * e1 + (2 - rho) * e2
        elif objective == "cross_entropy":
            z = 1.0 / (1.0 + np.exp(-s))
            g, h = z - y64, z * (1.0 - z)
        else:
            raise ValueError(objective)
        if w is not None:
            g, h = g * w64, h * w64
        return g.astype(f32), h.astype(f32)


# ------------------------------------------------------------------------------------------------ point-wise objectives
def _param_string(p):
    return " ".join("%s=%s" % (k, str(v).lower() if isinstance(v, bool) else v) for k, v in p.items())


POINTWISE = [  # (objective, params, label kind)
    ("regression", {}, "real"),
    ("huber", {"alpha": HUBER_ALPHA}, "real"),
    ("fair", {"fair_c": 1.3}, "real"),
    ("poisson", {"poisson_max_delta_step": 0.0}, "count"),
    ("poisson", {"poisson_max_delta_step": 0.7}, "count"),
    ("gamma", {}, "count"),
    ("tweedie", {"tweedie_variance_power": 1.1}, "count"),
    ("tweedie", {"tweedie_variance_power": 1.5}, "count"),
    ("tweedie", {"tweedie_variance_power": 1.9}, "count"),
    ("regression_l1", {}, "real"),
    ("quantile", {"alpha": 0.7}, "real"),      # 0.7 is not a float: alpha is used as score_t
    ("mape", {}, "mape"),
    ("cross_entropy", {}, "prob"),
]
CASES = [(o, p, lk, wm) for o, p, lk in POINTWISE for wm in ("none", "uniform", "zeros", "wide")]
_BINARY = [(sg, ub, pr, spw) for sg in (0.5, 1.0, 2.0) for ub in (False, True) for pr in (0.2, 0.8) for spw in (1.0, 3.0)]   # pr: rate of positives
CASES += [("binary", {"sigmoid": sg, "is_unbalance": ub, "scale_pos_weight": spw, "_pos_rate": pr}, "binary", ("none", "uniform", "zeros", "wide")[j % 4])
          for j, (sg, ub, pr, spw) in enumerate(_BINARY)]
CASES += [("binary", {"_pos_rate": 0.0}, "binary", "none")]      # one class only: the class is not trained, gradients are 0
CASES += [("multiclass", {"num_class": K}, "class", wm) for K in (2, 3, 7, 30) for wm in ("none", "wide")]
CASES += [("multiclassova", {"num_class": 4, "sigmoid": sg, "_absent": 2}, "class", wm) for sg, wm in ((1.0, "none"), (2.0, "zeros"))]


def _case_id(c):
    o, p, _, wm = c
    return "-".join([o] + ["%s=%s" % (k.lstrip("_"), v) for k, v in p.items()] + ["w=" + wm])


@pytest.fixture(scope="module")
def big_ds(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(100)
    return capi.Dataset.from_mat(rng.standard_normal((N, 2)), DS_PARAMS)


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_gradients_match_numpy(big_ds, case):
    from mmlspark_b200 import capi
    objective, p, label_kind, wmode = case
    rng = np.random.default_rng(zlib.crc32(_case_id(case).encode()))
    n = N
    K = p.get("num_class", 1) if objective in ("multiclass", "multiclassova") else 1
    if label_kind == "binary":
        y = (rng.random(n) < p["_pos_rate"]).astype(np.float32)
    elif label_kind == "class":
        y = rng.integers(0, K, n)
        if "_absent" in p:
            y[y == p["_absent"]] = (p["_absent"] + 1) % K
        y = y.astype(np.float32)
    else:
        y = _labels(label_kind, rng, n)
    s = np.concatenate([_scores(rng, n) for _ in range(K)])
    if objective == "huber":                 # |score - label| == alpha exactly
        at = np.nonzero(rng.random(n) < 0.05)[0]
        s[at] = y[at].astype(np.float64) + np.where(rng.random(len(at)) < 0.5, HUBER_ALPHA, -HUBER_ALPHA)
    if objective == "multiclass":            # spreads over 700 within a row
        at = np.nonzero(rng.random(n) < 0.05)[0]
        top = rng.integers(0, K, len(at))
        s[top * n + at] = 800.0
        s[((top + 1 + rng.integers(0, K - 1, len(at))) % K) * n + at] = -800.0 + rng.standard_normal(len(at))
    w = _weights(wmode, rng, n)
    big_ds.set_field("label", y).set_field("init_score", s).set_field("weight", w if w is not None else np.zeros(0, np.float32))
    params = {k: v for k, v in p.items() if not k.startswith("_")}
    b = capi.Booster(big_ds, BASE + "objective=%s %s" % (objective, _param_string(params)))
    try:
        g, h = b.get_gradients()
    finally:
        b.free()
    big_ds.set_field("init_score", np.zeros(0))
    rg, rh = reference_gradients(objective, params, s, y, w)
    ng = _compare(g, rg, 1, _case_id(case) + " grad")
    nh = _compare(h, rh, 1, _case_id(case) + " hess")
    print("[gradients] %s: %d grad / %d hess of %d not bit-equal" % (_case_id(case), ng, nh, g.size))
    if objective == "multiclassova":
        k = p["_absent"]
        assert not g[k * n:(k + 1) * n].any() and not h[k * n:(k + 1) * n].any()


# ------------------------------------------------------------------------------------------------ lambdarank
def lr_tile(truncation):
    """j-tile width of k_grad_lambdarank"""
    t = min((48 * 1024 // 8) // max(truncation, 1) - 1, 128)
    return max(t & ~31, 32)


def lambdarank_smem(max_q, truncation):
    """dynamic shared memory of k_grad_lambdarank: six per-document arrays and one j-tile of the pair matrix"""
    return max_q * 32 + 8 + truncation * (lr_tile(truncation) + 1) * 8


LR_SMEM_LIMIT = 200 * 1024
LR_BINS = 1024 * 1024
_SIGMOID_TABLES = {}


def _sigmoid_table(sig):
    """LightGBM's 2^20-entry table of 1 / (1 + exp(x * sigmoid)) over [-50 / sigmoid / 2, 50 / sigmoid / 2), with the host's exp"""
    if sig not in _SIGMOID_TABLES:
        min_in, max_in = -50.0 / sig / 2, 50.0 / sig / 2
        factor = LR_BINS / (max_in - min_in)
        x = (np.arange(LR_BINS, dtype=np.float64) / factor + min_in) * sig
        tab = np.array([1.0 / (1.0 + math.exp(v)) for v in x.tolist()]).astype(np.float32)
        _SIGMOID_TABLES[sig] = (tab, min_in, max_in, factor)
    return _SIGMOID_TABLES[sig]


def _lambdarank_query(s, y, truncation, norm, gain, disc, sig):
    """[LightGBM LambdarankNDCG::GetGradientsForOneQuery]: float32 lambdas / hessians of one query, in document order"""
    tab, min_in, max_in, factor = _sigmoid_table(sig)
    cnt = len(s)
    order = np.argsort(-s, kind="stable")
    ss, ll = s[order], y[order].astype(np.int64)
    k = min(truncation, cnt)
    m = 0.0
    for j, lab in enumerate(np.sort(ll)[::-1][:k]):
        m += disc[j] * gain[lab]
    imd = 1.0 / m if m > 0.0 else m
    teff = min(truncation, cnt - 1)
    lam, hes = np.zeros(cnt, np.float32), np.zeros(cnt, np.float32)
    if teff <= 0:
        return lam, hes
    worst = cnt - 1
    if worst > 0 and ss[worst] == -np.inf:
        worst -= 1
    do_div = norm and ss[0] != ss[worst]
    I, J = np.meshgrid(np.arange(teff), np.arange(cnt), indexing="ij")
    valid = (J > I) & (ss[I] != -np.inf) & (ss[J] != -np.inf) & (ll[I] != ll[J])
    with np.errstate(all="ignore"):
        ih = ll[I] > ll[J]
        hi, lo = np.where(ih, I, J), np.where(ih, J, I)
        ds = np.where(valid, ss[hi] - ss[lo], 0.0)
        delta = (gain[ll[hi]] - gain[ll[lo]]) * np.abs(disc[hi] - disc[lo]) * imd
        if do_div:
            delta = delta / (np.float64(np.float32(0.01)) + np.abs(ds))
        idx = np.clip((ds - min_in) * factor, 0, LR_BINS - 1).astype(np.int64)
        pl = np.where(ds <= min_in, tab[0], np.where(ds >= max_in, tab[-1], tab[idx])).astype(np.float64)
        ph = pl * (1.0 - pl)
        pl = pl * (-sig * delta)
        ph = ph * (sig * sig * delta)
    pl, ph = np.where(valid, pl, 0.0), np.where(valid, ph, 0.0)
    sum_lambdas = float(np.add.accumulate((-2.0 * pl)[valid])[-1]) if valid.any() else 0.0
    ci = np.where(ih, pl.astype(np.float32), -pl.astype(np.float32))      # added to the document at i; the one at j gets -ci
    ch = ph.astype(np.float32)
    # every document sums its pairs as float in the reference's order: (0,p) .. (p-1,p), then (p,p+1) .. (p,cnt-1)
    z = np.zeros((1, cnt - teff), np.float32)
    lam[teff:] = np.add.accumulate(np.vstack([z, -ci[:, teff:]]), axis=0, dtype=np.float32)[-1]
    hes[teff:] = np.add.accumulate(np.vstack([z, ch[:, teff:]]), axis=0, dtype=np.float32)[-1]
    for q in range(teff):
        lam[q] = np.add.accumulate(np.concatenate(([np.float32(0)], -ci[:q, q], ci[q, q + 1:])), dtype=np.float32)[-1]
        hes[q] = np.add.accumulate(np.concatenate(([np.float32(0)], ch[:q, q], ch[q, q + 1:])), dtype=np.float32)[-1]
    if norm and sum_lambdas > 0:
        nf = math.log2(1 + sum_lambdas) / sum_lambdas
        lam = (lam.astype(np.float64) * nf).astype(np.float32)
        hes = (hes.astype(np.float64) * nf).astype(np.float32)
    out_l, out_h = np.empty(cnt, np.float32), np.empty(cnt, np.float32)
    out_l[order], out_h[order] = lam, hes
    return out_l, out_h


def reference_lambdarank(s, y, w, sizes, truncation, norm, label_gain=None, sig=1.0):
    gain = np.array(label_gain if label_gain is not None else [0.0] + [float((1 << i) - 1) for i in range(1, 31)])
    disc = np.array([1.0 / math.log2(2.0 + i) for i in range(int(max(sizes)) + 1)])
    g, h = np.zeros(len(s), np.float32), np.zeros(len(s), np.float32)
    off = 0
    for c in sizes:
        g[off:off + c], h[off:off + c] = _lambdarank_query(s[off:off + c], y[off:off + c], truncation, norm, gain, disc, sig)
        off += c
    if w is not None:
        g = (g.astype(np.float64) * w).astype(np.float32)
        h = (h.astype(np.float64) * w).astype(np.float32)
    return g, h


PATTERNS = ("zeros", "ties", "neginf", "all_neginf_but_one")


def _query_scores(pattern, rng, c):
    if pattern == "zeros":            # as at the first iteration: every pair is a tie
        return np.zeros(c)
    if pattern == "ties":             # coarse: large tie groups, -0.0 among the zeros
        s = np.round(rng.standard_normal(c) * 2.0) / 2.0
        s[rng.random(c) < 0.1] = -0.0
        return s
    if pattern == "neginf":
        s = rng.standard_normal(c)
        s[rng.random(c) < 0.1] = -np.inf
        return s
    s = np.full(c, -np.inf)
    s[rng.integers(0, c)] = rng.standard_normal()
    return s


def _lambdarank_case(rng, sizes, max_label=5):
    s = np.concatenate([_query_scores(PATTERNS[q % len(PATTERNS)], rng, c) for q, c in enumerate(sizes)])
    y = rng.integers(0, max_label, int(sum(sizes))).astype(np.float32)
    return s, y


def _run_lambdarank(built, sizes, s, y, w, params):
    from mmlspark_b200 import capi
    n = int(sum(sizes))
    X = np.random.default_rng(7).standard_normal((n, 2))
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y).set_field("group", np.asarray(sizes, np.int32)).set_field("init_score", s)
    try:
        if w is not None:
            ds.set_field("weight", w)
        b = capi.Booster(ds, BASE + "objective=lambdarank " + params)
        try:
            return b.get_gradients()
        finally:
            b.free()
    finally:
        ds.free()


LR_SIZES = [1, 2, 31, 32, 33, 127, 128, 129, 300, 1000]


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("truncation", [1, 30, 180])
def test_lambdarank_matches_numpy(built, truncation, norm):
    """Every query size around the j-tile widths (128 at truncation <= 47, 32 at 180), each with every score pattern."""
    rng = np.random.default_rng(1000 + truncation + norm)
    sizes = [c for c in LR_SIZES for _ in PATTERNS]
    s, y = _lambdarank_case(rng, sizes)
    at = sum(sizes[:12])                  # one query of 32 documents whose labels are all equal
    y[at:at + sizes[12]] = 2.0
    g, h = _run_lambdarank(built, sizes, s, y, None, "lambdarank_truncation_level=%d lambdarank_norm=%s" % (truncation, str(norm).lower()))
    rg, rh = reference_lambdarank(s, y, None, sizes, truncation, norm)
    what = "lambdarank truncation=%d norm=%s" % (truncation, norm)
    ng, nh = _compare(g, rg, 2 if norm else 0, what + " grad"), _compare(h, rh, 2 if norm else 0, what + " hess")
    print("[gradients] %s: %d grad / %d hess of %d not bit-equal" % (what, ng, nh, g.size))
    if not norm:
        assert ng == 0 and nh == 0
    assert np.abs(g).max() > 0


@pytest.mark.parametrize("norm", [False, True])
def test_lambdarank_label_gain_and_weights(built, norm):
    rng = np.random.default_rng(2000 + norm)
    sizes = [c for c in (2, 33, 129, 300) for _ in PATTERNS]
    s, y = _lambdarank_case(rng, sizes)
    w = (0.25 + 2.0 * rng.random(len(s))).astype(np.float32)
    w[rng.random(len(s)) < 0.1] = 0.0
    g, h = _run_lambdarank(built, sizes, s, y, w, "label_gain=0,1,3,7,15 lambdarank_norm=%s" % str(norm).lower())
    rg, rh = reference_lambdarank(s, y, w, sizes, 30, norm, label_gain=[0, 1, 3, 7, 15])
    ng, nh = _compare(g, rg, 2 if norm else 0, "label_gain grad"), _compare(h, rh, 2 if norm else 0, "label_gain hess")
    if not norm:
        assert ng == 0 and nh == 0


def _max_query(truncation):
    q = (LR_SMEM_LIMIT - 8 - truncation * (lr_tile(truncation) + 1) * 8) // 32
    assert lambdarank_smem(q, truncation) <= LR_SMEM_LIMIT < lambdarank_smem(q + 1, truncation)
    return q


@pytest.mark.parametrize("norm", [False, True])
def test_lambdarank_query_at_the_shared_memory_limit(built, norm):
    rng = np.random.default_rng(3000 + norm)
    q = _max_query(30)                    # 5432 documents at truncation 30
    sizes = [q, 5, 40]
    s = np.concatenate([np.round(rng.standard_normal(q) * 4.0) / 4.0, rng.standard_normal(45)])
    s[rng.random(len(s)) < 0.02] = -np.inf
    y = rng.integers(0, 5, len(s)).astype(np.float32)
    g, h = _run_lambdarank(built, sizes, s, y, None, "lambdarank_truncation_level=30 lambdarank_norm=%s" % str(norm).lower())
    rg, rh = reference_lambdarank(s, y, None, sizes, 30, norm)
    ng, nh = _compare(g, rg, 2 if norm else 0, "smem limit grad"), _compare(h, rh, 2 if norm else 0, "smem limit hess")
    if not norm:
        assert ng == 0 and nh == 0


def test_lambdarank_query_over_the_shared_memory_limit_fails(built):
    from mmlspark_b200 import capi
    q = _max_query(30) + 1
    with pytest.raises(capi.LightGBMError, match="a query group is too large"):
        _run_lambdarank(built, [q], np.zeros(q), np.arange(q, dtype=np.float32) % 3, None, "lambdarank_truncation_level=30")


def test_lambdarank_blocks_loop_over_many_queries(built):
    """3000 queries: more than the kernel's num_sms * 16 blocks, so blocks take several queries one after the other."""
    rng = np.random.default_rng(4000)
    sizes = list(rng.integers(1, 60, 3000))
    s, y = _lambdarank_case(rng, sizes)
    w = (0.5 + rng.random(len(s))).astype(np.float32)
    g, h = _run_lambdarank(built, sizes, s, y, w, "")
    rg, rh = reference_lambdarank(s, y, w, sizes, 30, True)
    ng, nh = _compare(g, rg, 2, "3000 queries grad"), _compare(h, rh, 2, "3000 queries hess")
    print("[gradients] lambdarank 3000 queries: %d grad / %d hess of %d not bit-equal" % (ng, nh, g.size))


# ------------------------------------------------------------------------------------------------ the export leaves training alone
@pytest.mark.parametrize("boosting", ["gbdt", "rf", "goss", "dart"])
def test_get_gradients_leaves_the_model_unchanged(built, boosting):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(5000)
    n = 20000
    X = rng.standard_normal((n, 5))
    y = (X[:, 0] + 0.5 * X[:, 1] * X[:, 2] + 0.3 * rng.standard_normal(n)).astype(np.float32)
    params = BASE + "objective=regression boosting_type=%s" % boosting
    if boosting == "rf":
        params += " bagging_fraction=0.8 bagging_freq=1"
    models = []
    for probe in (False, True):
        ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
        b = capi.Booster(ds, params)
        for _ in range(4):
            if probe:
                g, h = b.get_gradients()
                s = b.get_scores(0)
                np.testing.assert_array_equal(g, (s - y.astype(np.float64)).astype(np.float32))
                np.testing.assert_array_equal(h, np.ones(n, np.float32))
            b.update_one_iter()
        models.append(b.save_model_to_string())
        b.free()
        ds.free()
    assert models[0] == models[1]
