"""NumPy restatement of LGBM_BoosterRefit (csrc/refit.cu, refit_kernels.cuh), from LightGBM v3.2.x GBDT::RefitTree and
SerialTreeLearner::FitByExistingTree.

For each iteration the objective's gradients at the current training scores (every row), then for each class k the model
m = it * K + k: per leaf l over the rows whose leaf index is l,
    sum_g = sum of g on K3's fixed-point grid, sum_h = kEpsilon + sum of h on the grid (constant hessians: kEpsilon + rows), cnt = rows;
    output = CalculateSplittedLeafOutput(sum_g, sum_h, l1, l2, max_delta_step), 0 for a leaf no row reaches; with path_smooth > kEpsilon
             and l > 0 smoothed with cnt rows toward leaf_parent(l), the parent's NODE INDEX (upstream passes it where a parent output
             is expected);
    leaf = MaybeRoundToZero(decay * leaf + (1 - decay) * output * shrinkage);
and the class's scores gain the new tree's value at each row's leaf.  The grid sums go through tree_check.quantized: every row's value is
an exact multiple of 2^-e, so their fp64 sums are exact (below 2^18 rows per leaf) and equal the engine's int64 sums times 2^-e."""
import numpy as np

import tree_check as TC

KEPS = float(np.float32(1e-15))      # LightGBM's kEpsilon
ZERO = 1e-35                         # MaybeRoundToZero's threshold, as the engine's HostTree


def gradients(objective, score, y, w=None, num_class=1, sigmoid=1.0):
    """(g, h) float32 class-major [K * n] of regression, binary and multiclass, as tests/test_gpu_gradients.py pins them (binary
    without is_unbalance or scale_pos_weight)"""
    y64 = y.astype(np.float64)
    w64 = None if w is None else np.asarray(w, np.float32).astype(np.float64)
    if objective == "regression":
        g, h = score - y64, np.ones_like(score)
        if w64 is not None:
            g, h = g * w64, h * w64
        return g.astype(np.float32), h.astype(np.float32)
    if objective == "binary":
        lab = np.where(y > 0, 1.0, -1.0)
        response = -lab * sigmoid / (1.0 + np.exp(lab * sigmoid * score))
        ar = np.abs(response)
        g, h = response, ar * (sigmoid - ar)
        if w64 is not None:
            g, h = g * w64, h * w64
        return g.astype(np.float32), h.astype(np.float32)
    if objective == "multiclass":
        K, n = num_class, len(y)
        sk = score.reshape(K, n)
        wmax = sk[0].copy()
        for k in range(1, K):
            wmax = np.maximum(wmax, sk[k])
        wsum = np.zeros(n)
        for k in range(K):
            wsum = wsum + np.exp(sk[k] - wmax)
        factor = K / (K - 1.0)
        li = y.astype(np.int64)
        g, h = np.zeros((K, n), np.float32), np.zeros((K, n), np.float32)
        for k in range(K):
            pk = np.exp(sk[k] - wmax) / wsum
            gk, hk = np.where(li == k, pk - 1.0, pk), factor * pk * (1.0 - pk)
            if w64 is not None:
                gk, hk = gk * w64, hk * w64
            g[k], h[k] = gk, hk
        return g.ravel(), h.ravel()
    raise ValueError(objective)


def leaf_parent(tree):
    """the parent node of every leaf, from the child arrays (-1 for the leaf of a one-leaf tree)"""
    nl = tree["num_leaves"]
    lp = [-1] * nl
    for i in range(nl - 1):
        for c in (int(tree["left_child"][i]), int(tree["right_child"][i])):
            if c < 0:
                lp[~c] = i
    return lp


def calc_output(sg, sh, l1=0.0, l2=0.0, max_delta_step=0.0):
    """CalculateSplittedLeafOutput without constraints"""
    if l1 > 0:
        sg = float(np.sign(sg)) * max(0.0, abs(sg) - l1)
    ret = -sg / (sh + l2)
    if max_delta_step > 0 and abs(ret) > max_delta_step:
        ret = float(np.sign(ret)) * max_delta_step
    return ret


def leaf_sums(leaf, g, h, L, const_hessian):
    """per leaf (sum_g, sum_h without kEpsilon, rows) on the fixed-point grid of this class's g and h (over every rank's rows)"""
    qg = TC.quantized(np.asarray(g, np.float32))
    cnt = np.bincount(leaf, minlength=L)
    sg = np.zeros(L)
    np.add.at(sg, leaf, qg)
    if const_hessian:
        return sg, cnt.astype(np.float64), cnt
    sh = np.zeros(L)
    np.add.at(sh, leaf, TC.quantized(np.asarray(h, np.float32)))
    return sg, sh, cnt


def refit_tree(tree, leaf, g, h, const_hessian, decay, l1=0.0, l2=0.0, max_delta_step=0.0, path_smooth=0.0):
    """the new leaf values of one tree (parse_model dict with num_leaves, leaf_value, children and shrinkage)"""
    L = tree["num_leaves"]
    sg, sh, cnt = leaf_sums(leaf, g, h, L, const_hessian)
    lp = leaf_parent(tree)
    shrinkage = float(tree.get("shrinkage", 1.0))
    old = np.asarray(tree["leaf_value"], np.float64)
    out = np.zeros(L)
    for l in range(L):
        o = 0.0      # a leaf no row reaches
        if cnt[l] > 0:
            o = calc_output(float(sg[l]), KEPS + float(sh[l]), l1, l2, max_delta_step)
            if path_smooth > KEPS and l > 0:
                wgt = int(cnt[l]) / path_smooth
                o = o * wgt / (wgt + 1) + lp[l] / (wgt + 1)
        v = decay * float(old[l]) + (1.0 - decay) * (o * shrinkage)
        out[l] = v if abs(v) > ZERO else 0.0
    return out


def refit(trees, K, leaf, y, objective, decay, w=None, init_score=None, num_class=1, const_hessian=None, first_grads=None, **opts):
    """every tree's new leaf values and the final training scores (class-major [K * n]).  leaf: (n, models) int; opts: l1, l2,
    max_delta_step, path_smooth; const_hessian: default unweighted regression; first_grads: (g, h) to use at iteration 0 instead of
    NumPy's (the engine's own, read just before the refit)"""
    n = len(y)
    if const_hessian is None:
        const_hessian = objective == "regression" and w is None
    score = np.zeros(K * n) if init_score is None else np.asarray(init_score, np.float64).copy()
    new = []
    for it in range(len(trees) // K):
        g, h = gradients(objective, score, y, w, num_class) if it > 0 or first_grads is None else first_grads
        for k in range(K):
            m = it * K + k
            v = refit_tree(trees[m], leaf[:, m], g[k * n:(k + 1) * n], h[k * n:(k + 1) * n], const_hessian, decay, **opts)
            new.append(v)
            score[k * n:(k + 1) * n] += v[leaf[:, m]]
    return new, score
