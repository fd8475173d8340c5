"""NumPy restatement of LightGBM's prediction early stopping ([UPSTREAM] LightGBM 3.2 Predictor, GBDT::PredictRaw and
prediction_early_stop.cpp, from knowledge), over the decision rule of tree_walk_ref.

A predict call's parameter string may give pred_early_stop (bool, default false), pred_early_stop_freq (int, default 10) and
pred_early_stop_margin (double, default 10.0).  Early stopping applies when the key is true, the prediction is normal or raw, and the
model's objective is one whose predictions need not be accurate: binary, multiclass, multiclassova, lambdarank, rank_xendcg.  Then the
iterations of the range are summed one at a time, K trees each, in model order, and after every freq iterations a row whose margin
exceeds the threshold (strictly) walks no more trees.  The margin is 2|s| for one score and the largest minus the second largest score
(ties give 0) for K >= 2.  An averaged (rf) model still divides by the whole range's iteration count."""
import numpy as np

import tree_walk_ref as R

OBJECTIVES = ("binary", "multiclass", "multiclassova", "lambdarank", "rank_xendcg")


def applies(objective, predict_type, on=True):
    """whether early stopping runs for a model whose objective= header line is `objective`"""
    name = objective.split()[0] if objective else ""
    return bool(on) and predict_type in (0, 1) and name in OBJECTIVES


def margin(s):
    if len(s) == 1:
        return 2.0 * abs(float(s[0]))
    top = sorted((float(v) for v in s), reverse=True)
    return top[0] - top[1]


def raw_scores(trees, X, K=1, start_iteration=0, num_iteration=-1, freq=10, margin_threshold=10.0, average=False):
    """([rows][K] raw scores, [rows] iterations walked).  freq=None walks every tree (early stopping off)."""
    t0, t1 = R.iteration_range(len(trees), K, start_iteration, num_iteration)
    iters = (t1 - t0) // K
    out = np.zeros((len(X), K))
    walked = np.zeros(len(X), dtype=np.int64)
    for i, x in enumerate(X):
        s = [0.0] * K
        c = 0
        n = 0
        for it in range(t0 // K, t1 // K):
            for k in range(K):
                tree = trees[it * K + k]
                s[k] += float(tree["leaf_value"][R.leaf_index(tree, x)])
            n += 1
            c += 1
            if freq is not None and c == freq:
                if margin(s) > margin_threshold:
                    break
                c = 0
        out[i] = s
        walked[i] = n
    if average and iters > 0:
        out /= iters
    return out, walked
