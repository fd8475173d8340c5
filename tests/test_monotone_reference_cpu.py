"""The monotone-constraints restatement (monotone_ref.py) on its own: the clamp and the given-output gain, direction rejection in both
numerical passes, the leaf bounds, the penalty factor, and a histogram where the constraint changes the chosen threshold."""
import math

import numpy as np
import pytest

import monotone_ref as M
import split_scan_ref as ref
import tree_ref

INF = math.inf


def test_clamp_and_given_output_gain():
    p = ref.Params()
    # unclamped: the given-output gain at the optimum equals GetLeafGain
    g, h = -6.0, 3.0
    out = M.constrained_output(g, h, p, 0.0, -INF, INF)
    assert out == 2.0
    assert M.gain_given_output(g, h, p, 0.0, out) == pytest.approx(ref.leaf_gain(g, h, p, 0.0), rel=1e-15)
    # clamped to the bound: -(2 g out + h out^2)
    out = M.constrained_output(g, h, p, 0.0, -INF, 0.5)
    assert out == 0.5
    assert M.gain_given_output(g, h, p, 0.0, out) == -(2.0 * -6.0 * 0.5 + 3.0 * 0.25)
    assert M.constrained_output(g, h, p, 0.0, 2.5, INF) == 2.5
    # lambda_l1 soft-thresholds g in both the output and the gain
    p1 = ref.Params(lambda_l1=1.0, lambda_l2=1.0)
    out = M.constrained_output(g, h, p1, 1.0, -INF, 1.0)
    assert out == 1.0                                  # -(-5) / 4 = 1.25, clamped
    assert M.gain_given_output(g, h, p1, 1.0, out) == -(2.0 * -5.0 * 1.0 + 4.0 * 1.0)
    # max_delta_step applies before the bounds
    pm = ref.Params(max_delta_step=0.75)
    assert M.constrained_output(g, h, pm, 0.0, -INF, INF) == 0.75
    assert M.constrained_output(g, h, pm, 0.0, 1.0, INF) == 1.0
    assert M.constrained_output(g, h, pm, 0.0, -INF, 0.25) == 0.25


def test_direction_rejection():
    p = ref.Params()
    # left output 1, right output -1
    lg, lh, rg, rh = -2.0, 2.0, 3.0, 3.0
    assert M.split_gain(lg, lh, rg, rh, p, 0.0, -INF, INF, +1) == 0.0
    assert M.split_gain(lg, lh, rg, rh, p, 0.0, -INF, INF, -1) > 0.0
    assert M.split_gain(lg, lh, rg, rh, p, 0.0, -INF, INF, 0) == M.split_gain(lg, lh, rg, rh, p, 0.0, -INF, INF, -1)
    # bounds that squeeze both outputs to the same value: no violation, gain at the clamped outputs
    assert M.split_gain(lg, lh, rg, rh, p, 0.0, 0.0, 0.0, +1) == 0.0 + 0.0


def _hist(values_g, values_h):
    return np.asarray(values_g, np.float64), np.asarray(values_h, np.float64)


@pytest.mark.parametrize("mono", [+1, -1])
def test_direction_rejected_in_both_numerical_passes(mono):
    """bins 1..4 plus a NaN bin: gradients fall with the bin (outputs rise), so only +1 keeps every candidate of either pass"""
    nb = 6
    hg, hh = _hist([0, 40, 20, -20, -40, 10], [0, 40, 40, 40, 40, 40])
    n = 200
    sg, sh = float(hg.sum()), float(hh.sum())
    p = ref.Params(min_data_in_leaf=10)
    r0 = ref.find_best_numerical(hg, hh, nb, 2, 1, sg, sh, n, p)
    passes = {c[5][0] for c in r0.candidates}
    assert passes == {"rev", "fwd"}
    r = M.find_best_numerical(hg, hh, nb, 2, 1, sg, sh, n, p, 0, (-INF, INF), mono)
    for c in r.candidates:
        lo = M.constrained_output(c[1], c[2], p, 0.0, -INF, INF)
        ro = M.constrained_output(c[3], c[4], p, 0.0, -INF, INF)
        breaks = lo > ro if mono > 0 else lo < ro
        assert (c[0] == 0.0) == breaks, c
    kept = [c for c in r.candidates if c[0] > r.shift]
    assert {c[5][0] for c in r.candidates if c[0] == 0.0} <= passes
    if mono > 0:
        assert kept and r.gain > 0
    else:
        assert all(c[0] == 0.0 for c in r.candidates if c[5][0] == "rev")
        assert any(c[0] == 0.0 for c in r.candidates if c[5][0] == "fwd")


def test_bounds_update():
    b = (-INF, INF)
    l, r = M.child_bounds(b, +1, False, 1.0, 3.0)
    assert l == (-INF, 2.0) and r == (2.0, INF)
    l, r = M.child_bounds(b, -1, False, 3.0, 1.0)
    assert l == (2.0, INF) and r == (-INF, 2.0)
    # a non-monotone split inherits the parent's bounds unchanged
    assert M.child_bounds((0.5, 1.5), 0, False, 0.6, 1.4) == ((0.5, 1.5), (0.5, 1.5))
    # a categorical split never narrows them
    assert M.child_bounds((0.5, 1.5), +1, True, 0.6, 1.4) == ((0.5, 1.5), (0.5, 1.5))
    # narrowing keeps the tighter of the old bound and mid
    l, r = M.child_bounds((0.0, 1.0), +1, False, 0.2, 0.6)
    assert l == (0.0, 0.4) and r == (0.4, 1.0)
    l, r = M.child_bounds((0.0, 1.0), +1, False, 0.5, 2.5)
    assert l == (0.0, 1.0) and r == (1.5, 1.0)


@pytest.mark.parametrize("penalty", [0.0, 0.5, 1.0, 2.5, 10.0])
def test_penalty_factor(penalty):
    eps = float(np.float32(1e-15))
    for d in range(5):
        f = M.penalty_factor(d, penalty)
        if penalty >= d + 1:
            want = eps
        elif penalty <= 1:
            want = 1.0 - penalty / 2.0 ** d + eps
        else:
            want = 1.0 - 2.0 ** (penalty - 1.0 - d) + eps
        assert f == want
        assert 0 < f <= 1.0 + 2 * eps
    # spot values
    assert M.penalty_factor(0, 0.0) == 1.0 + eps
    assert M.penalty_factor(1, 0.5) == 0.75 + eps
    assert M.penalty_factor(0, 1.0) == eps
    assert M.penalty_factor(2, 2.5) == 1.0 - 2.0 ** -0.5 + eps
    assert M.penalty_factor(4, 10.0) == eps


def test_constraint_changes_the_threshold():
    """a histogram whose best unconstrained threshold breaks +1, while a later one keeps it"""
    nb = 5
    # bin outputs -g/h = [., 2, -1, -1, 1.5]: thresholds 1 (best, 2 | -1/6) and 2 (1/2 | 1/4) break +1, threshold 3 (0 | 1.5) keeps it
    hg, hh = _hist([0, -60, 30, 30, -45], [0, 30, 30, 30, 30])
    n, sg, sh = 120, float(hg.sum()), float(hh.sum())
    p = ref.Params(min_data_in_leaf=10)
    free = ref.find_best_numerical(hg, hh, nb, 0, 0, sg, sh, n, p)
    up = M.find_best_numerical(hg, hh, nb, 0, 0, sg, sh, n, p, 0, (-INF, INF), +1)
    down = M.find_best_numerical(hg, hh, nb, 0, 0, sg, sh, n, p, 0, (-INF, INF), -1)
    assert free.threshold == 1 and down.threshold == 1 and up.threshold == 3
    assert up.gain == pytest.approx(45.0 ** 2 / 30 - 45.0 ** 2 / 120, rel=1e-12)
    assert up.gain > 0 and up.threshold != free.threshold
    lo = M.constrained_output(up.left_g, up.left_h, p, 0.0, -INF, INF)
    ro = M.constrained_output(sg - up.left_g, sh + 2 * ref.K_EPS - up.left_h, p, 0.0, -INF, INF)
    assert lo <= ro


def test_all_zero_list_uses_the_given_output_gain():
    """an all-zero list keeps the unconstrained splits, at gains computed from the outputs (equal up to rounding)"""
    rng = np.random.default_rng(1)
    nb = 12
    hg = np.round(rng.normal(0, 20, nb) * 1024) / 1024
    hh = np.round(rng.uniform(5, 30, nb) * 1024) / 1024
    hg[0] = hh[0] = 0
    n, sg, sh = int(hh.sum()), float(hg.sum()), float(hh.sum())
    p = ref.Params(min_data_in_leaf=5)
    free = ref.find_best_numerical(hg, hh, nb, 0, 0, sg, sh, n, p)
    zero = M.find_best_numerical(hg, hh, nb, 0, 0, sg, sh, n, p, 0, (-INF, INF), 0)
    assert zero.threshold == free.threshold
    assert zero.gain == pytest.approx(free.gain, rel=1e-12)


def test_grow_tree_is_monotone():
    """a whole restated tree under +1 on feature 0 and -1 on feature 1: leaf values follow the directions along each feature"""
    rng = np.random.default_rng(2)
    n = 4000
    bins = np.stack([rng.integers(0, 20, n), rng.integers(0, 20, n), rng.integers(0, 8, n)], axis=1)
    y = np.sin(bins[:, 0] / 3.0) - 0.05 * bins[:, 1] ** 1.5 + 0.3 * (bins[:, 2] % 2) + 0.3 * rng.standard_normal(n)
    g = np.round(-y * 1024) / 1024
    h = np.ones(n)
    feats = [ref.Feature(0, 20), ref.Feature(1, 20), ref.Feature(2, 8)]
    p = ref.Params(min_data_in_leaf=20)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 16, mono=[1, -1, 0], penalty=0.0)
    assert T["num_leaves"] > 4

    def leaf_of(row):
        node = 0
        while True:
            f, t = T["split_feature"][node], T["threshold_bin"][node]
            nxt = T["left_child"][node] if row[f] <= t else T["right_child"][node]
            if nxt < 0:
                return ~nxt
            node = nxt

    base = bins[rng.integers(0, n, 50)]
    for f, sign in ((0, 1), (1, -1)):
        for row in base:
            vals = []
            for b in range(20):
                r = row.copy(); r[f] = b
                vals.append(T["leaf_value"][leaf_of(r)])
            d = np.diff(vals) * sign
            assert (d >= 0).all(), (f, vals)
    for lv, (lo, hi) in zip(T["leaf_value"], T["bounds"]):
        assert lo <= lv <= hi
