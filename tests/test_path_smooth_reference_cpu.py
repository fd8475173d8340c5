"""The path-smoothing restatement (path_smooth_ref.py) on its own: the smoothed output and its operation order, the root's identity,
the kEpsilon threshold, the limit of a very large path_smooth, smoothing before the monotone clamp, the smoothed min_gain_shift, the
min_data_in_leaf rule and the estimator's parameter string."""
import math

import numpy as np
import pytest

import monotone_ref as M
import path_smooth_ref as PS
import split_scan_ref as ref
import tree_ref

INF = math.inf


def _data(seed, n=3000):
    rng = np.random.default_rng(seed)
    bins = np.stack([rng.integers(0, 30, n), rng.integers(0, 8, n), rng.integers(0, 3, n), rng.integers(0, 12, n)], axis=1)
    g = np.round((0.05 * bins[:, 0] - (bins[:, 1] > 3) + 0.7 * (bins[:, 2] == 1) + 0.3 * rng.standard_normal(n)) * 1024) / 1024
    h = rng.integers(512, 1536, n) / 1024
    feats = [ref.Feature(0, 30), ref.Feature(1, 8, missing_type=2), ref.Feature(2, 3, is_cat=True), ref.Feature(3, 12, is_cat=True)]
    return bins, g, h, feats


def test_smoothed_output_formula_and_order():
    p = ref.Params()
    g, h, n, parent, s = -6.0, 3.0, 7, 0.25, 3.0
    w = n / s
    want = 2.0 * w / (w + 1) + parent / (w + 1)
    assert PS.smoothed_output(g, h, n, parent, p, 0.0, s) == want
    # upstream's order, not the algebraically equal weighted mean: these differ in the last bits for some inputs
    hits = 0
    for n in range(1, 400):
        w = n / s
        got = PS.smoothed_output(g, h, n, parent, p, 0.0, s)
        assert got == 2.0 * w / (w + 1) + parent / (w + 1)
        hits += got != (2.0 * n + parent * s) / (n + s)
    assert hits > 0
    # L1, l2 and max_delta_step apply before the smoothing
    p1 = ref.Params(lambda_l1=1.0, max_delta_step=1.0)
    w = n / s
    assert PS.smoothed_output(g, h, n, parent, p1, 1.0, s) == 1.0 * w / (w + 1) + parent / (w + 1)


def test_smoothing_off_at_and_below_kepsilon():
    p = ref.Params()
    for s in (0.0, 1e-16, PS.K_EPS_F):
        assert not PS.active(s)
        assert PS.smoothed_output(-6.0, 3.0, 5, 100.0, p, 0.0, s) == 2.0
        assert PS.leaf_gain(-6.0, 3.0, 5, 100.0, p, 0.0, s) == ref.leaf_gain(-6.0, 3.0, p, 0.0)
    assert PS.active(np.nextafter(PS.K_EPS_F, 1.0))


def test_root_identity():
    """the root's parent_output is its own output, so smoothing it gives it back"""
    _, g, h, _ = _data(0)
    p = ref.Params(lambda_l2=1.5)
    root = PS.root_output(math.fsum(g), math.fsum(h), p)
    assert root == ref.calc_output(math.fsum(g), math.fsum(h), p, 1.5)
    for s in (0.5, 10.0, 1e6):
        assert PS.smoothed_output(math.fsum(g), math.fsum(h), len(g), root, p, 1.5, s) == pytest.approx(root, rel=1e-15)


def test_min_gain_shift_is_smoothed_and_never_clamped():
    bins, g, h, feats = _data(1)
    p = ref.Params()
    sg, sh, n = math.fsum(g), math.fsum(h), len(g)
    parent = 0.2
    col = bins[:, 0]
    hg, hh = np.bincount(col, weights=g, minlength=30), np.bincount(col, weights=h, minlength=30)
    r = PS.find_best_numerical(hg, hh, 30, 0, 0, sg, sh, n, p, 0, 10.0, parent)
    assert r.shift == PS.leaf_gain(sg, sh + 2 * ref.K_EPS, n, parent, p, 0.0, 10.0)
    assert r.shift != ref.leaf_gain(sg, sh + 2 * ref.K_EPS, p, 0.0)
    rc = PS.find_best_numerical(hg, hh, 30, 0, 0, sg, sh, n, p, 0, 10.0, parent, bounds=(-0.001, 0.001))
    assert rc.shift == r.shift


@pytest.mark.parametrize("s", [0.0, 1e-16])
def test_off_grows_the_plain_trees(s):
    bins, g, h, feats = _data(2)
    p = ref.Params()
    for extra in ({}, dict(mono=[1, -1, 0, 0], penalty=0.5)):
        a = PS.grow_tree(bins, g, h, feats, p, 12, smooth=s, **extra)
        b = tree_ref.grow_tree(bins, g, h, feats, p, 12, **extra)
        for k in ("split_feature", "threshold_bin", "cat_bins", "leaf_value", "internal_value", "leaf_count", "split_gain"):
            assert a[k] == b[k], k


KEYS = ("split_feature", "threshold_bin", "default_left", "cat_bins", "split_gain", "left_child", "right_child", "internal_value",
        "internal_weight", "internal_count", "leaf_value", "leaf_weight", "leaf_count", "bounds", "masks", "branches", "draws",
        "scanned_counts", "scan_masks")


@pytest.mark.parametrize("s", [0.0, 1e-16])
def test_off_is_tree_ref_with_every_option(s):
    """path_smooth_ref.grow_tree repeats tree_ref.grow_tree's rounds: with smoothing off it grows tree_ref's tree, key for key, with
    each option the smoothed tests combine (fresh streams and samplers on both sides)"""
    import bynode_ref as B
    import extra_trees_ref as X3
    bins, g, h, feats = _data(7)
    p = ref.Params(min_data_per_group=20, cat_smooth=5)
    options = [dict(), dict(used={0, 2, 3}), dict(mono=[1, -1, 0, 0], penalty=1.5), dict(constraints=[[0, 2], [1, 2, 3]]),
               dict(max_depth=2), lambda: dict(streams=X3.Streams(feats, 4)), lambda: dict(sampler=B.ColSampler(feats, 1.0, 0.5))]
    for opt in options:
        a = PS.grow_tree(bins, g, h, feats, p, 12, smooth=s, **(opt() if callable(opt) else opt))
        b = tree_ref.grow_tree(bins, g, h, feats, p, 12, **(opt() if callable(opt) else opt))
        assert a["num_leaves"] > 2
        for k in KEYS:
            assert a[k] == b[k], (opt, k)


def test_small_smoothing_is_close_to_the_plain_tree_and_changes_it():
    bins, g, h, feats = _data(3)
    p = ref.Params()
    plain = tree_ref.grow_tree(bins, g, h, feats, p, 12)
    tiny = PS.grow_tree(bins, g, h, feats, p, 12, smooth=1e-9)
    assert tiny["split_feature"] == plain["split_feature"] and tiny["threshold_bin"] == plain["threshold_bin"]
    np.testing.assert_allclose(tiny["leaf_value"], plain["leaf_value"], rtol=1e-9)
    big = PS.grow_tree(bins, g, h, feats, p, 12, smooth=10.0)
    assert big["leaf_value"] != plain["leaf_value"]


def test_very_large_smoothing_gives_every_leaf_the_root_output():
    bins, g, h, feats = _data(4)
    p = ref.Params()
    root = PS.root_output(math.fsum(g), math.fsum(h), p)
    T = PS.grow_tree(bins, g, h, feats, p, 12, smooth=1e12)
    assert T["num_leaves"] > 1
    np.testing.assert_allclose(T["leaf_value"], root, rtol=1e-6)
    np.testing.assert_allclose(T["internal_value"][1:], root, rtol=1e-6)


def test_children_outputs_use_the_estimated_counts():
    bins, g, h, feats = _data(5)
    p = ref.Params()
    T = PS.grow_tree(bins, g, h, feats, p, 2, smooth=5.0)
    s = T["picks"][0][0][1]
    root = PS.root_output(math.fsum(g), math.fsum(h), p)
    assert T["leaf_value"][0] == PS.smoothed_output(s.left_g, s.left_h, s.left_count, root, p, s.l2, 5.0)
    sh2 = math.fsum(h) + 2 * ref.K_EPS
    assert T["leaf_value"][1] == PS.smoothed_output(math.fsum(g) - s.left_g, sh2 - s.left_h, len(g) - s.left_count, root, p, s.l2, 5.0)


def test_smoothing_before_the_monotone_clamp():
    p = ref.Params()
    g, h, n, parent, s = -6.0, 3.0, 3, -1.0, 3.0          # unsmoothed 2.0, smoothed 0.5
    assert PS.output(g, h, n, parent, p, 0.0, s, -INF, INF) == 0.5
    assert PS.output(g, h, n, parent, p, 0.0, s, -INF, 1.0) == 0.5        # the clamp of the unsmoothed output would give 1.0 -> 0.0
    assert PS.output(g, h, n, parent, p, 0.0, s, 0.75, INF) == 0.75
    assert M.clamp(PS.smoothed_output(g, h, n, parent, p, 0.0, s), -INF, 1.0) == 0.5
    # the given-output gain at the clamped output; 0 when the outputs break the direction
    gain = PS.split_gain(g, h, 6.0, 3.0, n, n, parent, p, 0.0, s, -INF, INF, 1)
    assert gain == 0.0                                    # left 0.5 > right -(2 + 1) / 2 = -1.5 under +1
    gain = PS.split_gain(g, h, 6.0, 3.0, n, n, parent, p, 0.0, s, -INF, INF, -1)
    assert gain == M.gain_given_output(g, h, p, 0.0, 0.5) + M.gain_given_output(6.0, 3.0, p, 0.0, -1.5)


def test_monotone_trees_stay_monotone_when_smoothed():
    bins, g, h, feats = _data(6)
    p = ref.Params()
    T = PS.grow_tree(bins, g, h, feats, p, 16, mono=[1, 0, 0, 0], penalty=0.0, smooth=10.0)
    for (lo, hi), v in zip(T["bounds"], T["leaf_value"]):
        assert lo - 1e-12 <= v <= hi + 1e-12


def test_min_data_in_leaf_rule():
    assert PS.min_data_in_leaf(1.0, 0) == 2 and PS.min_data_in_leaf(1.0, 1) == 2
    assert PS.min_data_in_leaf(1.0, 2) == 2 and PS.min_data_in_leaf(1.0, 20) == 20
    assert PS.min_data_in_leaf(0.0, 1) == 1 and PS.min_data_in_leaf(1e-16, 0) == 0


def test_estimator_parameter_string():
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    df = Frame({"features": np.zeros((10, 5)), "label": np.zeros(10)})
    assert LightGBMRegressor(pathSmooth=10.0).getTrainParams(1, df).to_string().endswith("path_smooth=10.0 ")
    assert LightGBMRegressor(pathSmooth=1e-16).getTrainParams(1, df).to_string().endswith("path_smooth=1.0E-16 ")
    assert "path_smooth" not in LightGBMRegressor().getTrainParams(1, df).to_string()
    assert "path_smooth" not in LightGBMRegressor(pathSmooth=0.0).getTrainParams(1, df).to_string()
    assert LightGBMRegressor(pathSmooth=0.0).getTrainParams(1, df).to_string() == LightGBMRegressor().getTrainParams(1, df).to_string()
