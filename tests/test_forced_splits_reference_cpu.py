"""The forced-splits restatement (forced_splits_ref.py) on its own: the threshold evaluation against brute-force sums, the plan's order and
leaf ids, and each way the forced phase ends."""
import math

import numpy as np
import pytest

import forced_splits_ref as FS
import split_scan_ref as ref


def _rows(seed, n=400, num_bin=12, const_h=True):
    """with constant hessians the counts rebuilt from them are the true row counts"""
    rng = np.random.default_rng(seed)
    col = rng.integers(0, num_bin, n)
    g = np.round(rng.standard_normal(n) * 1024) / 1024
    h = np.ones(n) if const_h else rng.integers(512, 1536, n) / 1024
    return col, g, h


@pytest.mark.parametrize("b", [0, 3, 9])
@pytest.mark.parametrize("missing_type", [0, 2])
def test_numerical_sums_match_brute_force(b, missing_type):
    num_bin = 12
    col, g, h = _rows(b + 10 * missing_type, num_bin=num_bin)
    f = ref.Feature(0, num_bin, missing_type)
    hg, hh = np.bincount(col, g, num_bin), np.bincount(col, h, num_bin)
    p = ref.Params(min_data_in_leaf=1000)      # ignored by a forced node
    s, _, _ = FS.evaluate(hg, hh, f, b, math.fsum(g), math.fsum(h), len(g), p)
    nan_bin = num_bin - 1 if missing_type == 2 else None
    right = (col > b) & (col != nan_bin)
    assert s is not None
    assert s.threshold == b and s.default_left and not s.is_cat
    assert math.isclose(s.left_g, g[~right].sum(), rel_tol=1e-12, abs_tol=1e-9)
    assert math.isclose(s.left_h - ref.K_EPS, h[~right].sum(), rel_tol=1e-12)
    assert s.left_count == int((~right).sum())
    left = ref.goes_left(col, f, s)
    assert (left == ~right).all()      # NaN goes left with the other bins at or below the threshold


def test_categorical_left_is_the_category():
    col, g, h = _rows(3, num_bin=6)
    f = ref.Feature(0, 6, 0, 0, True)
    hg, hh = np.bincount(col, g, 6), np.bincount(col, h, 6)
    s, _, _ = FS.evaluate(hg, hh, f, 4, math.fsum(g), math.fsum(h), len(g), ref.Params())
    assert s is not None and s.is_cat and s.cat_bins == (4,) and not s.default_left
    assert s.left_count == int((col == 4).sum())
    assert math.isclose(s.left_g, g[col == 4].sum(), rel_tol=1e-12, abs_tol=1e-12)
    for bad in (0, 6, 9):      # bin 0 (rare or unseen categories) and bins the feature does not have
        assert FS.evaluate(hg, hh, f, bad, math.fsum(g), math.fsum(h), len(g), ref.Params())[0] is None


def test_unseen_category_maps_to_bin_zero():
    f = ref.Feature(3, 4, 0, 0, True)
    b2c = [-1, 7, 2, 5]
    assert FS.value_to_bin(5, f, None, b2c) == 3
    assert FS.value_to_bin(6, f, None, b2c) == 0
    assert FS.value_to_bin(-1, f, None, b2c) == 0


def test_numerical_value_to_bin():
    f = ref.Feature(0, 5, 2)
    ub = np.array([1.0, 2.0, 3.0, np.inf, np.nan])
    assert [FS.value_to_bin(v, f, ub, None) for v in (0.5, 1.0, 1.5, 3.0, 99.0)] == [0, 0, 1, 2, 3]


def test_min_gain_shift():
    col, g, h = _rows(5, const_h=False)
    f = ref.Feature(0, 12, 0)
    hg, hh = np.bincount(col, g, 12), np.bincount(col, h, 12)
    s, _, (gain, shift) = FS.evaluate(hg, hh, f, 5, math.fsum(g), math.fsum(h), len(g), ref.Params())
    assert s is not None and s.gain == gain - shift > 0
    # a min_gain_to_split just above the split's gain over the parent's makes the node invalid
    p = ref.Params(min_gain_to_split=gain - ref.leaf_gain(math.fsum(g), math.fsum(h) + 2 * ref.K_EPS, ref.Params(), 0.0) + 1e-6)
    assert FS.evaluate(hg, hh, f, 5, math.fsum(g), math.fsum(h), len(g), p)[0] is None
    # the whole leaf on one side never beats the leaf's own gain by more than rounding
    s_all, _, (g_all, sh_all) = FS.evaluate(hg, hh, f, 11, math.fsum(g), math.fsum(h), len(g), ref.Params(min_gain_to_split=1e-9))
    assert s_all is None


def _node(f, t, left=None, right=None, **extra):
    d = dict(feature=f, threshold=t, **extra)
    if left is not None:
        d["left"] = left
    if right is not None:
        d["right"] = right
    return d


def test_leaf_ids_balanced():
    plan = _node(0, 1, _node(1, 2, _node(2, 3), _node(2, 4)), _node(1, 5, _node(2, 6), _node(2, 7)))
    nodes = FS.flatten(plan)
    assert [n["threshold"] for n in nodes] == [1, 2, 5, 3, 4, 6, 7]
    assert [n["leaf"] for n in nodes] == [0, 0, 1, 0, 2, 1, 3]
    assert [(n["left"], n["right"]) for n in nodes] == [(1, 2), (3, 4), (5, 6), (-1, -1), (-1, -1), (-1, -1), (-1, -1)]


def test_leaf_ids_chain_and_left_only():
    chain = _node(0, 1, right=_node(1, 2, right=_node(2, 3)))
    assert [n["leaf"] for n in FS.flatten(chain)] == [0, 1, 2]
    left_only = _node(0, 1, left=_node(1, 2, left=_node(2, 3)))
    assert [n["leaf"] for n in FS.flatten(left_only)] == [0, 0, 0]


def test_children_without_feature_or_threshold_and_unknown_keys_are_ignored():
    plan = _node(0, 1, left={"feature": 1}, right={"threshold": 2, "left": _node(2, 3)}, comment="x")
    assert len(FS.flatten(plan)) == 1


def _grid_data(seed, n=3000):
    rng = np.random.default_rng(seed)
    bins = np.stack([rng.integers(0, 10, n), rng.integers(0, 8, n), rng.integers(0, 6, n)], axis=1)
    g = np.round((-1.0 * (bins[:, 0] > 4) - 0.5 * (bins[:, 1] > 2) + 0.3 * rng.standard_normal(n)) * 1024) / 1024
    h = np.ones(n)
    feats = [ref.Feature(0, 10), ref.Feature(1, 8), ref.Feature(2, 6)]
    return bins, g, h, feats


def _nodes(plan):
    return [dict(n, bin=int(n["threshold"])) for n in FS.flatten(plan)]


def test_phase_runs_out_of_plan_then_grows_freely():
    bins, g, h, feats = _grid_data(1)
    nodes = _nodes(_node(2, 2, _node(1, 5)))
    T = FS.grow_tree(bins, g, h, feats, ref.Params(), 8, nodes)
    assert T["forced"] == [0, 1] and T["phase_end"] == "plan"
    assert T["split_feature"][:2] == [2, 1] and T["threshold_bin"][:2] == [2, 5]
    assert T["num_leaves"] == 8
    assert not FS.undecided(T)


def test_phase_ends_at_an_invalid_node():
    bins, g, h, feats = _grid_data(2)
    # node 1 asks for a split of a categorical-free feature at its last bin: everything goes left, which never beats the leaf's gain
    nodes = _nodes(_node(0, 4, _node(1, 7), _node(2, 1)))
    T = FS.grow_tree(bins, g, h, feats, ref.Params(min_gain_to_split=1e-6), 6, nodes)
    assert T["forced"] == [0] and T["phase_end"] == "invalid"
    assert T["evals"][1][0] is None and T["evals"][2][0] is not None


def test_phase_ends_at_an_unscanned_leaf():
    bins, g, h, feats = _grid_data(3)
    nodes = _nodes(_node(0, 4, _node(1, 2, _node(2, 3))))
    T = FS.grow_tree(bins, g, h, feats, ref.Params(), 8, nodes, max_depth=2)
    assert T["forced"] == [0, 1] and T["phase_end"] == "unscanned"


def test_phase_ends_when_the_tree_is_full():
    bins, g, h, feats = _grid_data(4)
    nodes = _nodes(_node(0, 4, _node(1, 2, _node(2, 1), _node(2, 3)), _node(1, 5)))
    T = FS.grow_tree(bins, g, h, feats, ref.Params(), 3, nodes)
    assert T["forced"] == [0, 1] and T["phase_end"] == "full" and T["num_leaves"] == 3
