"""The interaction-constraints restatement (interaction_ref.py, grown by tree_ref.py) on its own: the engine's set masks equal LightGBM's
branch rule, a single set of every feature grows the unconstrained tree, and constrained trees keep every path inside one set while
scanning as without constraints."""
import numpy as np
import pytest

import extra_trees_ref as X3
import interaction_ref as I
import split_scan_ref as ref
import tree_ref


def _random_constraints(rng, nf):
    k = int(rng.integers(1, 7))
    return [sorted(set(rng.choice(nf, int(rng.integers(1, nf + 1)), replace=True).tolist())) for _ in range(k)]


@pytest.mark.parametrize("seed", range(20))
def test_mask_equals_branch_rule(seed):
    """along random paths that only split on allowed features, the mask form allows exactly what GetByNode's branch rule allows"""
    rng = np.random.default_rng(seed)
    nf = int(rng.integers(2, 12))
    feats = list(range(nf))
    for _ in range(30):
        cons = _random_constraints(rng, nf)
        sets = I.sets_of(cons, nf)
        branch, mask = (), I.ALL
        for _ in range(8):
            want = I.allowed_by_branch(cons, branch, feats)
            assert I.allowed_by_mask(sets, mask, feats) == want, (cons, branch)
            if not want:
                break
            f = int(rng.choice(sorted(want)))
            branch, mask = branch + (f,), mask & sets[f]
            assert any(set(branch) <= set(c) for c in cons), "a reachable branch lies inside one set"


def test_feature_in_no_set_is_never_allowed():
    assert I.allowed_by_branch([[0, 1], [2]], (), range(4)) == {0, 1, 2}
    assert I.allowed_by_mask(I.sets_of([[0, 1], [2]], 4), I.ALL, range(4)) == {0, 1, 2}
    assert I.allowed_by_branch([[0, 1], [1, 2]], (1,), range(3)) == {0, 1, 2}
    assert I.allowed_by_branch([[0, 1], [1, 2]], (1, 0), range(3)) == {0, 1}


def _data(seed, n=4000):
    rng = np.random.default_rng(seed)
    bins = np.stack([rng.integers(0, 20, n), rng.integers(0, 20, n), rng.integers(0, 8, n), rng.integers(0, 12, n)], axis=1)
    y = np.sin(bins[:, 0] / 3.0) + 0.05 * bins[:, 1] * (bins[:, 2] % 3) + 0.2 * (bins[:, 3] > 5) + 0.3 * rng.standard_normal(n)
    g = np.round(-y * 1024) / 1024
    h = np.round(rng.uniform(0.5, 1.5, n) * 1024) / 1024
    feats = [ref.Feature(0, 20), ref.Feature(1, 20), ref.Feature(2, 8), ref.Feature(3, 12)]
    return bins, g, h, feats


_SHAPE = ("split_feature", "threshold_bin", "default_left", "left_child", "right_child", "leaf_value", "leaf_count", "split_gain")


def test_one_set_of_every_feature_is_unconstrained():
    bins, g, h, feats = _data(3)
    p = ref.Params(min_data_in_leaf=20)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 16, constraints=[[0, 1, 2, 3]])
    U = tree_ref.grow_tree(bins, g, h, feats, p, 16)
    assert T["num_leaves"] == U["num_leaves"] > 8
    for k in _SHAPE:
        assert T[k] == U[k], k
    E = tree_ref.grow_tree(bins, g, h, feats, p, 16, constraints=[[3, 2, 1, 0]], streams=X3.Streams(feats, 5))
    V = tree_ref.grow_tree(bins, g, h, feats, p, 16, streams=X3.Streams(feats, 5))
    for k in _SHAPE:
        assert E[k] == V[k], k


@pytest.mark.parametrize("cons", [[[0, 1], [2, 3]], [[0], [1], [2, 3]], [[0, 1, 2], [2, 3]], [[1, 2]]])
def test_paths_stay_inside_one_set(cons):
    bins, g, h, feats = _data(4)
    T = tree_ref.grow_tree(bins, g, h, feats, ref.Params(min_data_in_leaf=20), 16, constraints=cons)
    assert T["num_leaves"] > 2
    sets = I.sets_of(cons, 4)
    for branch, mask in zip(T["branches"], T["masks"]):
        assert any(set(branch) <= set(c) for c in cons), branch
        want = I.ALL
        for f in branch:
            want &= sets[f]
        assert mask == want
    assert set(T["split_feature"]) <= {f for c in cons for f in c}


def test_scans_and_flags_run_as_without_constraints():
    """the root scans every feature the tree samples, allowed or not, so the disallowed features' flags and extra_trees draws advance"""
    bins, g, h, feats = _data(5)
    p = ref.Params(min_data_in_leaf=20)
    s1 = X3.Streams(feats, 7)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 8, constraints=[[0]], streams=s1)
    assert set(T["split_feature"]) == {0}
    root_scans = T["rounds"][0][0][2]
    assert set(root_scans) == {0, 1, 2, 3}
    # every stream drew once per scan: the disallowed features' streams moved as the unconstrained tree's would
    s2 = X3.Streams(feats, 7)
    for rnd in T["rounds"]:
        for _, _, scans in rnd:
            for fi in scans:
                s2.rand[fi]._next()
    assert {f: s1.rand[f].x for f in s1.rand} == {f: s2.rand[f].x for f in s2.rand}
