"""The NumPy restatement of LGBM_BoosterRefit (refit_ref) on its own: l2 at decay 0 against a brute-force per-leaf mean, decay 1, an empty
leaf, a one-leaf tree, path smoothing toward the parent's node index, L1 with max_delta_step, and the score chain; and the JNI shim's
LGBM_1BoosterRefit native."""
import os

import numpy as np
import pytest

import refit_ref as R

GRID = 1.0 / 1024


def _tree(leaf_value, shrinkage=0.1):
    """a three-leaf tree: node 0 splits into leaf 0 and node 1, node 1 into leaves 1 and 2"""
    return dict(num_leaves=3, leaf_value=np.asarray(leaf_value, np.float64), left_child=np.array([-1, -2]), right_child=np.array([1, -3]),
                shrinkage=str(shrinkage))


def _rows(seed, n=3000, L=3):
    rng = np.random.default_rng(seed)
    leaf = rng.integers(0, L, n)
    y = (np.round(rng.standard_normal(n) / GRID) * GRID).astype(np.float32)      # on the grid: every sum is exact
    return leaf, y


def test_leaf_parent_from_children():
    assert R.leaf_parent(_tree([0, 0, 0])) == [0, 1, 1]
    assert R.leaf_parent(dict(num_leaves=1, left_child=[], right_child=[])) == [-1]


def test_l2_decay_zero_is_the_leaf_mean_of_the_residuals():
    leaf, y = _rows(1)
    t = _tree([0.3, -0.2, 0.7], shrinkage=0.1)
    new, score = R.refit([t], 1, leaf[:, None], y, "regression", 0.0)
    for l in range(3):
        want = float(np.mean(y[leaf == l].astype(np.float64))) * 0.1
        assert new[0][l] == pytest.approx(want, rel=1e-12)
    np.testing.assert_allclose(score, new[0][leaf], rtol=0, atol=0)


def test_decay_one_keeps_the_leaves():
    leaf, y = _rows(2)
    t = _tree([0.3, -0.2, 0.7])
    new, _ = R.refit([t], 1, leaf[:, None], y, "regression", 1.0)
    assert np.array_equal(new[0], t["leaf_value"])


def test_empty_leaf_gets_output_zero():
    leaf, y = _rows(3)
    leaf[leaf == 2] = 1
    t = _tree([0.3, -0.2, 0.7])
    new, _ = R.refit([t], 1, leaf[:, None], y, "regression", 0.5)
    assert new[0][2] == 0.5 * 0.7
    new, _ = R.refit([t], 1, leaf[:, None], y, "regression", 0.5, path_smooth=3.0)      # no smoothing toward the parent either
    assert new[0][2] == 0.5 * 0.7


def test_one_leaf_tree():
    _, y = _rows(4)
    t = dict(num_leaves=1, leaf_value=np.array([0.25]), left_child=np.array([], int), right_child=np.array([], int), shrinkage="1")
    new, score = R.refit([t], 1, np.zeros((len(y), 1), int), y, "regression", 0.25)
    out = -float(np.sum(-y.astype(np.float64))) / (R.KEPS + len(y))
    assert new[0][0] == pytest.approx(0.25 * 0.25 + 0.75 * out, rel=1e-12)
    assert np.all(score == new[0][0])


def test_smoothing_goes_toward_the_parent_node_index():
    leaf, y = _rows(5)
    t = _tree([0.0, 0.0, 0.0], shrinkage=1.0)
    ps = 7.0
    new, _ = R.refit([t], 1, leaf[:, None], y, "regression", 0.0, path_smooth=ps)
    for l, parent in ((0, None), (1, 1), (2, 1)):
        r = y[leaf == l].astype(np.float64)
        o = -float(np.sum(-r)) / (R.KEPS + len(r))
        if parent is not None:
            w = len(r) / ps
            o = o * w / (w + 1) + parent / (w + 1)
        assert new[0][l] == pytest.approx(o, rel=1e-12)
    # leaf 0 is not smoothed even though its parent is node 0; leaves 1 and 2 are pulled toward 1.0, the index of node 1
    assert abs(new[0][1] - 1.0) < abs(np.mean(y[leaf == 1]) - 1.0)


def test_l1_and_max_delta_step():
    leaf, y = _rows(6)
    t = _tree([0.0, 0.0, 0.0], shrinkage=1.0)
    new, _ = R.refit([t], 1, leaf[:, None], (y * 100).astype(np.float32), "regression", 0.0, l1=5.0, l2=2.0, max_delta_step=0.05)
    for l in range(3):
        sg = float(np.sum(-(y[leaf == l] * 100).astype(np.float32).astype(np.float64)))
        sh = R.KEPS + np.count_nonzero(leaf == l)
        o = -np.sign(sg) * max(0.0, abs(sg) - 5.0) / (sh + 2.0)
        o = np.sign(o) * min(abs(o), 0.05)
        assert new[0][l] == pytest.approx(o, rel=1e-12)


def test_score_chain_feeds_the_next_iteration():
    """the second tree's gradients are taken at the scores the first refit tree left"""
    leaf, y = _rows(7)
    t = [_tree([0.1, 0.2, 0.3], 1.0), _tree([0.0, 0.0, 0.0], 1.0)]
    lp = np.stack([leaf, leaf], axis=1)
    new, score = R.refit(t, 1, lp, y, "regression", 0.0)
    # at decay 0 with shrinkage 1 the first tree already fits the leaf means, so the second one has almost nothing left
    assert np.all(np.abs(new[1]) < 1e-6)      # float32 gradients leave a residue
    np.testing.assert_allclose(score, new[0][leaf] + new[1][leaf], rtol=0, atol=0)


@pytest.mark.parametrize("objective,K", [("binary", 1), ("multiclass", 3)])
def test_gradients_match_the_pinned_formulas(objective, K):
    rng = np.random.default_rng(8)
    n = 200
    y = rng.integers(0, max(K, 2), n).astype(np.float32)
    s = rng.standard_normal(K * n)
    g, h = R.gradients(objective, s, y, num_class=K)
    if objective == "binary":
        p = 1.0 / (1.0 + np.exp(-s))
        np.testing.assert_allclose(g, p - y, rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(h, p * (1 - p), rtol=1e-6, atol=1e-7)
    else:
        e = np.exp(s.reshape(K, n))
        p = e / e.sum(axis=0)
        np.testing.assert_allclose(g.reshape(K, n), p - (np.arange(K)[:, None] == y[None, :]), rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(h.reshape(K, n), K / (K - 1.0) * p * (1 - p), rtol=1e-6, atol=1e-7)


def test_jni_shim_defines_refit(built, tmp_path):
    """jvm/b200gbm_jni.c compiled as tests/test_capi_cpu.py compiles it: the LGBM_1BoosterRefit native is defined and links"""
    import shutil
    import subprocess
    import __graft_entry__ as g
    cc = shutil.which("gcc")
    if cc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "lib_lightgbm_swig.so")
    cmd = [cc, "-shared", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(root, "jvm", "stub"), "-I" + os.path.join(root, "include"),
           os.path.join(root, "jvm", "b200gbm_jni.c"), "-L" + os.path.dirname(g.LIB), "-lb200gbm", "-Wl,--no-undefined", "-o", out]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    syms = subprocess.run(["nm", "-D", "--defined-only", out], check=True, capture_output=True, text=True).stdout
    assert "Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_LGBM_1BoosterRefit" in syms
