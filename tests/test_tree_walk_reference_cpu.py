"""The tree walks of the host predictor against the NumPy restatement of LightGBM's decision rules (tree_walk_ref), without a GPU.

The restatement is pinned first on hand-worked nodes of every kind and on the x86 conversions it relies on.  Then the host predictor
(LGBM_BoosterLoadModelFromString, then predict_for_mat, predict_for_mat_single and predict_for_csr_single) must give its leaf indices
exactly, its raw scores bit for bit and brute-force Shapley values to 1e-10, on a hand-written forest and on the committed golden models,
at rows that put every feature on the edges of the nodes that split on it: thresholds and their neighbouring doubles, +-0, +-1e-35,
subnormals, +-1e300, +-1e308, +-inf, NaN, and negative, fractional, huge and out-of-bitset categories.  Rows with a NaN in a
categorical feature are checked on their own: LightGBM sends them right at every categorical node."""
import importlib.util
import json
import os

import numpy as np
import pytest

import tree_walk_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "oracle_golden.json")))["models"]
RANGES = [(0, -1), (1, 2)]


@pytest.fixture(scope="module")
def capi(built):
    from mmlspark_b200 import capi
    capi.load()
    return capi


# ---------------------------------------------------------------- the restatement itself
def _one_node(dt, thr=0.0, cats=None):
    t = dict(num_leaves=2, decision_type=[dt], threshold=[thr], left_child=[-1], right_child=[-2], split_feature=[0])
    if cats is not None:
        words = [0] * (max(cats) // 32 + 1)
        for c in cats:
            words[c >> 5] |= 1 << (c & 31)
        t.update(threshold=[0.0], cat_boundaries=[0, len(words)], cat_threshold=words)
    return t


def _left(t, v):
    return R.decide(t, 0, v) == -1


def test_x86_int_conversion():
    assert R.x86_int(-0.5) == 0 and R.x86_int(-0.0) == 0 and R.x86_int(0.99) == 0 and R.x86_int(31.9) == 31 and R.x86_int(-1.5) == -1
    assert R.x86_int(2.0 ** 31 - 1) == 2 ** 31 - 1 and R.x86_int(2.0 ** 31 - 0.5) == 2 ** 31 - 1 and R.x86_int(-2.0 ** 31) == -2 ** 31
    for v in (np.nan, np.inf, -np.inf, 2.0 ** 31, 3e9, -3e9, -2.0 ** 31 - 1, 1e300):
        assert R.x86_int(v) == R.INT_MIN, v


def test_numerical_nodes_by_hand():
    for dl in (0, 2):
        none = _one_node(0 | dl, 0.5)                 # missing type None: NaN is 0.0, whatever the default direction
        assert _left(none, 0.5) and not _left(none, np.nextafter(0.5, 1)) and _left(none, np.nan) and _left(none, -np.inf)
        assert not _left(none, np.inf) and _left(none, -0.0)
        neg = _one_node(0 | dl, -2.25)
        assert not _left(neg, np.nan) and _left(neg, -2.25) and not _left(neg, np.nextafter(-2.25, 0))
        zero = _one_node(4 | dl, 0.5)                 # missing type Zero: |x| <= 1e-35 and NaN take the default direction
        for v in (0.0, -0.0, 1e-35, -1e-35, R.SUBNORMAL, np.nan):
            assert _left(zero, v) == bool(dl), v
        assert _left(zero, np.nextafter(1e-35, 1)) and _left(zero, np.nextafter(-1e-35, -1)) and not _left(zero, 0.6)
        nan = _one_node(8 | dl, 1e300)                # missing type NaN: only NaN takes the default direction
        assert _left(nan, np.nan) == bool(dl) and _left(nan, 0.0) and _left(nan, 1e300)
        assert not _left(nan, np.nextafter(1e300, np.inf)) and not _left(nan, 1e308) and not _left(nan, np.inf)
    tiny = _one_node(0, -1e-35)
    assert _left(tiny, -1e-35) and not _left(tiny, -0.0) and not _left(tiny, -R.SUBNORMAL) and _left(tiny, np.nextafter(-1e-35, -1))


def test_categorical_nodes_by_hand():
    for mt in (0, 2):
        t = _one_node(1 | mt << 2, cats=[0, 31, 32, 63, 64, 95])
        for v in (0.0, -0.0, -0.5, 0.5, 0.99, 31.0, 31.9, 32.0, 63.5, 64.0, 95.0):
            assert _left(t, v), v
        for v in (np.nan, -1.0, 1.0, 30.99, 33.0, 96.0, 2.0 ** 31 - 1, 2.0 ** 31, 3e9, -3e9, np.inf, -np.inf):
            assert not _left(t, v), v
        one = _one_node(1 | mt << 2, cats=[3])
        assert _left(one, 3.7) and not _left(one, 0.0) and not _left(one, 35.0)       # 35 is past the single word


def test_binned_nodes_by_hand():
    meta = R.feature_meta(5, 1, [-1.0, 1e-35, 2.0, np.inf, np.nan])
    t = _one_node(8, 1e300)                           # "numbers vs NaN": the bound +inf is written as 1e300
    assert [R.decide_bin(t, 0, b, meta) for b in range(5)] == [-1, -1, -1, -1, -2]
    assert R.decide(t, 0, 1e308) == -2 and R.decide(t, 0, np.inf) == -2           # the raw walk sends them right
    t = _one_node(2, 2.0)
    assert [R.decide_bin(t, 0, b, meta) for b in range(5)] == [-1, -1, -1, -2, -2]
    z = _one_node(4, 2.0)
    assert [R.decide_bin(z, 0, b, meta) for b in range(5)] == [-1, -2, -1, -2, -2]      # Zero: the default bin goes the default way
    cmeta = R.feature_meta(4, 0, [], [-1, 5, 0, 40])
    c = _one_node(1, cats=[0, 40])
    assert [R.decide_bin(c, 0, b, cmeta) for b in range(4)] == [-2, -2, -1, -1]         # bin 0 (NaN, negative, unseen) never goes left


# ---------------------------------------------------------------- the host predictor against it
def _golden_rows(name, trees, F):
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "golden", "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    X, _ = mg.dataset(123, 2000, F)
    X = mg.variant(X, name)
    base = [np.zeros(F)] + [np.nan_to_num(X[i], nan=0.5) for i in range(3)]
    return R.edge_rows(trees, F, base)


def _case(name):
    from mmlspark_b200.modeltext import parse_model
    if name == "hand":
        text = R.hand_forest_text()
    else:
        text = GOLDEN[name]["model"]
    m = parse_model(text)
    K = int(m["header"]["num_tree_per_iteration"])
    F = int(m["header"]["max_feature_idx"]) + 1
    X = R.edge_rows(m["trees"], F, R.HAND_BASE_ROWS) if name == "hand" else _golden_rows(name, m["trees"], F)
    return text, m["trees"], K, F, X, "\naverage_output\n" in text


def _split_rows(trees, X):
    cat = R.categorical_features(trees)
    nan_cat = np.isnan(X[:, cat]).any(axis=1) if cat else np.zeros(len(X), bool)
    return {"edges": X[~nan_cat], "categorical_nan": X[nan_cat]}


CASES = [("hand", "edges"), ("hand", "categorical_nan")] + [(n, "edges") for n in GOLDEN] + \
        [(n, "categorical_nan") for n in GOLDEN if "categorical_feature" in n]


@pytest.mark.parametrize("name,rows", CASES)
def test_host_predictor_walks_like_lightgbm(capi, name, rows):
    text, trees, K, F, X, avg = _case(name)
    X = _split_rows(trees, X)[rows]
    assert len(X) > 0
    b = capi.Booster(model_str=text)
    for s, k in RANGES:
        leaves = R.leaf_indices(trees, X, K, s, k)
        raw = R.scores_from_leaves(trees, leaves, K, s, k, avg)
        np.testing.assert_array_equal(b.predict_for_mat(X, capi.PREDICT_LEAF_INDEX, s, k), leaves, err_msg="leaf %d %d" % (s, k))
        np.testing.assert_array_equal(b.predict_for_mat(X, capi.PREDICT_RAW_SCORE, s, k), raw, err_msg="raw %d %d" % (s, k))
        for i, x in enumerate(X):
            np.testing.assert_array_equal(b.predict_for_mat_single(x, capi.PREDICT_LEAF_INDEX, s, k), leaves[i], err_msg="single row %d" % i)
            np.testing.assert_array_equal(b.predict_for_mat_single(x, capi.PREDICT_RAW_SCORE, s, k), raw[i], err_msg="single row %d" % i)
            nz = np.nonzero(x)[0]                     # CSR without the zeros: an omitted entry is 0.0; NaN is stored
            np.testing.assert_array_equal(b.predict_for_csr_single(nz, x[nz], F, capi.PREDICT_RAW_SCORE, s, k), raw[i], err_msg="csr row %d" % i)
            np.testing.assert_array_equal(b.predict_for_csr_single(nz, x[nz], F, capi.PREDICT_LEAF_INDEX, s, k), leaves[i], err_msg="csr row %d" % i)
    # contributions: brute force is exponential in a tree's features, so the golden models check a sample of the rows
    pick = np.arange(len(X)) if name == "hand" else np.random.default_rng(len(X)).choice(len(X), min(len(X), 40), replace=False)
    for s, k in RANGES:
        got = b.predict_for_mat(X[pick], capi.PREDICT_CONTRIB, s, k)
        want = np.array([R.contributions(trees, X[i], F, K, s, k) for i in pick])
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-10, err_msg="contrib %d %d" % (s, k))


def test_edge_rows_reach_every_leaf_of_the_hand_forest():
    """the rows of the hand-written forest reach every leaf of every tree, on both sides of each categorical NaN"""
    from mmlspark_b200.modeltext import parse_model
    trees = parse_model(R.hand_forest_text())["trees"]
    X = R.edge_rows(trees, R.HAND_NUM_FEATURE, R.HAND_BASE_ROWS)
    leaves = R.leaf_indices(trees, X, R.HAND_K)
    for t, tr in enumerate(trees):
        assert set(leaves[:, t].astype(int)) == set(range(int(tr["num_leaves"]))), t
