"""Prediction early stopping (pred_early_stop, pred_early_stop_freq, pred_early_stop_margin) in the host predictor against the NumPy
restatement pred_early_stop_ref, without a GPU.  Hand-written model strings are loaded with LGBM_BoosterLoadModelFromString and predicted
with LGBM_BoosterPredictForMatSingle, LGBM_BoosterPredictForCSRSingle and LGBM_BoosterPredictForMat: raw scores must equal the
restatement bit for bit, and the stop points the cases are built for (the first period, a middle one, never) are asserted from it."""
import numpy as np
import pytest

import pred_early_stop_ref as E
import tree_walk_ref as R

N = R.N


@pytest.fixture(scope="module")
def capi(built):
    from mmlspark_b200 import capi
    capi.load()
    return capi


def model_text(specs, K, objective, num_feature=4, average=False):
    head = ["tree", "version=v3", "num_class=%d" % K, "num_tree_per_iteration=%d" % K, "label_index=0", "max_feature_idx=%d" % (num_feature - 1)]
    if objective is not None:
        head.append("objective=" + objective)
    if average:
        head.append("average_output")
    head += ["feature_names=" + " ".join("f%d" % f for f in range(num_feature)), "feature_infos=" + " ".join(["[-1e+308:1e+308]"] * num_feature), ""]
    body = "".join("Tree=%d\n%s\n" % (t, R._tree_text(s, t)) for t, s in enumerate(specs))
    return "\n".join(head) + body + "end of trees\n"


def trees_of(text):
    from mmlspark_b200.modeltext import parse_model
    return parse_model(text)["trees"]


def random_specs(rng, n_trees, scale, num_feature=4):
    def node(depth):
        if depth == 0:
            return float(rng.normal() * scale)
        return N(int(rng.integers(num_feature)), float(np.round(rng.normal(), 3)), int(rng.choice([0, 2, 8, 10])), node(depth - 1), node(depth - 1))
    return [node(2) for _ in range(n_trees)]


def params(freq, margin, on="true"):
    return "pred_early_stop=%s pred_early_stop_freq=%s pred_early_stop_margin=%s" % (on, freq, margin)


def host_all(b, X, pt, s, k, parameter):
    """the three host entries on the same rows; they must agree bit for bit"""
    mat = b.predict_for_mat(X, pt, s, k, parameter=parameter)
    single = np.array([b.predict_for_mat_single(x, pt, s, k, parameter=parameter) for x in X])
    csr = np.array([b.predict_for_csr_single(np.arange(len(x)), x, len(x), pt, s, k, parameter=parameter) for x in X])
    np.testing.assert_array_equal(single, mat)
    np.testing.assert_array_equal(csr, mat)
    return mat


def transform(objective, raw):
    name = objective.split()[0]
    if name == "binary" or name == "multiclassova":
        return 1.0 / (1.0 + np.exp(-raw))
    if name == "multiclass":
        e = np.exp(raw - raw.max(axis=1, keepdims=True))
        return e / e.sum(axis=1, keepdims=True)
    return raw


def check(capi, text, X, K, objective, freq, margin, s=0, k=-1, average=False):
    """raw and normal outputs of every host entry against the restatement; returns the iterations walked per row"""
    b = capi.Booster(model_str=text)
    trees = trees_of(text)
    want, walked = E.raw_scores(trees, X, K, s, k, freq, margin, average)
    p = params(freq, margin)
    got = host_all(b, X, capi.PREDICT_RAW_SCORE, s, k, p)
    np.testing.assert_array_equal(got, want)
    norm = host_all(b, X, capi.PREDICT_NORMAL, s, k, p)
    np.testing.assert_allclose(norm, transform(objective, want), rtol=1e-14, atol=0)
    return walked


# ---------------------------------------------------------------- the restatement itself
def test_margin_rule_by_hand():
    assert E.margin([3.0]) == 6.0 and E.margin([-2.5]) == 5.0 and E.margin([0.0]) == 0.0
    assert E.margin([1.0, 1.0, 0.0]) == 0.0 and E.margin([2.0, 1.0, 5.0]) == 3.0 and E.margin([-1.0, -4.0]) == 3.0
    assert E.applies("binary sigmoid:1", 0) and E.applies("multiclassova num_class:3 sigmoid:1", 1) and E.applies("rank_xendcg", 0)
    assert not E.applies("binary sigmoid:1", 2) and not E.applies("regression", 0) and not E.applies("", 0) and not E.applies("custom", 1)
    assert not E.applies("binary", 0, on=False)


# ---------------------------------------------------------------- stop points by construction
# binary: row A (x0 <= 0) adds about 1 per tree, row B (x0 > 0, x1 <= 0) about 0.5, row C (both > 0) about 0.01.  With freq 3 and
# margin 5 A stops after the first period (2 * 3.x > 5), B after the second (2 * 3.x > 5), and C never.
STOP_SPECS = [N(0, 0.0, 0, 1.0 + 0.013 * t, N(1, 0.0, 0, 0.5 + 0.007 * t, 0.01 * (t % 3 - 0.5))) for t in range(12)]
STOP_ROWS = np.array([[-1.0, 0.0, 0.0, 0.0], [1.0, -1.0, 0.0, 0.0], [1.0, 1.0, 0.0, 0.0]])


def test_binary_rows_stop_in_the_first_period_a_middle_one_and_never(capi):
    text = model_text(STOP_SPECS, 1, "binary sigmoid:1")
    walked = check(capi, text, STOP_ROWS, 1, "binary sigmoid:1", 3, 5.0)
    assert list(walked) == [3, 6, 12]
    b = capi.Booster(model_str=text)
    off = b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE)
    on = b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE, parameter=params(3, 5.0))
    assert on[0, 0] < off[0, 0] and on[1, 0] < off[1, 0] and on[2, 0] == off[2, 0]


def test_period_that_does_not_divide_the_range_and_iteration_ranges(capi):
    text = model_text(STOP_SPECS, 1, "binary sigmoid:1")
    # freq 5 over 12 iterations: checks after 5 and 10, the last 2 always walked unless stopped
    assert list(check(capi, text, STOP_ROWS, 1, "binary sigmoid:1", 5, 5.5)) == [5, 10, 12]
    # iterations [2, 9): periods of 3 end at iterations 5 and 8
    assert list(check(capi, text, STOP_ROWS, 1, "binary sigmoid:1", 3, 5.0, s=2, k=7)) == [3, 6, 7]
    assert list(check(capi, text, STOP_ROWS, 1, "binary sigmoid:1", 4, 2.5, s=5, k=-1)) == [4, 4, 7]


@pytest.mark.parametrize("objective,K", [("binary sigmoid:1", 1), ("multiclass num_class:3", 3), ("multiclassova num_class:3 sigmoid:1", 3),
                                         ("lambdarank", 1)])
def test_random_forests_match_the_restatement(capi, objective, K):
    rng = np.random.default_rng(7 + K)
    text = model_text(random_specs(rng, 10 * K, 0.6), K, objective)
    X = rng.normal(size=(60, 4))
    X[::7, 1] = np.nan
    seen = set()
    for freq, margin, s, k in ((1, 1.0, 0, -1), (2, 2.0, 0, -1), (3, 1.5, 0, -1), (4, 3.0, 1, 7), (10, 0.5, 0, -1), (20, 0.0, 0, -1)):
        walked = check(capi, text, X, K, objective, freq, margin, s, k)
        total = min(10 - s, k if k > 0 else 10)
        seen |= {"first" if w == min(freq, total) and w < total else "never" if w == total else "middle" for w in walked}
    assert seen == {"first", "middle", "never"}


def test_margin_zero_does_not_stop_a_zero_score(capi):
    # row Z sums 0.5, 0, 0.5, 0, 0.5: at the checks after 2 and 4 iterations its margin is exactly 0, which is not > 0
    specs = [N(0, 0.0, 0, 0.5 if t % 2 == 0 else -0.5, 0.25) for t in range(5)]
    text = model_text(specs, 1, "binary sigmoid:1")
    rows = np.array([[-1.0, 0, 0, 0], [1.0, 0, 0, 0]])
    assert list(check(capi, text, rows, 1, "binary sigmoid:1", 2, 0.0)) == [5, 2]
    b = capi.Booster(model_str=text)
    assert b.predict_for_mat(rows, capi.PREDICT_RAW_SCORE, parameter=params(2, 0.0))[0, 0] == 0.5


def test_tied_top_two_classes_give_margin_zero(capi):
    # x0 <= 0: classes 0 and 1 tie at every check, so margin 0 never stops the row; x0 > 0: class 0 leads by 1.9 per iteration
    specs = []
    for t in range(6):
        specs += [N(0, 0.0, 0, 1.0, 2.0), N(0, 0.0, 0, 1.0, 0.1), N(0, 0.0, 0, -1.0, 0.0)]
    rows = np.array([[-1.0, 0, 0, 0], [1.0, 0, 0, 0]])
    for obj in ("multiclass num_class:3", "multiclassova num_class:3 sigmoid:1"):
        text = model_text(specs, 3, obj)
        assert list(check(capi, text, rows, 3, obj, 2, 0.0)) == [6, 2]
        assert list(check(capi, text, rows, 3, obj, 1, 3.5)) == [6, 2]


def test_rf_model_divides_by_the_whole_range(capi):
    text = model_text(STOP_SPECS, 1, "binary sigmoid:1", average=True)
    assert list(check(capi, text, STOP_ROWS, 1, "binary sigmoid:1", 3, 5.0, average=True)) == [3, 6, 12]
    b = capi.Booster(model_str=text)
    got = b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE, parameter=params(3, 5.0))
    sums, _ = E.raw_scores(trees_of(text), STOP_ROWS, 1, freq=3, margin_threshold=5.0)
    np.testing.assert_array_equal(got, sums / 12)


@pytest.mark.parametrize("objective", ["regression", "cross_entropy", "custom", None, "regression_l1", "poisson"])
def test_other_objectives_ignore_the_keys(capi, objective):
    text = model_text(STOP_SPECS, 1, objective)
    b = capi.Booster(model_str=text)
    for pt in (capi.PREDICT_NORMAL, capi.PREDICT_RAW_SCORE):
        want = host_all(b, STOP_ROWS, pt, 0, -1, "")
        for p in (params(3, 5.0), params(0, 5.0), params(3, -1.0), params(-2, "nan")):
            np.testing.assert_array_equal(host_all(b, STOP_ROWS, pt, 0, -1, p), want)


@pytest.mark.parametrize("objective,K", [("binary sigmoid:1", 1), ("multiclass num_class:3", 3)])
def test_leaf_and_contribution_predictions_ignore_the_keys(capi, objective, K):
    rng = np.random.default_rng(3)
    text = model_text(random_specs(rng, 6 * K, 2.0), K, objective)
    b = capi.Booster(model_str=text)
    X = rng.normal(size=(8, 4))
    for pt in (capi.PREDICT_LEAF_INDEX, capi.PREDICT_CONTRIB):
        want = host_all(b, X, pt, 0, -1, "")
        for p in (params(1, 0.0), params(0, -1.0)):
            np.testing.assert_array_equal(host_all(b, X, pt, 0, -1, p), want)


def test_no_key_false_null_and_huge_margin_equal_todays_output(capi):
    rng = np.random.default_rng(11)
    text = model_text(random_specs(rng, 30, 1.0), 3, "multiclass num_class:3")
    b = capi.Booster(model_str=text)
    X = rng.normal(size=(20, 4))
    want, _ = E.raw_scores(trees_of(text), X, 3, freq=None)
    for p in ("", None, "max_bin=255", params(1, 0.0, on="false"), params(0, -1.0, on="false"), params(1, 1e300), params(11, 0.0)):
        np.testing.assert_array_equal(host_all(b, X, capi.PREDICT_RAW_SCORE, 0, -1, p), want, err_msg=str(p))
    np.testing.assert_array_equal(b.predict_for_mat(X, capi.PREDICT_RAW_SCORE), want)


@pytest.mark.parametrize("bad,message", [(params(0, 5.0), "Check failed: (early_stop_freq) > (0)"),
                                         (params(-3, 5.0), "Check failed: (early_stop_freq) > (0)"),
                                         (params(10, -0.5), "Check failed: (early_stop_margin) >= (0)"),
                                         (params(10, "nan"), "Check failed: (early_stop_margin) >= (0)")])
def test_checks_fail_the_call_and_leave_the_booster_usable(capi, bad, message):
    text = model_text(STOP_SPECS, 1, "binary sigmoid:1")
    b = capi.Booster(model_str=text)
    want = b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE)
    for call in (lambda: b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE, parameter=bad),
                 lambda: b.predict_for_mat_single(STOP_ROWS[0], capi.PREDICT_NORMAL, parameter=bad),
                 lambda: b.predict_for_csr_single(np.arange(4), STOP_ROWS[0], 4, capi.PREDICT_RAW_SCORE, parameter=bad)):
        with pytest.raises(capi.LightGBMError, match=message.replace("(", r"\(").replace(")", r"\)")):
            call()
    np.testing.assert_array_equal(b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE), want)
    np.testing.assert_array_equal(b.predict_for_mat(STOP_ROWS, capi.PREDICT_RAW_SCORE, parameter=bad.replace("=true", "=false")), want)
    assert b.predict_for_mat(STOP_ROWS, capi.PREDICT_LEAF_INDEX, parameter=bad).shape == (3, 12)
