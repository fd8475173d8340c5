"""The split scans (K5/K6: k_scan, k_scan_wide) and the pick step (d_pick_block / d_choose_leaf) against the NumPy restatement of
LightGBM 3.2's split search in split_scan_ref.py, tree by tree.

Binning and K4 are taken out of the comparison on purpose: the bins are read back from the dataset, and gradients and hessians lie on a
2^-10 grid (scaled by a power of two) with at most 65 536 rows, so K4's fixed-point quantisation is exact, every int64 sum fits in
53 bits, and the fp64 histogram NumPy builds equals the engine's bit for bit.  Only the scan and the pick are under test.

Bar: identical structure (feature, threshold bin, default direction, category set, which leaf splits, counts), leaf values and
weights within 4 fp64 ulps (-O3 contracts to FMA), internal values and weights as printed (%g), split_gain equal to the reference's
float(gain + min_gain_to_split) printed with %g.  Every case must be *decided* on the reference side first (split_scan_ref.undecided):
a case whose winner could flip with the last bits of a gain or a count at a .5 boundary fails instead of passing by luck."""
import numpy as np
import pytest

import split_scan_ref as ref
import tree_check as tc
import tree_ref

pytestmark = pytest.mark.gpu

GRID = tc.GRID


def _on_grid(x):
    return np.round(np.asarray(x, np.float64) / GRID) * GRID


def _train(X, g, h, params, ds_params="", cat=(), label=None):
    """one boosting iteration with learning_rate 1; custom (g, h) unless `label` is given (objective=regression, constant hessian)"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    dsp = "max_bin=255 min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0 " + ds_params
    if cat:
        dsp += " categorical_feature=" + ",".join(str(c) for c in cat)
    ds = capi.Dataset.from_mat(X, dsp)
    ds.set_field("label", np.zeros(len(X), np.float32) if label is None else label)
    F = X.shape[1]
    infos = [ds.feature_info(f) for f in range(F)]
    feats = [ref.Feature(f, infos[f]["num_bin"], infos[f]["missing_type"], int(infos[f]["most_freq_bin"] == 0), f in cat)
             for f in range(F) if not infos[f]["is_trivial"]]
    bins = ds.get_bins16()
    full = ("objective=regression boost_from_average=false learning_rate=1 num_iterations=1 verbosity=-1 " + dsp + " " + params)
    b = capi.Booster(ds, full)
    if label is None:
        b.update_one_iter_custom(g.astype(np.float32), h.astype(np.float32))
    else:
        b.update_one_iter()
    text = b.save_model_to_string()
    side = dict(ub={f.real_index: ds.upper_bounds(f.real_index) for f in feats},
                b2c={f.real_index: ds.bin_to_cat(f.real_index) for f in feats if f.is_cat})
    b.free(); ds.free()
    return parse_model(text), text, feats, bins, side


def _check(X, g, h, params, num_leaves, ds_params="", cat=(), label=None, expect_leaves=None):
    """train, restate, assert decided, compare; returns (reference tree, model text)"""
    p = ref.Params(**params)
    extra = "num_leaves=%d %s" % (num_leaves, p.as_string())
    m, text, feats, bins, side = _train(X, g, h, extra, ds_params, cat, label)
    if label is not None:              # regression from a zero score: g = -label, h = 1
        g, h = -label.astype(np.float64), np.ones(len(X))
    for v in (g, h):                   # the premise of the exact comparison: fp32-exact values on a (scaled) 2^-10 grid
        v = np.asarray(v, np.float64)
        assert len(v) <= 65536 and np.array_equal(v.astype(np.float32).astype(np.float64), v)
        nz = np.abs(v[v != 0])
        if len(nz):
            step = 2.0 ** (np.floor(np.log2(nz.max())) - 23)
            assert np.array_equal(np.round(v / step) * step, v)
    T = tree_ref.grow_tree(bins, np.asarray(g, np.float64), np.asarray(h, np.float64), feats, p, num_leaves)
    T["features"] = {f.real_index: f for f in feats}
    why = ref.undecided(T)
    assert not why, "the case does not discriminate:\n" + "\n".join(why[:10])
    if expect_leaves is not None:
        assert T["num_leaves"] == expect_leaves, "the case was built to grow %d leaves, the reference grows %d" % (expect_leaves, T["num_leaves"])
    tc.compare_tree(m["trees"][0], T, side["ub"], side["b2c"])
    return T, text


def _step_case(num_bin, split_at, seed, rows_per_bin=24, nan_rows=0, scale=1.0):
    """one integer feature with `num_bin` values (plus a NaN value when nan_rows > 0) whose gradients step at value `split_at`,
    and a weaker random feature; grid noise keeps every gain distinct"""
    rng = np.random.default_rng(seed)
    v = np.repeat(np.arange(num_bin, dtype=np.float64), rows_per_bin)
    if nan_rows:
        v = np.concatenate([v, np.full(nan_rows, np.nan)])
    n = len(v)
    w = rng.integers(0, 13, n).astype(np.float64)
    g = np.where(v <= split_at, -2.0, 1.5) + 0.25 * (w - 6) / 6 + tc.grid(rng, -0.5, 0.5, n)
    if nan_rows:
        g[np.isnan(v)] = -3.0 + tc.grid(rng, -0.25, 0.25, nan_rows)
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([v, w], axis=1)
    perm = rng.permutation(n)
    return X[perm], np.round(g[perm] / GRID) * GRID * scale, h[perm] * scale


# ---------------------------------------------------------------- bin counts and lane boundaries (k_scan: one bin per thread)
@pytest.mark.parametrize("num_bin", [2, 3, 8, 9, 31, 32, 33, 255, 256])
@pytest.mark.parametrize("where", ["first", "last", "lane"])
def test_root_scan_bin_counts(built, num_bin, where):
    split_at = {"first": 0, "last": num_bin - 2, "lane": min(7, num_bin - 2)}[where]
    if where == "lane" and num_bin > 32:
        split_at = 31
    X, g, h = _step_case(num_bin, split_at, seed=num_bin * 7 + len(where))
    _check(X, g, h, dict(min_data_in_leaf=5), 2, ds_params="max_bin=%d" % max(255, num_bin), expect_leaves=2)


@pytest.mark.parametrize("max_bin", [300, 1024, 4097])
def test_wide_numerical_scan(built, max_bin):
    """features with more than 256 bins: k_scan_wide's block scan, several bins per thread"""
    X, g, h = _step_case(max_bin, max_bin // 3 + 1, seed=max_bin, rows_per_bin=4, nan_rows=40)
    _check(X, g, h, dict(min_data_in_leaf=3), 4, ds_params="max_bin=%d" % max_bin)


# ---------------------------------------------------------------- missing values
@pytest.mark.parametrize("num_bin,nan_rows,sign", [(16, 200, -1), (16, 200, +1), (40, 64, -1), (200, 300, +1)])
def test_nan_two_way_scan(built, num_bin, nan_rows, sign):
    """NaN rows with gradients like the low side (reverse pass wins, NaN left) or like the high side (forward pass wins, NaN right)"""
    X, g, h = _step_case(num_bin, num_bin // 2, seed=num_bin + nan_rows, nan_rows=nan_rows)
    nan = np.isnan(X[:, 0])
    g[nan] = (-2.0 if sign < 0 else 1.5) + np.round(np.linspace(-0.3, 0.3, nan.sum()) / GRID) * GRID
    T, _ = _check(X, g, h, dict(min_data_in_leaf=10), 3)
    assert T["split_feature"][0] == 0 and T["default_left"][0] == (sign < 0)


@pytest.mark.parametrize("sign", [-1, +1])
def test_nan_offset_zero(built, sign):
    """negative and positive values: the zero bin sits in the middle, so most_freq_bin != 0 and offset == 0 (every other NaN feature
    here holds non-negative values only, which puts the zero bin first).  The forward pass then accumulates from bin 0 itself.  NaN rows
    like the low side: the reverse pass wins, NaN left; like the high side: the forward pass wins, NaN right."""
    rng = np.random.default_rng(50 + sign)
    n = 8000
    v = rng.integers(-10, 11, n).astype(np.float64)
    v[rng.random(n) < 0.1] = np.nan
    g = np.where(v <= 2, -1.0, 1.0) + tc.grid(rng, -0.5, 0.5, n)
    g[np.isnan(v)] = sign * 1.25 + tc.grid(rng, -0.25, 0.25, int(np.isnan(v).sum()))
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([v, rng.integers(0, 5, n).astype(np.float64)], axis=1)
    T, _ = _check(X, g, h, dict(min_data_in_leaf=20), 3)
    f0 = T["features"][0]
    assert f0.missing_type == 2 and f0.offset == 0, "the case must exercise the offset-0 forward pass"
    assert T["split_feature"][0] == 0 and T["default_left"][0] == (sign < 0)


def test_nan_offset_one_forward_pass(built):
    """most_freq_bin == 0 (the zero bin holds 60 % of the rows) with NaN: the forward pass starts from the implicit bin 0 (as in the
    other NaN cases with non-negative values), here with the first threshold the winning one"""
    rng = np.random.default_rng(5)
    n = 6000
    v = np.where(rng.random(n) < 0.6, 0.0, rng.integers(1, 20, n).astype(np.float64))
    v[rng.random(n) < 0.1] = np.nan
    g = np.where(np.isnan(v) | (v > 9), 1.0, -1.0) + tc.grid(rng, -0.5, 0.5, n)
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([v, rng.integers(0, 5, n).astype(np.float64)], axis=1)
    T, _ = _check(X, g, h, dict(min_data_in_leaf=20), 2, expect_leaves=2)
    assert T["features"][0].offset == 1 and T["default_left"][0] is False


def test_use_missing_false(built):
    X, g, h = _step_case(24, 11, seed=77, nan_rows=100)
    _check(X, g, h, dict(min_data_in_leaf=10), 3, ds_params="use_missing=false")


# ---------------------------------------------------------------- constraints at their boundary
def _blocks(sizes, gs, hs):
    """one integer feature: value i on sizes[i] rows with per-row g = gs[i], h = hs[i], and a second feature whose best split is
    clearly worse than feature 0's"""
    v = np.repeat(np.arange(len(sizes), dtype=np.float64), sizes)
    g = np.repeat(np.asarray(gs, np.float64), sizes)
    h = np.repeat(np.asarray(hs, np.float64), sizes)
    w = (np.arange(len(v)) % 7).astype(np.float64)
    g = g + (w - 3) * GRID * 4
    return np.stack([v, w], axis=1), g, h


@pytest.mark.parametrize("min_data", [30, 31])
def test_min_data_in_leaf_boundary(built, min_data):
    """the best threshold leaves exactly 30 rows on the right: allowed at min_data_in_leaf=30, not at 31"""
    X, g, h = _blocks([40, 40, 40, 30], [-1, -1.25, -0.75, 4.0], [1, 1, 1, 1])
    T, _ = _check(X, g, h, dict(min_data_in_leaf=min_data), 2, expect_leaves=2)
    assert T["split_feature"][0] == 0 and (T["threshold_bin"][0] == 2) == (min_data == 30)


@pytest.mark.parametrize("direction", [+1, -1])
def test_rebuilt_count_crosses_min_data(built, direction):
    """the rebuilt count of the small side differs from its true count (hessians per row 1.25 or 0.75 there): with
    min_data_in_leaf = 25 the 22-row side passes, rebuilt as 26.8 -> 27 rows, and the 28-row side fails, rebuilt as 21.7 -> 22"""
    rows = 22 if direction > 0 else 28
    hr = 1.25 if direction > 0 else 0.75
    X, g, h = _blocks([100, 100, rows], [-1, -0.5, 3.0], [1, 1, hr])
    T, _ = _check(X, g, h, dict(min_data_in_leaf=25), 2, expect_leaves=2)
    assert (T["threshold_bin"][0] == 1) == (direction > 0)


def test_rebuilt_count_rounds_up_to_min_data(built):
    """the small side's rebuilt count is 24.65 (25 rows at h = 63/64 among rows at h = 1): RoundInt makes it 25 and the threshold
    meets min_data_in_leaf = 25; truncating would make it 24 and reject the best threshold"""
    X, g, h = _blocks([100, 100, 25], [-1, -0.5, 3.0], [1, 1, 63 / 64])
    T, _ = _check(X, g, h, dict(min_data_in_leaf=25), 2, expect_leaves=2)
    x = 25 * 63 / 64 * len(h) / (h.sum() + 2 * ref.K_EPS)
    assert 24.5 < x < 25 and T["split_feature"][0] == 0 and T["threshold_bin"][0] == 1


def test_min_sum_hessian_met_exactly(built):
    X, g, h = _blocks([50, 50, 50, 40], [-1, -1.25, -0.75, 4.0], [1, 1, 1, 1.0])
    T, _ = _check(X, g, h, dict(min_data_in_leaf=5, min_sum_hessian_in_leaf=40.0), 2, expect_leaves=2)
    assert T["threshold_bin"][0] == 2
    T, _ = _check(X, g, h, dict(min_data_in_leaf=5, min_sum_hessian_in_leaf=40.0 + GRID), 2)
    assert T["num_leaves"] == 1 or T["threshold_bin"][0] != 2


def test_min_gain_to_split_equal_to_best_gain_is_rejected(built):
    """min_gain_to_split chosen so that min_gain_shift equals the best gain in fp64 (%r of a double round-trips through the parameter
    string): the scan's test is `gain <= min_gain_shift`, so the root must not split.  Gains without L1 or max_delta_step are a product,
    a division and a sum, which no FMA contraction changes, so the equality holds on the device as well."""
    X, g, h = _blocks([64, 64, 64, 64], [-1, -0.5, 0.5, 1], [1, 1, 1, 1])
    feats = [ref.Feature(0, 4), ref.Feature(1, 7)]
    p0 = ref.Params(min_data_in_leaf=5)
    scans = tree_ref.scan_leaf(X.astype(np.int64), g, h, np.arange(len(g)), float(g.sum()), float(h.sum()), len(g), feats, {0: True, 1: True}, p0)
    best, base = max(c[0] for sc in scans.values() for c in sc.candidates), scans[0].shift
    mg = best - base
    while base + mg < best:
        mg = np.nextafter(mg, np.inf)
    while base + mg > best:
        mg = np.nextafter(mg, -np.inf)
    assert base + mg == best
    for mgs, leaves in ((float(mg), 1), (float(np.nextafter(mg, -np.inf)), 2)):
        p = dict(min_data_in_leaf=5, min_gain_to_split=mgs)
        m, _, feats, bins, _ = _train(X, g, h, "num_leaves=2 " + ref.Params(**p).as_string())
        T = tree_ref.grow_tree(bins, g, h, feats, ref.Params(**p), 2)
        assert T["num_leaves"] == leaves and m["trees"][0]["num_leaves"] == leaves


# ---------------------------------------------------------------- regularisation
@pytest.mark.parametrize("params,num_leaves", [(dict(lambda_l1=50.0), 4), (dict(lambda_l1=130.0), 4), (dict(lambda_l2=7.5), 4),
                                               (dict(max_delta_step=1.5), 2), (dict(max_delta_step=0.6), 2),
                                               (dict(lambda_l1=20.0, lambda_l2=3.0, max_delta_step=0.9), 4)])
def test_regularisation(built, params, num_leaves):
    """lambda_l1 above and below |sum_g| of a side (the high side sums to about +120, the low side to about -160), lambda_l2, and
    max_delta_step clipping one side (1.5) or both (0.6).  Where both sides of most thresholds clip, their gains equal
    min_gain_shift up to rounding and the splittable flags are not decided: those cases stop at the root."""
    X, g, h = _step_case(24, 13, seed=31, rows_per_bin=10)
    p = dict(min_data_in_leaf=10)
    p.update(params)
    _check(X, g, h, p, num_leaves)


# ---------------------------------------------------------------- negative hessians: the scan ends where LightGBM breaks
def test_negative_hessians_break_hides_a_better_threshold(built):
    """feature 0: values 0..7 (h = +1), 8 (h = -8) and 9 (h = +10), 100 rows each, so the leaf's hessian sum is 1000 = num_data and
    every rebuilt count is exact.  The reverse scan adds value 9 first: 1000 rebuilt rows on the right leave 0 on the left, which fails
    min_data_in_leaf and ends the scan.  The threshold between 7 and 8 (gain far above feature 1's) lies beyond that break: LightGBM
    never evaluates it, finds no split on feature 0 and splits on feature 1.  A scan that continues past the break splits on feature 0."""
    rng = np.random.default_rng(3)
    v = np.repeat(np.arange(10, dtype=np.float64), 100)
    h = np.where(v == 8, -8.0, np.where(v == 9, 10.0, 1.0))
    w = rng.integers(0, 4, len(v)).astype(np.float64)
    g = np.where(v <= 7, -1.0, 2.0) + np.where(w >= 2, 0.5, -0.5) + tc.grid(rng, -0.125, 0.125, len(v))
    X = np.stack([v, w], axis=1)
    T, _ = _check(X, g, h, dict(min_data_in_leaf=20), 2, expect_leaves=2)
    assert T["split_feature"][0] == 1


# ---------------------------------------------------------------- ties made exact by construction
def test_empty_bins_in_children_reverse_keeps_the_higher_threshold(built):
    """values 0..3 and 6..9 and NaN: the binner makes no bin for absent values, so the root has no empty bin; after the root splits
    between 3 and 6, each child holds no rows in the other side's bins, neighbouring thresholds there give the same partition with
    bit-identical sums, and the reverse pass keeps the higher one"""
    rng = np.random.default_rng(8)
    v = np.concatenate([rng.integers(0, 4, 3000), rng.integers(6, 10, 3000), np.full(500, -1)]).astype(np.float64)
    v[v < 0] = np.nan
    g = np.where(np.isnan(v), 2.0, np.where(v < 5, -1.0, 1.0)) + tc.grid(rng, -0.25, 0.25, len(v))
    h = tc.grid(rng, 0.5, 1.5, len(v))
    X = np.stack([v, rng.integers(0, 3, len(v)).astype(np.float64)], axis=1)
    _check(X, g, h, dict(min_data_in_leaf=20), 3, ds_params="max_bin=12")


def test_empty_bins_in_a_child_forward_keeps_the_lower_threshold(built):
    """forward-pass tie: in the child a == 0, feature 1 holds values 0..2, 7..9 and NaN only, so the forward thresholds 2..6 give
    the same partition with bit-identical sums.  NaN rows have the high side's gradients, the forward pass (NaN right) wins, and it
    keeps the lowest of the tied thresholds, 2"""
    rng = np.random.default_rng(61)
    n = 8000
    a = np.repeat([0.0, 1.0], n // 2)
    v = np.where(a == 0, rng.choice([0, 1, 2, 7, 8, 9], n), rng.integers(0, 10, n)).astype(np.float64)
    v[rng.random(n) < 0.1] = np.nan
    hi = np.isnan(v) | (v >= 7)
    g = np.where(a == 0, np.where(hi, 1.0, -1.0) - 2.0, 2.0 + 0.25 * np.where(v > 4, 1, -1)) + tc.grid(rng, -0.125, 0.125, n)
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([a, v], axis=1)
    T, _ = _check(X, g, h, dict(min_data_in_leaf=20), 3, expect_leaves=3)
    assert T["split_feature"] == [0, 1] and T["left_child"][0] == 1           # the second split is in the child a == 0
    assert T["default_left"][1] is False and T["threshold_bin"][1] == 2


def test_duplicate_columns_smaller_real_index_wins(built):
    """column 2 is a copy of column 0 and column 3 a wide (> 256 bins) copy of column 1 placed before a tile copy at column 4: on a
    tie the smaller real index wins, also between k_scan_wide and k_scan candidates"""
    rng = np.random.default_rng(9)
    n = 9000
    a = rng.integers(0, 20, n).astype(np.float64)
    wide = rng.integers(0, 300, n).astype(np.float64)
    g = np.where(wide < 120, -1.0, 1.0) + 0.5 * np.where(a < 7, -1.0, 1.0) + tc.grid(rng, -0.25, 0.25, n)
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([a, rng.integers(0, 5, n).astype(np.float64), a, wide, np.minimum(wide, 119.0) + (wide >= 120) * 120], axis=1)
    T, _ = _check(X, g, h, dict(min_data_in_leaf=20), 4, ds_params="max_bin=300")
    assert 3 in T["split_feature"] and 0 in T["split_feature"] and 2 not in T["split_feature"]


# ---------------------------------------------------------------- gradient scale
@pytest.mark.parametrize("scale_log2", [-60, -20, 0, 20, 60])
def test_gradient_scale(built, scale_log2):
    X, g, h = _step_case(20, 9, seed=4, scale=2.0 ** scale_log2)
    _check(X, g, h, dict(min_data_in_leaf=10, min_sum_hessian_in_leaf=1e-3 * 2.0 ** scale_log2), 4)


def test_all_zero_gradients_give_no_split(built):
    X, _, h = _step_case(20, 9, seed=4)
    T, _ = _check(X, np.zeros(len(X)), h, dict(min_data_in_leaf=10), 4)
    assert T["num_leaves"] == 1


# ---------------------------------------------------------------- constant hessian (objective=regression)
@pytest.mark.parametrize("num_leaves", [2, 3, 4])
def test_constant_hessian_regression(built, num_leaves):
    rng = np.random.default_rng(20 + num_leaves)
    n = 20000
    X = np.stack([rng.integers(0, 50, n), rng.integers(0, 7, n), rng.integers(0, 200, n)], axis=1).astype(np.float64)
    y = (np.where(X[:, 0] < 17, -1.0, 1.0) + np.where(X[:, 2] < 150, 0.75, -0.5) + tc.grid(rng, -0.5, 0.5, n)).astype(np.float32)
    _check(X, None, None, dict(min_data_in_leaf=20), num_leaves, label=y, expect_leaves=num_leaves)


@pytest.mark.parametrize("larger", ["left", "right"])
def test_second_round_larger_child_from_subtraction(built, larger):
    """num_leaves=4: the root's larger child is scanned through parent - smaller; which side is larger alternates"""
    rng = np.random.default_rng(40 if larger == "left" else 41)
    n = 12000
    v = rng.integers(0, 40, n).astype(np.float64)
    cut = 29 if larger == "left" else 10
    X = np.stack([v, rng.integers(0, 30, n).astype(np.float64), rng.integers(0, 9, n).astype(np.float64)], axis=1)
    g = np.where(v <= cut, -1.5, 1.5) + np.where(X[:, 1] < 12, -0.5, 0.5) + 0.25 * np.where(X[:, 2] < 4, -1, 1) + tc.grid(rng, -0.25, 0.25, n)
    h = tc.grid(rng, 0.5, 1.5, n)
    T, _ = _check(X, g, h, dict(min_data_in_leaf=20), 4, expect_leaves=4)
    (l_leaf, l_cnt), (r_leaf, r_cnt) = T["scanned_counts"][1]
    assert T["split_feature"][0] == 0 and l_leaf == 0 and r_leaf == 1
    assert (l_cnt > r_cnt) == (larger == "left")


def test_equal_gain_leaves_smaller_leaf_index_wins(built):
    """the root's children hold mirror images (feature 1 shifted by 10, same hessians, negated gradients): their best gains are
    bit-identical and the smaller leaf index splits first.  At the root both features separate the halves with the same partition,
    and the smaller real index wins that tie."""
    rng = np.random.default_rng(12)
    m = 3000
    a = rng.integers(0, 10, m).astype(np.float64)
    ga = np.where(a < 4, -1.0, 1.0) + 0.5 + tc.grid(rng, -0.25, 0.25, m)
    ha = tc.grid(rng, 0.5, 1.5, m)
    X = np.stack([np.concatenate([np.zeros(m), np.ones(m)]), np.concatenate([a, a + 10])], axis=1)
    T, _ = _check(X, np.concatenate([ga, -ga]), np.concatenate([ha, ha]), dict(min_data_in_leaf=20), 3, expect_leaves=3)
    assert T["left_child"][0] == 1 and T["right_child"][0] == ~1      # the second split (node 1) took leaf 0, not leaf 1


# ---------------------------------------------------------------- categorical
@pytest.mark.parametrize("ncat,onehot", [(3, 4), (4, 4), (5, 4)])
def test_categorical_one_hot_boundary(built, ncat, onehot):
    """num_bin <= max_cat_to_onehot searches one-vs-rest; one category (bin) more switches to many-vs-many"""
    rng = np.random.default_rng(ncat)
    n = 4000
    c = rng.integers(0, ncat, n).astype(np.float64)
    eff = np.array([-1.0, 1.5, 0.3125, -0.625, 0.8125])[:ncat]
    g = eff[c.astype(int)] + tc.grid(rng, -0.25, 0.25, n)
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([c, rng.integers(0, 5, n).astype(np.float64)], axis=1)
    _check(X, g, h, dict(min_data_in_leaf=20, max_cat_to_onehot=onehot, min_data_per_group=20, cat_smooth=5.0), 3, cat=(0,))


@pytest.mark.parametrize("params", [dict(), dict(max_cat_threshold=3), dict(min_data_per_group=150), dict(cat_l2=0.5, cat_smooth=20.0),
                                    dict(cat_smooth=30.0)])
def test_categorical_many_vs_many(built, params):
    """20 categories of 40..400 rows whose effects rank differently from their bins: max_cat_threshold binding, min_data_per_group
    ending the walk and skipping groups, cat_l2 in the leaf outputs, cat_smooth as the row threshold of a used bin (one category holds
    exactly 30 rows)"""
    rng = np.random.default_rng(17)
    sizes = rng.integers(40, 400, 20)
    sizes[5] = 30
    c = np.repeat(np.arange(20, dtype=np.float64), sizes)
    eff = _on_grid(rng.permutation(np.linspace(-2, 2, 20)))
    g = eff[c.astype(int)] + tc.grid(rng, -0.5, 0.5, len(c))
    h = np.ones(len(c))
    X = np.stack([c, rng.integers(0, 5, len(c)).astype(np.float64)], axis=1)
    p = dict(min_data_in_leaf=20)
    p.update(params)
    _check(X, g, h, p, 4, cat=(0,))


def test_categorical_ctr_ties_are_stable_by_bin(built):
    """categories with identical (g, h) sums have equal ctr: the sort keeps them in bin order"""
    rng = np.random.default_rng(23)
    base = np.repeat(np.arange(12, dtype=np.float64), 100)
    eff = np.array([-2, -1, -1, -1, 0.5, 0.5, 1, 1, 1, 2, -0.25, 0.25])
    g = eff[base.astype(int)] + np.tile(np.arange(100) % 5 - 2, 12) * GRID * 8
    X = np.stack([base, np.tile(np.arange(100) % 3, 12).astype(np.float64)], axis=1)
    _check(X, g, np.ones(len(g)), dict(min_data_in_leaf=20, min_data_per_group=50, max_cat_threshold=2), 3, cat=(0,))


def test_wide_categorical(built):
    """more than 256 categories (min_data_in_bin=1): k_scan_wide's categorical search"""
    rng = np.random.default_rng(29)
    ncat = 600
    c = np.repeat(np.arange(ncat, dtype=np.float64), rng.integers(10, 40, ncat))
    eff = _on_grid(rng.permutation(np.linspace(-2, 2, ncat)))
    g = eff[c.astype(int)] + tc.grid(rng, -0.25, 0.25, len(c))
    X = np.stack([c, rng.integers(0, 5, len(c)).astype(np.float64)], axis=1)
    _check(X, g, tc.grid(rng, 0.75, 1.25, len(c)), dict(min_data_in_leaf=20, min_data_per_group=30), 3, ds_params="min_data_in_bin=1", cat=(0,))


def test_wide_categorical_selection_list_overflow(built):
    """k_scan_wide selects the max_cat_threshold smallest and largest ctr keys through a <= 512-entry candidate list.  Adversarial layout
    as in test_wide_categorical_selection_list_overflow_falls_back, on the exact grid: more than 512 bins owned by 31 of the 256 threads
    (bin % 256 < 31) carry the small keys, the list overflows and the round-based fallback selection must agree with the stable sort"""
    from mmlspark_b200 import capi
    rng = np.random.default_rng(11)
    ncat, per = 5200, 12
    cat = np.repeat(np.arange(ncat), per).astype(np.float64)
    rng.shuffle(cat)
    X = np.stack([cat, rng.integers(0, 5, len(cat)).astype(np.float64)], axis=1)
    dsp = "max_bin=255 min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0 min_data_in_bin=1 categorical_feature=0"
    ds = capi.Dataset.from_mat(X, dsp)
    bins = ds.get_bins16()[:, 0].astype(np.int64)
    ds.free()
    low = ((bins % 256) < 31) & ((bins // 256) < 20) & (bins > 0)
    assert len(np.unique(bins[low])) > 512
    noise = _on_grid(rng.standard_normal(int(bins.max()) + 1) * 0.05)       # distinct-ish ctr per category; equal keys sort by bin
    g = np.where(low, -5.0, 5.0) + noise[bins] + tc.grid(rng, -0.01, 0.01, len(cat))
    T, _ = _check(X, g, np.ones(len(cat)), dict(min_data_in_leaf=5, min_data_per_group=10, cat_smooth=10.0), 3,
                  ds_params="min_data_in_bin=1", cat=(0,))
    assert T["is_cat"][0]


def test_categorical_parameters_round_trip_in_the_model(built):
    """the parameter block reports the categorical parameters the scan ran with"""
    X, g, h = _step_case(20, 9, seed=4)
    p = dict(min_data_in_leaf=10, cat_l2=2.5, cat_smooth=5.0, max_cat_threshold=7, max_cat_to_onehot=6, min_data_per_group=33)
    _, text = _check(X, g, h, p, 2, cat=(1,))
    for k in ("cat_l2: 2.5", "cat_smooth: 5", "max_cat_threshold: 7", "max_cat_to_onehot: 6", "min_data_per_group: 33"):
        assert "[%s]" % k in text


# ---------------------------------------------------------------- is_splittable inheritance
def test_feature_without_root_split_is_not_split_in_children(built):
    """feature 1's gradients cancel at the root (its gain stays below min_gain_to_split), but inside the child a == 0 it would split
    with a gain of about 270.  Its is_splittable flag from the root is inherited, so the children are not split on it."""
    rng = np.random.default_rng(33)
    n = 6000
    a = np.repeat([0.0, 1.0], n // 2)
    b = np.tile(np.where(np.arange(n // 2) < 300, 1.0, 0.0), 2)
    g = np.where(a == 0, -1.0, 1.0) * np.where(b == 1, 2.0, 1.0) + tc.grid(rng, -0.125, 0.125, n)
    X = np.stack([a, b], axis=1)
    T, _ = _check(X, g, np.ones(n), dict(min_data_in_leaf=20, min_gain_to_split=100.0), 3, expect_leaves=2)
    assert not T["rounds"][0][0][2][1].splittable
