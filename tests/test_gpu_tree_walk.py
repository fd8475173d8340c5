"""Every tree walk of the engine against the NumPy restatement of LightGBM's decision rules (tree_walk_ref).

a. A hand-written multiclass forest with every kind of node, at rows on every edge of its decisions: the device dense predictor on
   float64 rows, on float32 rows and from a device pointer, the device CSR predictor with explicit values, explicit zeros and omitted
   entries, and the host predictor give the restatement's leaf indices exactly and its raw scores bit for bit, and brute-force Shapley
   values to 1e-10.  There are enough rows that the grid-stride loops of k_predict_* and k_csr_to_slots wrap.
b. The engine's own models (gbdt regression, binary and 3-class multiclass, rf, dart) on data whose walks meet edges: the validation
   scores (k_add_tree_binned on the validation bins) follow the restatement's walk on bins, the predictors follow its walk on raw values,
   the two agree wherever LightGBM's two walks agree, and the training scores equal the predictions on the training rows."""
import ctypes as C

import numpy as np
import pytest

import tree_walk_ref as R

pytestmark = pytest.mark.gpu

TYPES = ("PREDICT_LEAF_INDEX", "PREDICT_RAW_SCORE", "PREDICT_NORMAL", "PREDICT_CONTRIB")
RANGES = [(0, -1), (1, 1)]


# the largest grid predictor.cu launches is min(ceil(work / 256), 16 blocks per SM) blocks of 256 threads; 160 SMs is more than an H100
# (132) or a B200 (148) has, so a batch of more rows than this many threads wraps every grid-stride loop of the predict kernels
GRID_THREADS_BOUND = 160 * 16 * 256


def _predict_from_device_pointer(capi, b, X, pt, s, k):
    buf = capi.DeviceBuffer(X.nbytes)
    try:
        capi.memcpy(buf.ptr, X.ctypes.data, X.nbytes)
        n = C.c_int64(0)
        capi.check(capi.load().LGBM_BoosterCalcNumPredict(b.handle, C.c_int(X.shape[0]), C.c_int(pt), C.c_int(s), C.c_int(k), C.byref(n)))
        out = np.full(n.value, np.nan)
        ms = C.c_double(0)
        code = capi.DTYPE_FLOAT32 if X.dtype == np.float32 else capi.DTYPE_FLOAT64
        capi.check(capi.load().B200GBM_BoosterPredictForMatDevice(
            b.handle, buf.ptr, C.c_int(code), C.c_int64(X.shape[0]), C.c_int32(X.shape[1]), C.c_int(pt), C.c_int(s), C.c_int(k), C.byref(n),
            out.ctypes.data_as(C.POINTER(C.c_double)), C.byref(ms)))
        return out.reshape(X.shape[0], -1)
    finally:
        buf.free()


def _csr(X):
    """even rows store every entry (zeros included), odd rows omit their zeros; NaN is always stored"""
    keep = (X != 0) | np.isnan(X) | (np.arange(len(X)) % 2 == 0)[:, None]
    rows, cols = np.nonzero(keep)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=len(X)))]).astype(np.int64)
    return indptr, cols.astype(np.int32), np.ascontiguousarray(X[rows, cols])


def _softmax(r):
    e = np.exp(r - r.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


# ---------------------------------------------------------------- a. the hand-written forest
def test_hand_written_forest_on_every_predictor(built):
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    text = R.hand_forest_text()
    trees, K, F = parse_model(text)["trees"], R.HAND_K, R.HAND_NUM_FEATURE
    D = R.edge_rows(trees, F, R.HAND_BASE_ROWS)                          # distinct rows; the batches repeat them
    exact32 = np.all((D.astype(np.float32).astype(np.float64) == D) | np.isnan(D), axis=1)
    assert exact32.sum() > 50 and (~exact32).sum() > 50
    b = capi.Booster(model_str=text)
    for s, k in RANGES:
        leaves = R.leaf_indices(trees, D, K, s, k)
        raw = R.scores_from_leaves(trees, leaves, K, s, k)
        contrib = np.array([R.contributions(trees, x, F, K, s, k) for x in D])
        want = {capi.PREDICT_LEAF_INDEX: leaves, capi.PREDICT_RAW_SCORE: raw, capi.PREDICT_CONTRIB: contrib}
        for rows, tag in ((D, "float64"), (D[exact32].astype(np.float32), "float32")):
            reps = GRID_THREADS_BOUND // len(rows) + 1                      # more rows than threads: every grid-stride loop wraps
            X = np.ascontiguousarray(np.tile(rows, (reps, 1)))
            sel = np.tile(np.arange(len(D)) if tag == "float64" else np.nonzero(exact32)[0], reps)
            for name in TYPES:
                pt = getattr(capi, name)
                msg = "%s %s %d %d" % (tag, name, s, k)
                host = b.predict_for_mat(X, pt, s, k)
                got = {"dense": b.predict_device(X, pt, s, k), "device pointer": _predict_from_device_pointer(capi, b, X, pt, s, k)}
                if tag == "float64":
                    ip, ix, v = _csr(X)
                    got["csr"] = b.predict_csr_device(ip, ix, v, F, pt, s, k)
                for path, g in got.items():
                    if pt == capi.PREDICT_CONTRIB:
                        np.testing.assert_allclose(g, want[pt][sel], rtol=0, atol=1e-10, err_msg=path + " " + msg)
                        np.testing.assert_allclose(g, host, rtol=0, atol=1e-12, err_msg=path + " " + msg)      # host TreeSHAP does not fuse multiply-adds
                    else:
                        np.testing.assert_array_equal(g, host, err_msg=path + " " + msg)
                if pt == capi.PREDICT_NORMAL:
                    np.testing.assert_allclose(host, _softmax(raw[sel]), rtol=1e-14, atol=0, err_msg=msg)
                elif pt == capi.PREDICT_CONTRIB:
                    np.testing.assert_allclose(host, want[pt][sel], rtol=0, atol=1e-10, err_msg="host " + msg)
                else:
                    np.testing.assert_array_equal(host, want[pt][sel], err_msg="host " + msg)


# ---------------------------------------------------------------- b. the engine's own models: binned walks against the raw walk
CAT, WIDE_CAT, WIDE_NUM, SPARSE = 2, 3, 4, (5, 6)
DS = "max_bin=511 min_data_in_bin=1 is_pre_partition=True num_threads=0 categorical_feature=2,3"
PARAMS = ("num_leaves=15 learning_rate=0.2 min_data_in_leaf=5 verbosity=-1 categorical_feature=2,3 min_data_per_group=10 cat_smooth=2 "
          "max_cat_threshold=64")


def _train_data(rng, n):
    """f0 numerical with NaN (missing type NaN); f1 numerical without NaN (missing type None); f2 categorical 0..5, every category
    frequent (missing type None), category 0 carrying the largest effect; f3 categorical with 400 categories (> 256 bins); f4 numerical
    with hundreds of distinct values (> 256 bins under max_bin=511); f5, f6 sparse and mutually exclusive (one bundle)"""
    X = np.zeros((n, 7))
    X[:, 0] = np.round(rng.standard_normal(n), 1)
    X[rng.random(n) < 0.1, 0] = np.nan
    X[:, 1] = np.round(rng.standard_normal(n), 1)
    X[:, CAT] = rng.integers(0, 6, n)
    X[:, WIDE_CAT] = rng.integers(0, 400, n)
    X[:, WIDE_NUM] = rng.standard_normal(n)
    u = rng.random(n)
    X[u < 0.06, 5] = rng.integers(1, 20, (u < 0.06).sum()) * 0.37
    X[(u >= 0.06) & (u < 0.12), 6] = -rng.integers(1, 20, ((u >= 0.06) & (u < 0.12)).sum()) * 0.29
    eff = rng.standard_normal(400)
    y = (1.5 * np.nan_to_num(X[:, 0], nan=-2.0) - X[:, 1] + np.array([3.0, -1.0, 0.5, -0.5, 1.0, 0.0])[X[:, CAT].astype(int)]
         + eff[X[:, WIDE_CAT].astype(int)] + 0.7 * X[:, WIDE_NUM] + 0.5 * X[:, 5] - 0.8 * X[:, 6] + 0.3 * rng.standard_normal(n))
    return X, y


def _metas(ds, F):
    metas = []
    for f in range(F):
        info = ds.feature_info(f)
        metas.append(R.feature_meta(info["num_bin"], info["default_bin"], ds.upper_bounds(f), ds.bin_to_cat(f) if f in (CAT, WIDE_CAT) else None))
    return metas


def _validation_rows(ds, base):
    """training-like rows, then each numerical feature on every bin bound and one ulp either side, plus NaN, +-inf, +-1e308 and
    1e300's neighbours; each categorical feature at NaN, negative, fractional, huge, unseen and every seen category.  A sparse feature
    of the bundle is set with its partner at 0, so no row breaks the bundle's exclusivity."""
    rows = [r for r in base]
    k = 0

    def put(f, v):
        nonlocal k
        r = base[k % len(base)].copy()
        k += 1
        r[f] = v
        if f in SPARSE:
            r[SPARSE[1] if f == SPARSE[0] else SPARSE[0]] = 0.0
        rows.append(r)
    for f in (0, 1, WIDE_NUM) + SPARSE:
        ub = ds.upper_bounds(f)
        for u in ub[np.isfinite(ub)]:
            for v in (u, np.nextafter(u, -np.inf), np.nextafter(u, np.inf)):
                put(f, v)
        for v in (np.nan, np.inf, -np.inf, 1e308, -1e308, 1e300, np.nextafter(1e300, np.inf), -0.0, 0.0, R.SUBNORMAL, -R.SUBNORMAL):
            put(f, v)
    for f, unseen in ((CAT, (6.0, 7.0, 1000.0)), (WIDE_CAT, (400.0, 401.0, 5000.0))):
        for v in R.CATEGORY_EDGES + unseen + tuple(float(c) for c in ds.bin_to_cat(f) if c >= 0):
            put(f, v)
    return np.array(rows)


def _first_divergence(tree, x, bins, metas):
    """the node where the raw and the binned walk of a row part, or None"""
    node = 0
    while node >= 0:
        f = int(tree["split_feature"][node])
        a, b = R.decide(tree, node, x[f]), R.decide_bin(tree, node, bins[f], metas[f])
        if a != b:
            return node
        node = a
    return None


RUNS = {
    "regression": "objective=regression",
    "binary": "objective=binary",
    "multiclass": "objective=multiclass num_class=3",
    "rf": "objective=regression boosting_type=rf bagging_fraction=0.7 bagging_freq=1 feature_fraction=0.8",
    "dart": "objective=regression boosting_type=dart drop_rate=0.3 skip_drop=0.0 max_drop=3",
}


@pytest.fixture(scope="module")
def edge_data(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(2024)
    X, y = _train_data(rng, 20000)
    ds = capi.Dataset.from_mat(X, DS)
    F = X.shape[1]
    Xb, _ = _train_data(rng, 300)
    return dict(X=X, y=y, ds=ds, Xv=_validation_rows(ds, Xb), F=F)


def test_edge_data_meets_the_edges(edge_data):
    ds = edge_data["ds"]
    assert ds.feature_info(0)["missing_type"] == R.MISSING_NAN and ds.feature_info(1)["missing_type"] == R.MISSING_NONE
    assert ds.feature_info(CAT)["missing_type"] == R.MISSING_NONE
    assert ds.feature_info(WIDE_CAT)["num_bin"] > 256 and ds.feature_info(WIDE_NUM)["num_bin"] > 256
    _, column = ds.bundles()
    assert column[SPARSE[0]] == column[SPARSE[1]] >= 0
    assert np.isnan(edge_data["Xv"][:, 1]).any() and not np.isnan(edge_data["X"][:, 1]).any()


@pytest.mark.parametrize("run", list(RUNS))
def test_binned_walks_agree_with_the_raw_walk(edge_data, run):
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    X, y, Xv, F = (edge_data[k] for k in ("X", "y", "Xv", "F"))
    K = 3 if run == "multiclass" else 1
    label = (y > np.median(y)) if run == "binary" else np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])) if K == 3 else y
    ds = capi.Dataset.from_mat(X, DS).set_field("label", label.astype(np.float32))
    dv = capi.Dataset.from_mat(Xv, DS, reference=ds)
    metas, vbins = _metas(ds, F), dv.get_bins_rows(np.arange(len(Xv)))
    b = capi.Booster(ds, RUNS[run] + " " + PARAMS)
    b.add_valid(dv)
    for _ in range(8):
        b.update_one_iter()
    text = b.save_model_to_string()
    trees = parse_model(text)["trees"]
    avg = "\naverage_output\n" in text
    # zero_as_missing is rejected, so no trained node has missing type Zero: that is why k_add_tree_binned has no Zero branch
    dts = np.concatenate([t["decision_type"] for t in trees if t["num_leaves"] > 1])
    assert set(((dts >> 2) & 3).tolist()) <= {R.MISSING_NONE, R.MISSING_NAN}
    if run == "regression":                       # the data reaches the edges it was built for
        used = {(int(t["split_feature"][n]), bool(t["decision_type"][n] & 1)) for t in trees for n in range(t["num_leaves"] - 1)}
        assert {(CAT, True), (WIDE_CAT, True), (WIDE_NUM, False), (0, False), (1, False)} <= used
        assert any(R.is_categorical(t, n) and int(t["split_feature"][n]) == CAT and R.missing_type(t, n) == R.MISSING_NONE
                   and R.in_bitset(R.cat_words(t, n), 0) for t in trees for n in range(t["num_leaves"] - 1))
    # the raw walk: the predictors give the restatement's leaves and its sums bit for bit
    leaves = R.leaf_indices(trees, Xv, K)
    raw = R.scores_from_leaves(trees, leaves, K, average=avg)
    for pt, want in ((capi.PREDICT_LEAF_INDEX, leaves), (capi.PREDICT_RAW_SCORE, raw)):
        np.testing.assert_array_equal(b.predict_device(Xv, pt), want, err_msg="device %d" % pt)
        np.testing.assert_array_equal(b.predict_for_mat(Xv, pt), want, err_msg="host %d" % pt)
    # the binned walk: the validation scores are the restatement's sums over the leaves decide_bin reaches
    bleaves = np.array([[R.bin_leaf_index(t, vb, metas) for t in trees] for vb in vbins], dtype=np.float64)
    valid = b.get_scores(1).reshape(K, -1).T
    np.testing.assert_allclose(valid, R.scores_from_leaves(trees, bleaves, K, average=avg), rtol=0, atol=1e-9)
    # the walks agree wherever LightGBM's agree: the one known split is a value above 1e300 at a bound of +inf, written as 1e300 (AvoidInf),
    # which the bins send left and the raw value right
    same = (bleaves == leaves).all(axis=1)
    for i, t in zip(*np.nonzero(bleaves != leaves)):
        node = _first_divergence(trees[t], Xv[i], vbins[i], metas)
        f = int(trees[t]["split_feature"][node])
        assert not R.is_categorical(trees[t], node) and trees[t]["threshold"][node] == 1e300 and Xv[i, f] > 1e300, (i, t, node, Xv[i, f])
    np.testing.assert_allclose(valid[same], raw[same], rtol=0, atol=1e-9)
    assert same.mean() > 0.95
    # the training scores (the final partition, or the bins for rf and dart) equal the predictions on the training rows
    np.testing.assert_allclose(b.get_scores(0).reshape(K, -1).T, b.predict_device(X, capi.PREDICT_RAW_SCORE), rtol=0, atol=1e-9)
