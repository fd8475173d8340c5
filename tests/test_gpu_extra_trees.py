"""Extremely randomised trees (extra_trees, extra_seed): the scans' kExtra instantiations (k_scan, k_scan_wide) and the per-feature streams
the pick step advances, tree by tree and tree after tree, against the NumPy restatement in extra_trees_ref.py.

As in test_gpu_split_scan.py, gradients and hessians lie on a 2^-10 grid with few enough rows that K4's fixed-point histograms equal
NumPy's fp64 ones bit for bit, so only the scans, the draws and the pick are under test.  Every tree of a run is grown from the same
custom (g, h) through UpdateOneIterCustom: the trees differ only by the streams' state, which carries from tree to tree.

Bar: identical structure (feature, threshold bin, default direction, category set, counts), leaf values within 4 fp64 ulps, split gains
as printed.  Every tree must be decided on the reference side (split_scan_ref.undecided)."""
import threading

import numpy as np
import pytest

import extra_trees_ref as X3
import split_scan_ref as ref

pytestmark = pytest.mark.gpu

GRID = 1.0 / 1024
DS = "min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0"


def _grid(rng, lo, hi, n):
    return rng.integers(int(lo * 1024), int(hi * 1024) + 1, n) * GRID


def _data(seed, n=6000, cat=False, wide=False, const_h=False):
    """numerical features (one with NaN), optionally a one-hot (3 categories) and a many-vs-many (40 categories) categorical feature, or
    two numerical features of ~500 bins and a categorical one of 600 categories (max_bin=511)"""
    rng = np.random.default_rng(seed)
    cols = [rng.integers(0, 60, n).astype(np.float64), rng.standard_normal(n), rng.integers(0, 9, n).astype(np.float64)]
    cols[1][rng.random(n) < 0.15] = np.nan
    if cat:
        cols += [rng.integers(0, 3, n).astype(np.float64), rng.integers(0, 40, n).astype(np.float64)]
    if wide:
        cols += [rng.integers(0, 500, n).astype(np.float64), rng.standard_normal(n), rng.integers(0, 600, n).astype(np.float64)]
    X = np.stack(cols, axis=1)
    y = 0.02 * X[:, 0] + np.nan_to_num(X[:, 1]) + (X[:, 2] > 4)
    if cat:
        y += 0.8 * (X[:, 3] == 1) + 0.05 * (X[:, 4] % 7)
    if wide:
        w = 5 if cat else 3
        y += 0.004 * X[:, w] + 4.0 * (X[:, w + 2] % 3 == 0)
    g = np.round((-y + 0.3 * rng.standard_normal(n)) / GRID) * GRID
    h = np.ones(n) if const_h else _grid(rng, 0.5, 1.5, n)
    cats = ([3, 4] if cat else []) + ([7 if cat else 5] if wide else [])
    return X, g, h, cats


def _features(ds, F, cats):
    infos = [ds.feature_info(f) for f in range(F)]
    return [ref.Feature(f, infos[f]["num_bin"], infos[f]["missing_type"], int(infos[f]["most_freq_bin"] == 0), f in cats)
            for f in range(F) if not infos[f]["is_trivial"]]


def _params(num_leaves, extra, cats=(), max_bin=255):
    p = ("objective=regression boost_from_average=false learning_rate=1 verbosity=-1 num_leaves=%d min_data_in_leaf=20 max_bin=%d %s %s"
         % (num_leaves, max_bin, DS, extra))
    if cats:
        p += " categorical_feature=" + ",".join(str(c) for c in cats)
    return p


def _ds_params(cats, max_bin):
    return DS + " max_bin=%d" % max_bin + (" categorical_feature=" + ",".join(str(c) for c in cats) if cats else "")


def _run(X, g, h, params, iters, ds_params, reset=None):
    """the model text of `iters` trees on the same custom (g, h); reset = (after tree k, parameter string) calls ResetParameter"""
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, ds_params).set_field("label", np.zeros(len(X), np.float32))
    b = capi.Booster(ds, params)
    try:
        for k in range(iters):
            b.update_one_iter_custom(g.astype(np.float32), h.astype(np.float32))
            if reset is not None and reset[0] == k:
                b.reset_parameter(reset[1])
        return b.save_model_to_string()
    finally:
        b.free(); ds.free()


def _trees(model):
    return model.split("\nparameters:")[0]


def _split_features(model):
    from mmlspark_b200.modeltext import parse_model
    return {int(f) for t in parse_model(model)["trees"] for f in t["split_feature"]} if "split_feature=" in model else set()


def _ulps(a, b):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) / np.spacing(np.maximum(np.abs(a), np.abs(b)) + 1e-300)


def _compare(t, T, ub, b2c, lr=None):
    assert t["num_leaves"] == T["num_leaves"], (t["num_leaves"], T["num_leaves"])
    nl = T["num_leaves"]
    if nl > 1:
        assert t["split_feature"].tolist() == T["split_feature"], (t["split_feature"], T["split_feature"])
        assert t["left_child"].tolist() == T["left_child"] and t["right_child"].tolist() == T["right_child"]
        for i in range(nl - 1):
            f, dt = T["split_feature"][i], int(t["decision_type"][i])
            assert bool(dt & 1) == T["is_cat"][i], "node %d: categorical flag" % i
            if T["is_cat"][i]:
                k = int(t["threshold"][i])
                words = t["cat_threshold"][t["cat_boundaries"][k]:t["cat_boundaries"][k + 1]]
                cats = {32 * w + j for w, word in enumerate(words) for j in range(32) if (int(word) >> j) & 1}
                got = {b for b, c in enumerate(b2c[f]) if b > 0 and c in cats}
                assert got == set(T["cat_bins"][i]), "node %d: category bins %s vs %s" % (i, sorted(got), sorted(T["cat_bins"][i]))
            else:
                hit = np.nonzero(ub[f] == t["threshold"][i])[0]
                assert len(hit) == 1 and hit[0] == T["threshold_bin"][i], "node %d: threshold bin %s vs %d" % (i, hit, T["threshold_bin"][i])
                assert bool(dt & 2) == T["default_left"][i], "node %d: default_left" % i
            assert t["split_gain"][i] == float("%g" % T["split_gain"][i]), (i, t["split_gain"][i], T["split_gain"][i])
        assert t["leaf_count"].tolist() == T["leaf_count"] and t["internal_count"].tolist() == T["internal_count"]
    if lr is None:
        assert (_ulps(t["leaf_value"], T["leaf_value"]) <= 4).all(), (t["leaf_value"], T["leaf_value"])
    else:       # shrunk by the learning rate
        np.testing.assert_allclose(t["leaf_value"], np.asarray(T["leaf_value"]) * lr, rtol=1e-12, atol=1e-300)


def _check_run(X, g, h, cats, num_leaves, iters, extra_seed, max_bin=255, extra="", fraction=1.0, reset=None, restart_after=None):
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    dsp = _ds_params(cats, max_bin)
    params = _params(num_leaves, "extra_trees=true extra_seed=%d %s" % (extra_seed, extra), cats, max_bin)
    model = _run(X, g, h, params, iters, dsp, reset)
    ds = capi.Dataset.from_mat(X, dsp).set_field("label", np.zeros(len(X), np.float32))
    try:
        feats = _features(ds, X.shape[1], cats)
        bins = ds.get_bins16()
        ub = {f.real_index: ds.upper_bounds(f.real_index) for f in feats}
        b2c = {f.real_index: ds.bin_to_cat(f.real_index) for f in feats if f.is_cat}
    finally:
        ds.free()
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(min_data_in_leaf=20, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS})
    trees = parse_model(model)["trees"]
    assert len(trees) == iters
    used = X3.feature_fraction_sets(len(feats), fraction, 2, iters)
    streams = X3.Streams(feats, extra_seed)
    shapes = set()
    for k in range(iters):
        if restart_after is not None and k == restart_after + 1:
            streams = X3.Streams(feats, extra_seed)      # ResetParameter re-seeds every stream
        T = X3.grow_tree(bins, g, h, feats, p, num_leaves, True, extra_seed, streams, {feats[i].real_index for i in used[k]})
        why = ref.undecided(T)
        assert not why, "tree %d does not discriminate:\n%s" % (k, "\n".join(why[:10]))
        _compare(trees[k], T, ub, b2c)
        shapes.add((tuple(T["split_feature"]), tuple(T["threshold_bin"])))
    return model, shapes


# ---------------------------------------------------------------- tree after tree against the restatement
@pytest.mark.parametrize("seed", [6, 11, 12345])
def test_numerical_with_nan(built, seed):
    X, g, h, cats = _data(1)
    _, shapes = _check_run(X, g, h, cats, 8, 5, seed)
    assert len(shapes) > 1, "the streams must carry from tree to tree"


@pytest.mark.parametrize("seed", [6, 99])
def test_one_hot_and_many_vs_many(built, seed):
    X, g, h, cats = _data(2, cat=True)
    model, _ = _check_run(X, g, h, cats, 12, 5, seed, extra="min_data_per_group=20 cat_smooth=5")
    assert "cat_threshold=" in model, "the case must split on a categorical feature"


def test_feature_fraction(built):
    X, g, h, cats = _data(3, cat=True)
    _check_run(X, g, h, cats, 8, 6, 7, extra="feature_fraction=0.6 min_data_per_group=20 cat_smooth=5", fraction=0.6)


def test_wide_features(built):
    """max_bin=511: k_scan_wide's numerical scan and a categorical feature of 600 categories"""
    X, g, h, cats = _data(4, n=9000, wide=True)
    model, _ = _check_run(X, g, h, cats, 8, 4, 6, max_bin=511, extra="min_data_per_group=20 cat_smooth=5")
    assert _split_features(model) >= {3, 5}, "the case must split on the wide numerical and the wide categorical feature"


def test_reset_parameter_restarts_the_streams(built):
    """ResetParameter re-seeds every stream (LightGBM 3.2's HistogramPool::ResetConfig): the trees after a reset repeat those after
    the booster's creation"""
    X, g, h, cats = _data(5)
    model, _ = _check_run(X, g, h, cats, 8, 4, 6, reset=(1, "learning_rate=1"), restart_after=1)
    trees = _trees(model).split("Tree=")[1:]
    assert trees[0].split("\n", 1)[1] == trees[2].split("\n", 1)[1]


# ---------------------------------------------------------------- two ranks on one device
def _on_ranks(R, base_port, body, device_of=lambda r: 0):
    from mmlspark_b200 import capi
    machines = ",".join("127.0.0.1:%d" % (base_port + r) for r in range(R))
    out, errs = [None] * R, []

    def task(r):
        try:
            capi.set_device(device_of(r))
            capi.network_init(machines, base_port + r, 120, R)
            try:
                out[r] = body(r)
            finally:
                capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, str(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(R)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(300)
    assert not any(t.is_alive() for t in ts), "a rank-thread did not finish"
    return out, errs


def _two_ranks(port, device_of=lambda r: 0):
    """data-parallel on two shards with unit hessians (the reconstructed global counts are exact): the model equals the one-rank model"""
    from mmlspark_b200 import capi
    X, g, h, cats = _data(6, cat=True, const_h=True)
    dsp = _ds_params(cats, 255)
    params = _params(10, "extra_trees=true extra_seed=21 tree_learner=data num_machines=2 min_data_per_group=20 cat_smooth=5", cats)
    half = len(X) // 2

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ref_ds = capi.Dataset.from_mat(X, dsp)      # the bins of the whole data, as one rank would have them
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=ref_ds).set_field("label", np.zeros(half, np.float32))
        b = capi.Booster(ds, params)
        try:
            for _ in range(3):
                b.update_one_iter_custom(g[sl].astype(np.float32), h[sl].astype(np.float32))
            return b.save_model_to_string()
        finally:
            b.free(); ds.free(); ref_ds.free()

    res, errs = _on_ranks(2, port, body, device_of)
    assert not errs, errs
    assert _trees(res[0]) == _trees(res[1])
    single, _ = _check_run(X, g, h, cats, 10, 3, 21, extra="min_data_per_group=20 cat_smooth=5")
    assert _trees(res[0]) == _trees(single)


def test_two_ranks_on_one_device(built):
    _two_ranks(29600)


def test_two_ranks_nccl(built):
    import subprocess
    out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
    if len([l for l in out.splitlines() if l.startswith("GPU ")]) < 2:
        pytest.skip("needs 2 GPUs")
    _two_ranks(29620, device_of=lambda r: r)


def test_voting_rejects_at_create(built):
    from mmlspark_b200 import capi
    X, g, h, cats = _data(7)
    params = _params(8, "extra_trees=true tree_learner=voting top_k=2 num_machines=2")
    half = len(X) // 2

    def body(r):
        ds = capi.Dataset.from_mat(X[r * half:(r + 1) * half], _ds_params((), 255)).set_field("label", np.zeros(half, np.float32))
        try:
            with pytest.raises(Exception) as e:
                capi.Booster(ds, params)
            return str(e.value)
        finally:
            ds.free()

    res, errs = _on_ranks(2, 29640, body)
    assert not errs, errs
    assert all("does not support extra_trees" in m for m in res), res


# ---------------------------------------------------------------- the default stays as it was; seeds, bundles, model text
def test_baseline_seeds_and_model_text(built):
    from mmlspark_b200 import capi
    X, g, h, cats = _data(8, cat=True)
    dsp = _ds_params(cats, 255)
    run = lambda extra: _run(X, g, h, _params(12, extra, cats), 3, dsp)      # noqa: E731
    plain, off = run(""), run("extra_trees=false extra_seed=9")
    assert _trees(plain) == _trees(off)
    a, a2, b = run("extra_trees=true"), run("extra_tree=true extra_seed=6"), run("extra_trees=true extra_seed=7")
    assert _trees(a) == _trees(a2)
    assert _trees(a) != _trees(plain) and _trees(b) != _trees(a)
    assert "[extra_trees: 1]" in a and "[extra_seed: 6]" in a and "[extra_seed: 7]" in b
    assert "[extra_trees: 0]" in plain and "[extra_seed: 6]" in plain
    loaded = capi.Booster(model_str=b)
    try:
        assert loaded.save_model_to_string() == b
    finally:
        loaded.free()


def test_bundles_equal_unbundled(built):
    """sparse mutually exclusive features bundle into one column; the bundle members' scans draw as the plain features' do"""
    rng = np.random.default_rng(9)
    n = 8000
    which = rng.integers(0, 6, n)
    X = np.zeros((n, 8))
    for j in range(6):
        on = which == j
        X[on, j] = rng.integers(1, 12, on.sum())
    X[:, 6] = rng.standard_normal(n)
    X[:, 7] = rng.integers(0, 30, n)
    g = np.round((-(X[:, 0] * 0.2 + X[:, 3] * 0.1 + X[:, 6]) + 0.2 * rng.standard_normal(n)) / GRID) * GRID
    h = _grid(rng, 0.5, 1.5, n)
    models = []
    for bundle in ("true", "false"):
        dsp = DS + " max_bin=255 enable_bundle=" + bundle
        models.append(_run(X, g, h, _params(12, "extra_trees=true extra_seed=3 enable_bundle=" + bundle), 4, dsp))
    assert _trees(models[0]) == _trees(models[1])


def test_estimator(built):
    """LightGBMRegressor(extraTrees=True, extraSeed=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    rng = np.random.default_rng(10)
    n = 5000
    X = rng.standard_normal((n, 6))
    y = X[:, 0] + 0.5 * X[:, 1] ** 2 + 0.1 * rng.standard_normal(n)
    df = Frame({"features": X, "label": y})
    est = LightGBMRegressor(extraTrees=True, extraSeed=17, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert params.endswith("extra_trees=true extra_seed=17 ")
    assert "extra_trees" not in LightGBMRegressor(numIterations=5).getTrainParams(1, df).to_string()
    ds = capi.Dataset.from_mat(X, dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), []))
    ds.set_field("label", y.astype(np.float32))
    b = capi.Booster(ds, params)
    try:
        for _ in range(5):
            b.update_one_iter()
        low = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    assert _trees(model) == _trees(low)
    assert "[extra_trees: 1]" in model and "[extra_seed: 17]" in model


# ---------------------------------------------------------------- a round where only the larger leaf's many-vs-many search draws
@pytest.mark.parametrize("num_cats", [40, 600])
def test_larger_leaf_draws_after_an_empty_smaller_range(built, num_cats):
    """The root splits on a 0/1 feature (2 bins: no draw, one candidate).  In the smaller child the categorical feature holds 2
    categories (max_num_cat = 1: an empty range, no draw); in the larger one it holds `num_cats` (a draw, k_scan's or, for 600
    categories, k_scan_wide's).  The larger leaf's block must not step past a draw the smaller one never took: its prefix, and every later
    draw of the feature, would otherwise differ from the restatement's."""
    rng = np.random.default_rng(num_cats)
    n = 8000 if num_cats == 40 else 12000
    x0 = (rng.random(n) < 0.75).astype(np.float64)
    c = np.where(x0 == 1, rng.integers(0, num_cats, n), rng.integers(0, 2, n)).astype(np.float64)
    x2 = rng.standard_normal(n)
    y = 6.0 * x0 + 2.0 * (c % 2 == 0) * x0 + 0.1 * x2
    g = np.round((-y + 0.2 * rng.standard_normal(n)) / GRID) * GRID
    h = _grid(rng, 0.5, 1.5, n)
    X = np.stack([x0, c, x2], axis=1)
    cats = [1]
    extra = "min_data_per_group=20 cat_smooth=5"
    p = ref.Params(min_data_in_leaf=20, min_data_per_group=20, cat_smooth=5)
    # the premise, on the reference side: root split on feature 0, then an empty range for the smaller child, a non-empty one for the larger
    left, right = x0 == 0, x0 == 1
    for rows, want_draw in ((left, False), (right, True)):
        cb = c[rows].astype(np.int64)
        from mmlspark_b200 import capi
        ds = capi.Dataset.from_mat(X, _ds_params(cats, 255))
        try:
            bins = ds.get_bins16()[rows, 1].astype(np.int64)
            nb = ds.feature_info(1)["num_bin"]
        finally:
            ds.free()
        hh = np.bincount(bins, weights=h[rows], minlength=nb)
        assert (X3.categorical_range(hh, nb, h[rows].sum(), int(rows.sum()), p) > 0) == want_draw, (nb, len(set(cb)))
    model, _ = _check_run(X, g, h, cats, 6, 4, 6, extra=extra)
    from mmlspark_b200.modeltext import parse_model
    trees = parse_model(model)["trees"]
    assert all(int(t["split_feature"][0]) == 0 for t in trees)
    assert any(1 in t["split_feature"].tolist() for t in trees), "the categorical feature must be split on"


# ---------------------------------------------------------------- boosting runs on the engine's own gradients
def _quantized(v):
    """K3's fixed-point grid: q = rint(v * 2^e), e = 34 - ilogb(max |v|); NumPy's fp64 sums of q * 2^-e equal the engine's int64 sums"""
    m = np.float32(np.max(np.abs(v)))
    e = 34 - (int(np.frexp(m)[1]) - 1) if m > 0 and np.isfinite(m) else 0
    return np.rint(v.astype(np.float64) * 2.0 ** e) * 2.0 ** -e


def _bags(n, iters, fraction, seed):
    """GBDT::Bagging with bagging_freq = 1: per 1024-row block an LCG seeded seed + block, row j of a block takes the next draw
    ((x >> 16) & 0x7fff) / 32768 < fraction; the states carry over to the next iteration"""
    blocks = (n + 1023) // 1024
    x = np.arange(blocks, dtype=np.uint64) + np.uint64(seed)
    out = []
    for _ in range(iters):
        take = np.zeros(blocks * 1024, bool)
        for j in range(1024):
            live = j < n - np.arange(blocks) * 1024
            nx = (x * np.uint64(214013) + np.uint64(2531011)) & np.uint64(0xFFFFFFFF)
            x = np.where(live, nx, x)
            take[np.arange(blocks) * 1024 + j] = live & (((x >> np.uint64(16)) & np.uint64(0x7FFF)).astype(np.float64) / 32768.0 < fraction)
        out.append(take[:n])
    return out


def _boost(X, y, params, iters, dsp, rank_rows=None, port=None):
    """trains `iters` iterations on the objective's own gradients, read back before each; rank_rows: data-parallel shards, each rank a
    thread on this device.  Returns the model and, per iteration, the gradients of all rows."""
    from mmlspark_b200 import capi
    rank_rows = rank_rows or [len(X)]
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        full = capi.Dataset.from_mat(X, dsp)
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=full).set_field("label", np.asarray(y[sl], np.float32))
        b = capi.Booster(ds, params)
        try:
            seen = []
            for _ in range(iters):
                seen.append(b.get_gradients())
                b.update_one_iter()
            return b.save_model_to_string(), seen, b.get_info()["constant_hessian"]
        finally:
            b.free(); ds.free(); full.free()

    if len(rank_rows) == 1:
        res = [body(0)]
    else:
        res, errs = _on_ranks(len(rank_rows), port, body)
        assert not errs, errs
        assert all(_trees(r[0]) == _trees(res[0][0]) for r in res)
    grads = [(np.concatenate([r[1][it][0] for r in res]), np.concatenate([r[1][it][1] for r in res])) for it in range(iters)]
    if len(rank_rows) > 1:      # class-major per rank: regroup per class over all rows
        K = len(res[0][1][0][0]) // rank_rows[0]
        grads = [tuple(np.concatenate([r[1][it][j].reshape(K, -1) for r in res], axis=1).reshape(-1) for j in (0, 1)) for it in range(iters)]
    return res[0][0], grads, res[0][2]


def _check_boosting(X, y, objective, K, iters, extra, cats=(), extra_seed=6, fraction=1.0, bag=None, rank_rows=None, port=None):
    """every tree of the run equals extra_trees_ref.grow_tree on the gradients it was grown from (quantised as K3 does), over its bagged
    rows, with the feature streams carried from tree to tree (K trees per iteration share them)"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    lr, num_leaves = 0.3, 12
    dsp = _ds_params(cats, 255)
    params = ("objective=%s boost_from_average=false learning_rate=%g num_leaves=%d min_data_in_leaf=20 verbosity=-1 metric= "
              "extra_trees=true extra_seed=%d %s %s" % (objective, lr, num_leaves, extra_seed, dsp, extra))
    if rank_rows:
        params += " tree_learner=data num_machines=%d" % len(rank_rows)
    model, grads, const_h = _boost(X, y, params, iters, dsp, rank_rows, port)
    ds = capi.Dataset.from_mat(X, dsp)
    try:
        feats = _features(ds, X.shape[1], cats)
        bins = ds.get_bins16()
        ub = {f.real_index: ds.upper_bounds(f.real_index) for f in feats}
        b2c = {f.real_index: ds.bin_to_cat(f.real_index) for f in feats if f.is_cat}
    finally:
        ds.free()
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(min_data_in_leaf=20, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS})
    trees = parse_model(model)["trees"]
    assert len(trees) == iters * K
    used = X3.feature_fraction_sets(len(feats), fraction, 2, iters * K)
    bags = _bags(len(X), iters, bag[0], bag[1]) if bag else None
    streams = X3.Streams(feats, extra_seed)
    for it in range(iters):
        for k in range(K):
            g = grads[it][0].reshape(K, -1)[k]
            h = grads[it][1].reshape(K, -1)[k]
            gq, hq = _quantized(g), (np.ones(len(h)) if const_h else _quantized(h))
            rows = np.arange(len(g)) if bags is None else np.nonzero(bags[it])[0]
            T = X3.grow_tree(bins[rows], gq[rows], hq[rows], feats, p, num_leaves, True, extra_seed, streams,
                             {feats[i].real_index for i in used[it * K + k]})
            _compare(trees[it * K + k], T, ub, b2c, lr)
    return model


def test_boosting_regression_with_nan(built):
    X, g, h, cats = _data(20)
    y = -g
    _check_boosting(X, y, "regression", 1, 5, "")


def test_boosting_binary_categorical(built):
    X, g, h, cats = _data(21, cat=True)
    z = -g + 3.0 * (X[:, 4] % 2 == 0) + 2.0 * (X[:, 3] == 1)
    y = (z > np.median(z)).astype(np.float64)
    model = _check_boosting(X, y, "binary", 1, 5, "min_data_per_group=20 cat_smooth=5", cats)
    assert _split_features(model) >= {3, 4}, "the case must split on the one-hot and the many-vs-many feature"


def test_boosting_multiclass(built):
    X, g, h, cats = _data(22, cat=True)
    y = np.digitize(-g, np.quantile(-g, [1 / 3, 2 / 3])).astype(np.float64)
    _check_boosting(X, y, "multiclass", 3, 3, "num_class=3 min_data_per_group=20 cat_smooth=5", cats)


def test_boosting_bagging_feature_fraction(built):
    X, g, h, cats = _data(23, cat=True)
    _check_boosting(X, -g, "regression", 1, 5, "bagging_fraction=0.6 bagging_freq=1 bagging_seed=7 feature_fraction=0.7 "
                    "min_data_per_group=20 cat_smooth=5", cats, fraction=0.7, bag=(0.6, 7))


def test_boosting_two_ranks_on_one_device(built):
    """data-parallel regression (unit hessians: the reconstructed global counts are exact) on two unequal shards"""
    X, g, h, cats = _data(24, cat=True)
    _check_boosting(X, -g, "regression", 1, 4, "min_data_per_group=20 cat_smooth=5", cats, rank_rows=[3100, 2900], port=29660)


def test_voting_reset_parameter_rejected(built):
    """a ResetParameter that turns extra_trees on under multi-rank voting fails on every rank and changes nothing"""
    from mmlspark_b200 import capi
    X, g, h, cats = _data(25)
    params = _params(8, "tree_learner=voting top_k=2 num_machines=2 boost_from_average=false")
    half = len(X) // 2

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], _ds_params((), 255)).set_field("label", np.asarray(-g[sl], np.float32))
        b = capi.Booster(ds, params)
        try:
            b.update_one_iter()
            with pytest.raises(Exception) as e:
                b.reset_parameter("extra_trees=true")
            b.update_one_iter()
            return str(e.value), b.save_model_to_string()
        finally:
            b.free(); ds.free()

    res, errs = _on_ranks(2, 29680, body)
    assert not errs, errs
    assert all("does not support extra_trees" in m for m, _ in res), res
    assert all("[extra_trees: 0]" in t for _, t in res) and _trees(res[0][1]) == _trees(res[1][1])
