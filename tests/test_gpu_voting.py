"""Voting-parallel training (tree_learner=voting / parallelism="voting_parallel", LightGBM's VotingParallelTreeLearner): every rank scans its
local histograms, the ranks vote on top_k features per leaf, and only the voted features' histograms are all-reduced and scanned globally.

All ranks are rank-threads of this process on device 0 (the same-device communicator), so every test runs on one GPU; the NCCL variant
runs one rank per GPU and is skipped with fewer than two.  Trees are pinned against the NumPy restatement in voting_ref.py (grown by
tree_ref.py, compared at the bar tree_check.py describes) on custom gradients and hessians on a 2^-10 grid (as test_gpu_split_scan.py does for the serial scan): K4's fixed-point quantisation is exact there,
so the local and the reduced int64 histograms equal NumPy's fp64 ones bit for bit and only the scans, the vote and the pick are under test."""
import subprocess

import numpy as np
import pytest

import split_scan_ref as ref
import tree_check as tc
import tree_ref

pytestmark = pytest.mark.gpu

GRID = 1.0 / 1024
DS = "max_bin=63 min_data_in_bin=3 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"


def _ngpu():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return len([l for l in out.splitlines() if l.startswith("GPU ")])
    except Exception:
        return 0


def _skewed(seed, rank_rows, F=30, per_rank=5, nan_feature=29):
    """rank r's labels are driven by its own features [r*per_rank, (r+1)*per_rank) (coefficient 1), every rank's also by the shared
    feature R*per_rank (0.9): each rank prefers its own features locally, the pooled data the shared one.  Feature `nan_feature` holds NaN."""
    rng = np.random.default_rng(seed)
    R, n = len(rank_rows), int(sum(rank_rows))
    X = rng.standard_normal((n, F))
    X[:, nan_feature] = np.where(rng.random(n) < 0.2, np.nan, X[:, nan_feature])
    rank_of_row = np.repeat(np.arange(R), rank_rows)
    y = 0.9 * X[:, R * per_rank] + 0.3 * rng.standard_normal(n)
    for r in range(R):
        on = rank_of_row == r
        y[on] += X[on][:, r * per_rank:(r + 1) * per_rank].sum(axis=1)
    return X, y, rank_of_row


def _params(objective, R, learner, top_k, extra=""):
    return ("objective=%s tree_learner=%s top_k=%d num_machines=%d num_leaves=15 learning_rate=0.1 min_data_in_leaf=20 "
            "min_sum_hessian_in_leaf=0.001 boost_from_average=true verbosity=-1 metric= %s %s" % (objective, learner, top_k, R, DS, extra))


def _train(X, y, rank_rows, params, iters, port, device_of=lambda r: 0, grads=None, ds_params=DS):
    """every rank trains on its contiguous shard; grads = (g, h) over all rows trains one iteration on custom gradients"""
    from mmlspark_b200 import capi
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        ds = capi.Dataset.from_mat(X[sl], ds_params).set_field("label", np.asarray(y[sl], np.float32))
        b = capi.Booster(ds, params)
        try:
            seen = []      # the objective's (g, h) at the scores each iteration starts from
            if grads is not None:
                b.update_one_iter_custom(grads[0][sl].astype(np.float32), grads[1][sl].astype(np.float32))
            else:
                for _ in range(iters):
                    seen.append(b.get_gradients())
                    if b.update_one_iter():
                        break
            F = X.shape[1]
            infos = [ds.feature_info(f) for f in range(F)]
            return dict(model=b.save_model_to_string(), scores=b.get_scores(), comm=b.get_comm_info(), bins=ds.get_bins16(), infos=infos,
                        ub={f: ds.upper_bounds(f) for f in range(F)}, b2c={f: ds.bin_to_cat(f) for f in _categorical(ds_params)},
                        grads=seen, info=b.get_info(), bundles=ds.bundles())
        finally:
            b.free(); ds.free()

    res, errs = tc.on_ranks(len(rank_rows), port, body, device_of)
    assert not errs, errs
    return res


def _categorical(ds_params):
    return [int(c) for tok in ds_params.split() if tok.startswith("categorical_feature=") for c in tok.split("=")[1].split(",")]


def _grid_gradients(y, seed):
    rng = np.random.default_rng(seed)
    g = np.round(-np.clip(y, -30, 30) / GRID) * GRID
    h = rng.integers(512, 1537, len(y)) * GRID
    return g, h


def _features(res, F, cat=()):
    infos = res[0]["infos"]
    return [ref.Feature(f, infos[f]["num_bin"], infos[f]["missing_type"], int(infos[f]["most_freq_bin"] == 0), f in cat)
            for f in range(F) if not infos[f]["is_trivial"]]


def _check_against_reference(res, X, g, h, rank_of_row, R, top_k, num_leaves, cat=()):
    """every rank holds the same model; its tree equals tree_ref.grow_tree's voting tree on the same (g, h)"""
    from mmlspark_b200.modeltext import parse_model
    bins = np.concatenate([r["bins"] for r in res])
    T = tree_ref.grow_tree(bins, g, h, _features(res, X.shape[1], cat), ref.Params(min_data_in_leaf=20), num_leaves,
                           voting=(rank_of_row, R, top_k))
    for r in range(R):
        assert res[r]["model"] == res[0]["model"]
    tc.compare_tree(parse_model(res[0]["model"])["trees"][0], T, res[0]["ub"], res[0]["b2c"])
    return T


def _check_boosting(res, X, rank_rows, R, top_k, K, lr, num_leaves, bag=None):
    """every tree of a boosting run equals tree_ref.grow_tree's voting tree on the gradients the engine trained it on (read back before each
    iteration, quantised as K3 does) over the rows it was grown on (bag: (fraction, seed) of plain bagging)"""
    from mmlspark_b200.modeltext import parse_model
    trees = parse_model(res[0]["model"])["trees"]
    iters = len(res[0]["grads"])
    assert len(trees) == iters * K
    bins = np.concatenate([r["bins"] for r in res])
    rank_of_row = np.repeat(np.arange(R), rank_rows)
    feats = _features(res, X.shape[1])
    const_h = res[0]["info"]["constant_hessian"]
    bags = None
    if bag is not None:
        per_rank = [tc.bags(n_r, iters, bag[0], bag[1]) for n_r in rank_rows]
        bags = [np.concatenate([per_rank[r][it] for r in range(R)]) for it in range(iters)]
    for it in range(iters):
        for k in range(K):
            g = np.concatenate([r["grads"][it][0].reshape(K, -1)[k] for r in res])
            h = np.concatenate([r["grads"][it][1].reshape(K, -1)[k] for r in res])
            gq = tc.quantized(g)
            hq = np.ones(len(h)) if const_h else tc.quantized(h)
            rows = np.arange(len(g)) if bags is None else np.nonzero(bags[it])[0]
            T = tree_ref.grow_tree(bins[rows], gq[rows], hq[rows], feats, ref.Params(min_data_in_leaf=20), num_leaves,
                                   voting=(rank_of_row[rows], R, top_k))
            tc.compare_tree(trees[it * K + k], T, res[0]["ub"], res[0]["b2c"], lr)


def _custom_params(R, top_k, learner="voting", extra=""):
    return ("objective=regression tree_learner=%s top_k=%d num_machines=%d num_leaves=8 learning_rate=1 boost_from_average=false "
            "num_iterations=1 verbosity=-1 min_data_in_leaf=20 min_sum_hessian_in_leaf=0.001 %s %s" % (learner, top_k, R, DS, extra))


# ------------------------------------------------------------------------------------------------ the learner against the restatement
@pytest.mark.parametrize("R,top_k", [(2, 1), (2, 2), (2, 5), (3, 3), (4, 2), (4, 5)])
def test_voting_tree_matches_reference(built, R, top_k):
    rank_rows = [5000 + 37 * r for r in range(R)]          # unequal shards
    X, y, rank_of_row = _skewed(10 + R * 7 + top_k, rank_rows)
    g, h = _grid_gradients(y, 3)
    res = _train(X, y, rank_rows, _custom_params(R, top_k), 1, 27000 + 20 * R + top_k, grads=(g, h))
    T = _check_against_reference(res, X, g, h, rank_of_row, R, top_k, 8)
    assert all(len(v[0]) <= top_k for v in T["voted"])
    # the data-parallel learner on the same gradients splits the root on the shared feature, which no rank votes for at top_k <= 5
    dp = _train(X, y, rank_rows, _custom_params(R, top_k, "data_parallel"), 1, 27300 + 20 * R + top_k, grads=(g, h))
    assert tc.trees(dp[0]["model"]) != tc.trees(res[0]["model"])
    assert R * 5 not in T["voted"][0][0]


def test_voting_categorical_matches_reference(built):
    R, top_k = 2, 3
    rank_rows = [6000, 5400]
    X, y, rank_of_row = _skewed(77, rank_rows)
    rng = np.random.default_rng(78)
    X[:, 27] = rng.integers(0, 12, len(X))
    y = y + np.where(X[:, 27] % 3 == 0, 1.5, 0.0)
    g, h = _grid_gradients(y, 4)
    res = _train(X, y, rank_rows, _custom_params(R, top_k, extra="categorical_feature=27"), 1, 27500, grads=(g, h),
                 ds_params=DS + " categorical_feature=27")
    _check_against_reference(res, X, g, h, rank_of_row, R, top_k, 8, cat=(27,))


# ------------------------------------------------------------------------------------------------ boosting runs
def test_one_rank_equals_data_parallel(built):
    """with one rank both settings run the serial learner: the same trees byte for byte"""
    X, y, _ = _skewed(5, [20000], per_rank=5)
    a = _train(X, y, [20000], _params("regression", 1, "voting", 2), 10, 27600)
    b = _train(X, y, [20000], _params("regression", 1, "data_parallel", 2), 10, 27610)
    assert tc.trees(a[0]["model"]) == tc.trees(b[0]["model"])
    assert a[0]["comm"] == dict(hist_bytes=0, record_bytes=0, splits=10 * 14)


def _slot_bytes(res):
    """bytes of one histogram slot: every uint8 tile of 32 storage columns x 256 (g, h) int64 pairs (no wide features here)"""
    num_columns = res[0]["bundles"][0]
    return max(1, (num_columns + 31) // 32) * 32 * 256 * 16


@pytest.mark.parametrize("objective", ["regression", "binary"])
@pytest.mark.parametrize("R", [2, 4])
@pytest.mark.parametrize("top_k", [2, 5])
def test_voting_boosting(built, objective, R, top_k):
    """every tree of a boosting run equals the restatement on the engine's gradients; every rank holds the same model, it differs from the
    data-parallel model on shard-skewed data, and the byte counters match the buffers"""
    n = 6000 * R
    rank_rows = [n // R + (11 if r == 0 else 0) - (11 if r == R - 1 else 0) for r in range(R)]      # unequal shards, NaN in feature 29
    X, y, _ = _skewed(200 + R + top_k, rank_rows)
    if objective == "binary":
        y = (y > np.median(y)).astype(np.float64)
    port = 28000 + 100 * R + 10 * top_k + (0 if objective == "binary" else 50)
    iters, lr = 4, 0.3
    extra = "boost_from_average=false learning_rate=%g" % lr
    vt = _train(X, y, rank_rows, _params(objective, R, "voting", top_k, extra), iters, port)
    dp = _train(X, y, rank_rows, _params(objective, R, "data_parallel", top_k, extra), iters, port + 5)
    for r in range(R):
        assert vt[r]["model"] == vt[0]["model"]
    _check_boosting(vt, X, rank_rows, R, top_k, 1, lr, 15)
    assert tc.trees(vt[0]["model"]) != tc.trees(dp[0]["model"])
    splits = iters * 14
    assert vt[0]["comm"]["splits"] == splits and dp[0]["comm"]["splits"] == splits
    col = 256 * 16
    assert dp[0]["comm"]["hist_bytes"] == splits * _slot_bytes(dp) and dp[0]["comm"]["record_bytes"] == 0
    k = min(top_k, 30)
    assert vt[0]["comm"]["hist_bytes"] == splits * (2 * k * col + 2 * 16)
    assert vt[0]["comm"]["hist_bytes"] < dp[0]["comm"]["hist_bytes"]
    assert vt[0]["comm"]["record_bytes"] == splits * R * 2 * top_k * 24


@pytest.mark.parametrize("mode", ["multiclass", "bagging"])
def test_voting_boosting_modes_match_reference(built, mode):
    """K trees per iteration (each on its class's gradients) and bagged roots (the restated per-block LCG draw): every tree equals the
    restatement"""
    R, n = 2, 12000
    rank_rows = [n // 2 + 101, n - n // 2 - 101]
    X, y, _ = _skewed(300 + len(mode), rank_rows)
    extra, objective, K, bag = "boost_from_average=false learning_rate=0.3", "regression", 1, None
    if mode == "multiclass":
        objective, K = "multiclass", 3
        extra += " num_class=3"
        y = np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(np.float64)
    else:
        extra += " bagging_fraction=0.5 bagging_freq=1 bagging_seed=7"
        bag = (0.5, 7)
    res = _train(X, y, rank_rows, _params(objective, R, "voting", 3, extra), 4, 28900 + 10 * len(mode))
    assert res[1]["model"] == res[0]["model"]
    _check_boosting(res, X, rank_rows, R, 3, K, 0.3, 15, bag=bag)


def test_voting_goss(built):
    """GOSS-sampled roots (the sample and the amplified gradients stay inside the engine, so no tree-by-tree reference): the ranks agree,
    and the model predicts its own training scores"""
    R, n = 2, 30000
    rank_rows = [n // 2 + 101, n - n // 2 - 101]
    X, y, _ = _skewed(304, rank_rows)
    res = _train(X, y, rank_rows, _params("regression", R, "voting", 3, "boosting_type=goss"), 5, 28990)
    assert res[1]["model"] == res[0]["model"]
    from mmlspark_b200 import capi
    pred = capi.Booster(model_str=res[0]["model"]).predict_device(X, predict_type=1).reshape(-1)
    np.testing.assert_allclose(np.concatenate([r["scores"] for r in res]), pred, rtol=1e-6, atol=1e-6)


def test_voting_bundles_equal_unbundled(built):
    """sparse one-hot data: the voted bundle members are unbundled from their packed columns with the reduced leaf totals, so the model
    equals the one trained with enable_bundle=false"""
    import test_gpu_bundling as B
    X, z = B._one_hot_data(21, 12000)
    y = B._labels(z, "binary")
    rank_rows = [6000, 6000]
    ds = "max_bin=255 min_data_in_leaf=5 is_pre_partition=True num_threads=0"
    p = "objective=binary num_leaves=15 tree_learner=voting top_k=4 num_machines=2 verbosity=-1 metric= " + ds
    a = _train(X, y, rank_rows, p, 8, 29100, ds_params=ds)
    b = _train(X, y, rank_rows, p + " enable_bundle=false", 8, 29110, ds_params=ds + " enable_bundle=false")
    assert tc.trees(a[0]["model"]) == tc.trees(b[0]["model"])
    for r in range(2):
        assert np.array_equal(a[r]["scores"], b[r]["scores"])


def test_voting_nccl_two_gpus(built):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    rank_rows = [5000, 5037]
    X, y, rank_of_row = _skewed(401, rank_rows)
    g, h = _grid_gradients(y, 5)
    res = _train(X, y, rank_rows, _custom_params(2, 2), 1, 29200, device_of=lambda r: r, grads=(g, h))
    _check_against_reference(res, X, g, h, rank_of_row, 2, 2, 8)


# ------------------------------------------------------------------------------------------------ fail loudly at LGBM_BoosterCreate
@pytest.mark.parametrize("case", ["top_k", "wide"])
def test_voting_rejects_at_create(built, case):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(9)
    n = 4000
    X = rng.standard_normal((n, 4))
    ds_params = DS
    extra = ""
    if case == "wide":
        X[:, 2] = rng.integers(0, 600, n)
        ds_params = DS + " categorical_feature=2"
        extra = "categorical_feature=2"
    top_k = 0 if case == "top_k" else 3
    params = _params("regression", 2, "voting", top_k, extra)

    def body(r):
        ds = capi.Dataset.from_mat(X[r * n // 2:(r + 1) * n // 2], ds_params).set_field("label", np.ones(n // 2, np.float32))
        try:
            with pytest.raises(Exception) as e:
                capi.Booster(ds, params)
            return str(e.value)
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29300 + (0 if case == "top_k" else 10), body)
    assert not errs, errs
    want = "top_k > 0" if case == "top_k" else "more than 256 bins"
    assert all(want in m for m in res), res


# ------------------------------------------------------------------------------------------------ the estimator path
def test_estimator_voting_parallel(built):
    """LightGBMRegressor(parallelism="voting_parallel", topK=3, numTasks=2) trains the two-rank voting model of its two partitions: its trees
    equal the low-level two-rank run with the estimator's parameters on the same partitions, in one of the two rank orders (the driver
    numbers the ranks in the order the tasks reach it), and differ from parallelism="data_parallel"'s"""
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    rank_rows = [10000, 10000]
    X, y, _ = _skewed(500, rank_rows)
    df = Frame({"features": X, "label": y})
    est = LightGBMRegressor(parallelism="voting_parallel", topK=3, numTasks=2, numIterations=5, defaultListenPort=29400)
    mv = est.fit(df)
    md = LightGBMRegressor(parallelism="data_parallel", topK=3, numTasks=2, numIterations=5, defaultListenPort=29420).fit(df)
    assert tc.trees(mv.getNativeModel()) != tc.trees(md.getNativeModel())
    params = est.getTrainParams(2, df).to_string()
    assert "tree_learner=voting_parallel" in params and "top_k=3" in params
    ds = dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), [])
    swap = np.r_[10000:20000, 0:10000]
    low = [_train(X, y, rank_rows, params, 5, 29440, ds_params=ds), _train(X[swap], y[swap], rank_rows, params, 5, 29450, ds_params=ds)]
    assert tc.trees(mv.getNativeModel()) in [tc.trees(r[0]["model"]) for r in low]
