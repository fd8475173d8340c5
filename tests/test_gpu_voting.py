"""Voting-parallel training (tree_learner=voting / parallelism="voting_parallel", LightGBM's VotingParallelTreeLearner): every rank scans its
local histograms, the ranks vote on top_k features per leaf, and only the voted features' histograms are all-reduced and scanned globally.

All ranks are rank-threads of this process on device 0 (the same-device communicator), so every test runs on one GPU; the NCCL variant
runs one rank per GPU and is skipped with fewer than two.  Trees are pinned against the NumPy restatement in voting_ref.py on custom
gradients and hessians on a 2^-10 grid (as test_gpu_split_scan.py does for the serial scan): K4's fixed-point quantisation is exact there,
so the local and the reduced int64 histograms equal NumPy's fp64 ones bit for bit and only the scans, the vote and the pick are under test."""
import subprocess
import threading

import numpy as np
import pytest

import split_scan_ref as ref
import voting_ref as V

pytestmark = pytest.mark.gpu

GRID = 1.0 / 1024
DS = "max_bin=63 min_data_in_bin=3 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"


def _ngpu():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return len([l for l in out.splitlines() if l.startswith("GPU ")])
    except Exception:
        return 0


def _on_ranks(R, base_port, body, device_of=lambda r: 0):
    """body(r) on R rank-threads, rank r on device_of(r), between network_init and network_free; returns (results, errors)"""
    from mmlspark_b200 import capi
    machines = ",".join("127.0.0.1:%d" % (base_port + r) for r in range(R))
    out, errs = [None] * R, []

    def task(r):
        try:
            capi.set_device(device_of(r))
            if R == 1:
                out[r] = body(r)
                return
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

    res, errs = _on_ranks(len(rank_rows), port, body, device_of)
    assert not errs, errs
    return res


def _categorical(ds_params):
    return [int(c) for tok in ds_params.split() if tok.startswith("categorical_feature=") for c in tok.split("=")[1].split(",")]


def _trees(model):
    return model.split("\nparameters:")[0]


def _grid_gradients(y, seed):
    rng = np.random.default_rng(seed)
    g = np.round(-np.clip(y, -30, 30) / GRID) * GRID
    h = rng.integers(512, 1537, len(y)) * GRID
    return g, h


def _features(res, F, cat=()):
    infos = res[0]["infos"]
    return [ref.Feature(f, infos[f]["num_bin"], infos[f]["missing_type"], int(infos[f]["most_freq_bin"] == 0), f in cat)
            for f in range(F) if not infos[f]["is_trivial"]]


def _compare_tree(t, T, side, lr=1.0):
    """the engine's tree t (parse_model) against voting_ref's T: structure, thresholds, default directions, category sets and counts
    exact, split_gain equal to the reference's float32 gain as printed (%g), leaf values within 1e-12 relative"""
    assert t["num_leaves"] == T["num_leaves"]
    nl = T["num_leaves"]
    if nl > 1:
        assert t["split_feature"].tolist() == T["split_feature"]
        assert t["left_child"].tolist() == T["left_child"] and t["right_child"].tolist() == T["right_child"]
        assert t["leaf_count"].tolist() == T["leaf_count"] and t["internal_count"].tolist() == T["internal_count"]
        for i in range(nl - 1):
            f, dt = T["split_feature"][i], int(t["decision_type"][i])
            assert bool(dt & 1) == T["is_cat"][i], "node %d: categorical flag" % i
            if T["is_cat"][i]:
                k = int(t["threshold"][i])
                words = t["cat_threshold"][t["cat_boundaries"][k]:t["cat_boundaries"][k + 1]]
                cats = {32 * w + j for w, word in enumerate(words) for j in range(32) if (int(word) >> j) & 1}
                got = {b for b, c in enumerate(side["b2c"][f]) if b > 0 and c in cats}
                assert got == set(T["cat_bins"][i]), "node %d: category bins" % i
            else:
                hit = np.nonzero(side["ub"][f] == t["threshold"][i])[0]
                assert len(hit) == 1 and hit[0] == T["threshold_bin"][i], "node %d: threshold %r" % (i, t["threshold"][i])
                assert bool(dt & 2) == T["default_left"][i], "node %d: default_left" % i
            assert t["split_gain"][i] == float("%g" % T["split_gain"][i]), "node %d: split_gain %r vs %g" % (i, t["split_gain"][i], T["split_gain"][i])
    np.testing.assert_allclose(t["leaf_value"], np.asarray(T["leaf_value"]) * lr, rtol=1e-12, atol=1e-300)


def _check_against_reference(res, X, g, h, rank_of_row, R, top_k, num_leaves, cat=()):
    """every rank holds the same model; its tree equals voting_ref.grow_voting_tree on the same (g, h)"""
    from mmlspark_b200.modeltext import parse_model
    bins = np.concatenate([r["bins"] for r in res])
    T = V.grow_voting_tree(bins, g, h, _features(res, X.shape[1], cat), ref.Params(min_data_in_leaf=20), num_leaves, rank_of_row, R, top_k)
    for r in range(R):
        assert res[r]["model"] == res[0]["model"]
    _compare_tree(parse_model(res[0]["model"])["trees"][0], T, res[0])
    return T


def _quantized(v):
    """K3's fixed-point grid: q = rint(v * 2^e), e = 34 - ilogb(max |v|) over every rank's rows; the histograms are exact sums of q, so
    NumPy's fp64 sums of q * 2^-e equal the engine's int64 ones"""
    m = np.float32(np.max(np.abs(v)))
    e = 34 - (int(np.frexp(m)[1]) - 1) if m > 0 and np.isfinite(m) else 0
    return np.rint(v.astype(np.float64) * 2.0 ** e) * 2.0 ** -e


def _bags(n, iters, fraction, seed):
    """GBDT::Bagging with bagging_freq = 1 on one rank: per 1024-row block an LCG seeded seed + block, row j of a block takes the next
    draw ((x >> 16) & 0x7fff) / 32768 < fraction; the states carry over to the next iteration's draw"""
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


def _check_boosting(res, X, rank_rows, R, top_k, K, lr, num_leaves, bag=None):
    """every tree of a boosting run equals voting_ref.grow_voting_tree on the gradients the engine trained it on (read back before each
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
        per_rank = [_bags(n_r, iters, bag[0], bag[1]) for n_r in rank_rows]
        bags = [np.concatenate([per_rank[r][it] for r in range(R)]) for it in range(iters)]
    for it in range(iters):
        for k in range(K):
            g = np.concatenate([r["grads"][it][0].reshape(K, -1)[k] for r in res])
            h = np.concatenate([r["grads"][it][1].reshape(K, -1)[k] for r in res])
            gq = _quantized(g)
            hq = np.ones(len(h)) if const_h else _quantized(h)
            rows = np.arange(len(g)) if bags is None else np.nonzero(bags[it])[0]
            T = V.grow_voting_tree(bins[rows], gq[rows], hq[rows], feats, ref.Params(min_data_in_leaf=20), num_leaves, rank_of_row[rows], R, top_k)
            _compare_tree(trees[it * K + k], T, res[0], lr)


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
    assert _trees(dp[0]["model"]) != _trees(res[0]["model"])
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
    assert _trees(a[0]["model"]) == _trees(b[0]["model"])
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
    assert _trees(vt[0]["model"]) != _trees(dp[0]["model"])
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
    assert _trees(a[0]["model"]) == _trees(b[0]["model"])
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

    res, errs = _on_ranks(2, 29300 + (0 if case == "top_k" else 10), body)
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
    assert _trees(mv.getNativeModel()) != _trees(md.getNativeModel())
    params = est.getTrainParams(2, df).to_string()
    assert "tree_learner=voting_parallel" in params and "top_k=3" in params
    ds = dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), [])
    swap = np.r_[10000:20000, 0:10000]
    low = [_train(X, y, rank_rows, params, 5, 29440, ds_params=ds), _train(X[swap], y[swap], rank_rows, params, 5, 29450, ds_params=ds)]
    assert _trees(mv.getNativeModel()) in [_trees(r[0]["model"]) for r in low]
