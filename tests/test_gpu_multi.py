"""Data-parallel parity: R rank-threads in ONE process, thread i <-> GPU i <-> NCCL rank i — the reference's
local-mode model (all Spark tasks are threads of one JVM, SURVEY.md fact 8; the reference's suites use
numPartitions = 2, VerifyLightGBMClassifier.scala:126).  The R-rank run must produce the tree sequence of the
oracle's R-rank emulation (distributed bin finding, hessian-reconstructed global counts, mean-of-means init)."""
import os
import subprocess
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"


def _ngpu():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return len([l for l in out.splitlines() if l.startswith("GPU ")])
    except Exception:
        return 0


def _params(objective, machines, extra=""):
    return ("metric= boost_from_average=true is_pre_partition=True boosting_type=gbdt tree_learner=data_parallel top_k=20 num_iterations=100 "
            "learning_rate=0.1 num_leaves=31 max_bin=255 bagging_fraction=1.0 bagging_freq=0 feature_fraction=1.0 max_depth=-1 "
            "min_sum_hessian_in_leaf=0.001 num_machines=%d verbosity=-1 lambda_l1=0.0 lambda_l2=0.0 min_gain_to_split=0.0 max_delta_step=0.0 "
            "min_data_in_leaf=20 objective=%s num_threads=0 %s" % (machines, objective, extra))


def run_ranks(X, y, rank_rows, params, iters, base_port, weight=None, push_chunk=0):
    """Replays TrainUtils/LightGBMBase.trainLightGBM per rank-thread: NetworkInit -> DatasetCreateFromMat ->
    SetField -> BoosterCreate -> UpdateOneIter* -> (rank 0) SaveModelToString -> free -> NetworkFree."""
    from mmlspark_b200 import capi
    R = len(rank_rows)
    machines = ",".join("127.0.0.1:%d" % (base_port + r) for r in range(R))
    offs = np.concatenate([[0], np.cumsum(rank_rows)])
    out = [None] * R
    errs = []

    def task(r):
        try:
            capi.set_device(r)
            capi.network_init(machines, base_port + r, 120, R)
            sl = slice(int(offs[r]), int(offs[r + 1]))
            if push_chunk:       # the benchmark's ingestion path: bins from the rank's own column sample, rows pushed in chunks (f32)
                Xr = np.ascontiguousarray(X[sl], dtype=np.float32)
                rows = capi.sample_indices(len(Xr), 200000, 1)
                ds = capi.Dataset.from_sampled_columns(Xr[rows].astype(np.float64), len(Xr), DS_PARAMS)
                for off in range(0, len(Xr), push_chunk):
                    ds.push_rows(Xr[off:off + push_chunk], off)
            else:
                ds = capi.Dataset.from_mat(X[sl], DS_PARAMS)
            ds.set_field("label", y[sl])
            if weight is not None:
                ds.set_field("weight", weight[sl])
            b = capi.Booster(ds, params)
            evals = []
            for _ in range(iters):
                if b.update_one_iter():
                    break
                evals.append(b.get_eval(0))
            out[r] = dict(model=b.save_model_to_string(), bins=ds.get_bins(), evals=np.array(evals), scores=b.get_scores())
            b.free(); ds.free()
            capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, repr(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(R)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(180)
    assert not errs, errs
    return out


@pytest.mark.parametrize("objective,R", [("regression", 2), ("binary", 2), ("binary", 4), ("regression", 4)])
def test_data_parallel_matches_oracle_emulation(built, objective, R):
    if _ngpu() < R:
        pytest.skip("needs %d GPUs" % R)
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    rng = np.random.default_rng(100 + R)
    n, F = 80000, 30
    X = rng.standard_normal((n, F))
    X[:, 4] = np.where(rng.random(n) < 0.2, np.nan, X[:, 4])
    s = 1.5 * X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.3 * rng.standard_normal(n)
    y = (s > 0).astype(np.float32) if objective == "binary" else s.astype(np.float32)
    rank_rows = [n // R + (7 if r == 0 else 0) - (7 if r == R - 1 else 0) for r in range(R)]     # unequal shards
    params = _params(objective, R, "is_unbalance=false" if objective == "binary" else "")
    res = run_ranks(X, y, rank_rows, params, 15, 23000 + 40 * R + (0 if objective == "binary" else 20))
    ods = O.OracleDataset(X, DS_PARAMS, rank_rows=rank_rows).set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(15)
    # every rank binned its shard with the all-gathered mappers
    obins = ods.bins()
    offs = np.concatenate([[0], np.cumsum(rank_rows)])
    for r in range(R):
        assert np.array_equal(res[r]["bins"], obins[offs[r]:offs[r + 1]]), "rank %d bins differ" % r
    # all ranks hold the same model; it equals the oracle's R-rank emulation
    for r in range(1, R):
        assert res[r]["model"] == res[0]["model"]
    compare_models(parse_model(res[0]["model"]), parse_model(ob.model_string()))
    # averaged metrics are global: every rank reports the same value
    for r in range(1, R):
        np.testing.assert_allclose(res[r]["evals"], res[0]["evals"], rtol=1e-12)
    got_scores = np.concatenate([res[r]["scores"] for r in range(R)])
    np.testing.assert_allclose(got_scores, ob.scores(), rtol=1e-6, atol=1e-6)


def test_rank_with_single_class_does_not_hang(built):
    """'a partition with a single binary class' (VerifyLightGBMClassifier.scala:630-643): need_train is decided on
    GLOBAL class counts (R14)."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.modeltext import parse_model
    rng = np.random.default_rng(5)
    n, F = 20000, 10
    X = rng.standard_normal((n, F))
    y = (X[:, 0] > 0).astype(np.float32)
    order = np.argsort(-y, kind="stable")          # rank 0 only sees positives
    X, y = X[order], y[order]
    n0 = int(y.sum()) - 100
    res = run_ranks(X, y, [n0, n - n0], _params("binary", 2, "is_unbalance=false"), 5, 23700)
    m = parse_model(res[0]["model"])
    assert len(m["trees"]) == 5 and m["trees"][0]["num_leaves"] > 1


@pytest.mark.parametrize("mode", ["bagging", "goss"])
def test_data_parallel_row_sampling(built, mode):
    """Every rank bags its own shard with its own per-block LCGs (seeded bagging_seed + local block); root counts and sums are
    all-reduced over the in-bag rows only."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    rng = np.random.default_rng(321)
    n, F = 50000, 16
    X = rng.standard_normal((n, F))
    s = 1.5 * X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.3 * rng.standard_normal(n)
    y = (s > 0).astype(np.float32)
    rank_rows = [n // 2 + 333, n - n // 2 - 333]
    params = _params("binary", 2, "is_unbalance=false")
    if mode == "bagging":
        params = params.replace("bagging_fraction=1.0 bagging_freq=0", "bagging_fraction=0.5 bagging_freq=2")
    else:
        params = params.replace("boosting_type=gbdt", "boosting_type=goss").replace("learning_rate=0.1", "learning_rate=0.3")
    res = run_ranks(X, y, rank_rows, params, 8, 23900 + (0 if mode == "bagging" else 11))
    ods = O.OracleDataset(X, DS_PARAMS, rank_rows=rank_rows).set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(8)
    assert res[1]["model"] == res[0]["model"]
    compare_models(parse_model(res[0]["model"]), parse_model(ob.model_string()))
    got_scores = np.concatenate([res[r]["scores"] for r in range(2)])
    np.testing.assert_allclose(got_scores, ob.scores(), rtol=1e-6, atol=1e-6)


def test_data_parallel_push_rows_ingestion(built):
    """The path bench.py builds its shards with (LGBM_DatasetCreateFromSampledColumn + LGBM_DatasetPushRows, f32 chunks, ragged tail) on
    2 ranks: distributed bin finding from every rank's own sample, bins and trees equal to the oracle's 2-rank emulation."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    rng = np.random.default_rng(77)
    n, F = 120000, 40
    X = rng.standard_normal((n, F)).astype(np.float32).astype(np.float64)      # f32-representable: both paths see the same values
    X[:, 3] = np.where(rng.random(n) < 0.6, 0.0, X[:, 3])
    s = 1.5 * X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.3 * rng.standard_normal(n)
    y = (s > 0).astype(np.float32)
    rank_rows = [n // 2 + 1111, n - n // 2 - 1111]
    params = _params("binary", 2, "is_unbalance=false")
    res = run_ranks(X, y, rank_rows, params, 6, 24100, push_chunk=17000)
    ods = O.OracleDataset(X, DS_PARAMS, rank_rows=rank_rows).set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(6)
    obins = ods.bins()
    offs = np.concatenate([[0], np.cumsum(rank_rows)])
    for r in range(2):
        assert np.array_equal(res[r]["bins"], obins[offs[r]:offs[r + 1]]), "rank %d pushed bins differ" % r
    assert res[1]["model"] == res[0]["model"]
    compare_models(parse_model(res[0]["model"]), parse_model(ob.model_string()))
