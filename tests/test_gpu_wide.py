"""Categorical features that need more than 256 bins (BASELINE.json configs[4]: 64 columns of cardinality 10^3..10^5).  LightGBM does not
cap a categorical feature at max_bin — BinMapper::FindBin keeps categories until 99 % of the sampled mass is covered — so such a column
has hundreds to thousands of bins: uint16 columns, k4_hist_wide, k_scan_wide, bin-list splits.  Reference call sites: categorical slot
discovery LightGBMBase.scala:168-199, `categorical_feature=` in the dataset params LightGBMBase.scala:265-272."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0 categorical_feature=1,2,5"


def _params(objective, extra="", machines=1):
    return ("metric= boost_from_average=true is_pre_partition=True boosting_type=gbdt tree_learner=data_parallel num_iterations=100 "
            "learning_rate=0.1 num_leaves=31 max_bin=255 bagging_fraction=1.0 bagging_freq=0 feature_fraction=1.0 max_depth=-1 "
            "min_sum_hessian_in_leaf=0.001 num_machines=%d verbosity=-1 lambda_l1=0.0 lambda_l2=0.0 min_gain_to_split=0.0 max_delta_step=0.0 "
            "min_data_in_leaf=20 objective=%s num_threads=0 %s" % (machines, objective, extra))


def _data(seed, n):
    rng = np.random.default_rng(seed)
    c1 = np.floor(1500.0 ** rng.random(n)) - 1            # ~ 700-900 bins
    c2 = np.floor(30000.0 ** rng.random(n)) - 1           # thousands of bins, long tail folded into bin 0
    c5 = rng.integers(0, 40, n).astype(np.float64)        # an ordinary (narrow) categorical column
    c2[rng.random(n) < 0.01] = np.nan
    X = np.stack([rng.standard_normal(n), c1, c2, rng.standard_normal(n), np.where(rng.random(n) < 0.7, 0.0, rng.random(n)), c5,
                  rng.standard_normal(n)], axis=1)
    eff = rng.standard_normal(40000)
    s = X[:, 0] + 0.8 * eff[np.nan_to_num(c1).astype(int)] + 0.6 * eff[np.nan_to_num(c2).astype(int) + 2000] + 0.3 * eff[c5.astype(int) + 500] + 0.4 * rng.standard_normal(n)
    return X, s


def test_wide_bins_match_oracle_on_every_ingestion_path(built):
    from mmlspark_b200 import capi
    from oracle import oracle as O
    n = 210_000
    X, _ = _data(1, n)
    ods = O.OracleDataset(X, DS)
    want = ods.bins16()
    assert want[:, 1].max() > 255 and want[:, 2].max() > 1000
    ds = capi.Dataset.from_mat(X, DS)
    for f in (1, 2, 5):
        assert ds.feature_info(f) == ods.feature_info(f)
        assert np.array_equal(ds.bin_to_cat(f), ods.bin_to_cat(f))
    assert np.array_equal(ds.get_bins16(), want)
    with pytest.raises(capi.LightGBMError):
        ds.get_bins()                                       # the uint8 export refuses a wide dataset
    rows = capi.sample_indices(n, 200000, 1)
    dp = capi.Dataset.from_sampled_columns(X[rows], n, DS)
    for off in range(0, n, 64_000):
        dp.push_rows(X[off:off + 64_000], off)
    assert np.array_equal(dp.get_bins16(), want)
    pick = np.array([0, 5, n // 2, n - 1], dtype=np.int32)
    assert np.array_equal(dp.get_bins_rows(pick), want[pick])
    # CSR: zeros are implicit (category 0 / value 0), NaNs explicit
    stored = (X != 0) | np.isnan(X)
    indptr = np.concatenate([[0], np.cumsum(stored.sum(axis=1))]).astype(np.int32)
    dc = capi.Dataset.from_csr(indptr, np.nonzero(stored)[1].astype(np.int32), X[stored], X.shape[1], DS)
    assert np.array_equal(dc.get_bins16(), want)
    # validation data binned with the training mappers (unseen categories -> bin 0)
    Xv, _ = _data(2, 20_000)
    dv = capi.Dataset.from_mat(Xv, DS, reference=ds)
    b2c = ods.bin_to_cat(2)
    lut = {int(c): b for b, c in enumerate(b2c) if c >= 0}
    got = dv.get_bins16()[:, 2]
    wantv = np.array([0 if np.isnan(v) or v < 0 else lut.get(int(v), 0) for v in Xv[:, 2]])
    assert np.array_equal(got, wantv)


@pytest.mark.parametrize("objective", ["binary", "regression", "multiclass"])
def test_wide_categorical_training_matches_oracle(built, objective):
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    n = 120_000
    X, s = _data(3, n)
    Xv, sv = _data(4, 15_000)
    if objective == "binary":
        y, yv, extra = (s > 0).astype(np.float32), (sv > 0).astype(np.float32), "is_unbalance=false"
    elif objective == "regression":
        y, yv, extra = s.astype(np.float32), sv.astype(np.float32), ""
    else:
        cut = np.quantile(s, [0.2, 0.4, 0.6, 0.8])
        y, yv, extra = np.digitize(s, cut).astype(np.float32), np.digitize(sv, cut).astype(np.float32), "num_class=5"
    params = _params(objective, extra)
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y)
    dv = capi.Dataset.from_mat(Xv, DS, reference=ds).set_field("label", yv)
    ods = O.OracleDataset(X, DS).set_field("label", y)
    b = capi.Booster(ds, params)
    b.add_valid(dv)
    ob = O.OracleBooster(ods, params)
    iters = 4 if objective == "multiclass" else 8
    for _ in range(iters):
        assert b.update_one_iter() == ob.update()
    m, om = parse_model(b.save_model_to_string()), parse_model(ob.model_string())
    compare_models(m, om)
    wide_nodes = sum(int(np.isin(t["split_feature"][t["decision_type"] % 2 == 1], [1, 2]).sum()) for t in m["trees"] if t["num_leaves"] > 1)
    assert wide_nodes > 0, "the test data must actually split on the wide categorical features"
    np.testing.assert_allclose(b.get_scores(0), ob.scores(), rtol=1e-9, atol=1e-9)
    # validation scores are produced by walking the device tree on the validation BINS (bin-list decisions of the wide features)
    K = 5 if objective == "multiclass" else 1
    np.testing.assert_allclose(b.get_scores(1).reshape(K, -1).T, ob.predict_raw(Xv), rtol=1e-9, atol=1e-9)
    # the model text carries category VALUES: the raw-value predictors (host single row + GPU batch) agree with the oracle
    np.testing.assert_allclose(b.predict_device(Xv[:500], predict_type=capi.PREDICT_RAW_SCORE), ob.predict_raw(Xv[:500]), rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(b.predict_for_mat_single(Xv[3], predict_type=capi.PREDICT_RAW_SCORE), ob.predict_raw(Xv[3:4])[0], rtol=1e-9, atol=1e-9)


def test_wide_categorical_with_bagging_and_feature_fraction(built):
    """bagging scores every row by walking the tree on the bins; feature_fraction draws over the used features in real-index order
    although the wide features sit at the end of the inner order"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    n = 90_000
    X, s = _data(5, n)
    y = (s > 0).astype(np.float32)
    params = _params("binary", "is_unbalance=false").replace("bagging_fraction=1.0 bagging_freq=0", "bagging_fraction=0.6 bagging_freq=1").replace(
        "feature_fraction=1.0", "feature_fraction=0.6")
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y)
    ods = O.OracleDataset(X, DS).set_field("label", y)
    b = capi.Booster(ds, params)
    ob = O.OracleBooster(ods, params)
    for _ in range(8):
        assert b.update_one_iter() == ob.update()
    compare_models(parse_model(b.save_model_to_string()), parse_model(ob.model_string()))
    np.testing.assert_allclose(b.get_scores(0), ob.scores(), rtol=1e-9, atol=1e-9)


def test_wide_categorical_two_ranks(built):
    """data-parallel: the mappers of the wide features travel in the all-gather (variable record length), their histograms in the allreduce"""
    import subprocess
    out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
    if len([l for l in out.splitlines() if l.startswith("GPU ")]) < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    n = 100_000
    X, s = _data(6, n)
    y = (s > 0).astype(np.float32)
    rank_rows = [n // 2 + 500, n - n // 2 - 500]
    params = _params("binary", "is_unbalance=false", machines=2)
    machines = "127.0.0.1:24300,127.0.0.1:24301"
    offs = np.concatenate([[0], np.cumsum(rank_rows)])
    res, errs = [None, None], []

    def task(r):
        try:
            capi.set_device(r)
            capi.network_init(machines, 24300 + r, 120, 2)
            sl = slice(int(offs[r]), int(offs[r + 1]))
            ds = capi.Dataset.from_mat(X[sl], DS).set_field("label", y[sl])
            b = capi.Booster(ds, params)
            for _ in range(6):
                b.update_one_iter()
            res[r] = dict(model=b.save_model_to_string(), bins=ds.get_bins16())
            b.free(); ds.free()
            capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, repr(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(240)
    assert not errs, errs
    ods = O.OracleDataset(X, DS, rank_rows=rank_rows).set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(6)
    want = ods.bins16()
    for r in range(2):
        assert np.array_equal(res[r]["bins"], want[offs[r]:offs[r + 1]])
    assert res[0]["model"] == res[1]["model"]
    compare_models(parse_model(res[0]["model"]), parse_model(ob.model_string()))


@pytest.mark.parametrize("max_bin", [1023, 4000])
def test_numerical_max_bin_above_255(built, max_bin):
    """maxBin is a plain estimator parameter (LightGBMParams.scala:136-137): numerical features with more than 256 bins take the wide path
    (uint16 columns, block-wide two-pass scan).  Bins bit-exact, trees identical, incl. the NaN two-way scan and a mostly-zero column."""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    rng = np.random.default_rng(50 + max_bin)
    n = 150_000
    X = rng.standard_normal((n, 8))
    X[:, 1] = np.where(rng.random(n) < 0.3, np.nan, X[:, 1])            # NaN bin + forward pass
    X[:, 2] = np.where(rng.random(n) < 0.8, 0.0, rng.exponential(1.0, n))  # most_freq_bin is the zero bin
    X[:, 3] = rng.integers(0, 200, n)                                    # <= 256 distinct values: stays a tile feature
    X[:, 4] = np.round(X[:, 4], 2)                                       # ~800 distinct values
    s = X[:, 0] + np.where(np.isnan(X[:, 1]), 0.7, np.sin(3 * X[:, 1])) + 0.5 * X[:, 2] + 0.01 * X[:, 3] + X[:, 4] * X[:, 5] + 0.3 * rng.standard_normal(n)
    y = (s > 0.5).astype(np.float32)
    dsp = "max_bin=%d is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0" % max_bin
    ds = capi.Dataset.from_mat(X, dsp).set_field("label", y)
    ods = O.OracleDataset(X, dsp).set_field("label", y)
    infos = [ds.feature_info(f) for f in range(8)]
    assert max(i["num_bin"] for i in infos) > 256 and infos[3]["num_bin"] <= 256
    for f in range(8):
        assert infos[f] == ods.feature_info(f)
        assert ds.upper_bounds(f).tobytes() == ods.upper_bounds(f).tobytes()
    want = ods.bins16()
    assert np.array_equal(ds.get_bins16(), want)
    # the same bins from the streamed (sampled columns + pushed rows) and the CSR ingestion paths, NaN and mostly-zero columns included
    rows = capi.sample_indices(n, 200000, 1)
    dp = capi.Dataset.from_sampled_columns(X[rows], n, dsp)
    for off in range(0, n, 64_000):
        dp.push_rows(X[off:off + 64_000], off)
    assert np.array_equal(dp.get_bins16(), want)
    stored = (X != 0) | np.isnan(X)
    indptr = np.concatenate([[0], np.cumsum(stored.sum(axis=1))]).astype(np.int32)
    dc = capi.Dataset.from_csr(indptr, np.nonzero(stored)[1].astype(np.int32), X[stored], X.shape[1], dsp)
    assert np.array_equal(dc.get_bins16(), want)
    params = ("objective=binary boosting_type=gbdt num_leaves=31 learning_rate=0.1 min_data_in_leaf=20 min_sum_hessian_in_leaf=0.001 verbosity=-1 "
              "max_bin=%d is_unbalance=false" % max_bin)
    b = capi.Booster(ds, params)
    ob = O.OracleBooster(ods, params)
    for _ in range(8):
        assert b.update_one_iter() == ob.update()
    m = parse_model(b.save_model_to_string())
    # feature 1's NaN rows are separated early, so deeper nodes on it sit in NaN-free leaves where the scan direction is a rounding tie
    compare_models(m, parse_model(ob.model_string()), allow_nan_direction_ties=True)
    used = np.concatenate([t["split_feature"] for t in m["trees"] if t["num_leaves"] > 1])
    assert {0, 1, 2} <= set(used.tolist()), "wide numerical features must actually be split on"
    np.testing.assert_allclose(b.get_scores(0), ob.scores(), rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(b.predict_device(X[:300], predict_type=capi.PREDICT_RAW_SCORE)[:, 0], ob.predict_raw(X[:300])[:, 0], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("boosting", ["dart", "goss"])
def test_wide_categorical_with_dart_and_goss(built, boosting):
    """DART re-applies stored device trees (incl. their bin-list categorical nodes) to the binned rows; GOSS re-weights gradients"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    n = 60_000
    X, s = _data(7, n)
    y = (s > 0).astype(np.float32)
    params = _params("binary", "is_unbalance=false").replace("boosting_type=gbdt", "boosting_type=" + boosting)
    if boosting == "dart":
        params += " drop_rate=0.5 skip_drop=0.0"
    else:
        params = params.replace("learning_rate=0.1", "learning_rate=0.5")
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y)
    ods = O.OracleDataset(X, DS).set_field("label", y)
    b = capi.Booster(ds, params)
    ob = O.OracleBooster(ods, params)
    for _ in range(8):
        assert b.update_one_iter() == ob.update()
    compare_models(parse_model(b.save_model_to_string()), parse_model(ob.model_string()))
    np.testing.assert_allclose(b.get_scores(0), ob.scores(), rtol=1e-8, atol=1e-8)


def test_wide_categorical_selection_list_overflow_falls_back(built):
    """k_scan_wide selects the max_cat_threshold smallest / largest ctr keys through a threshold taken from the per-thread minima (maxima)
    and a <= 512-entry candidate list.  Adversarial layout: ~600 bins owned by only 31 of the 256 threads (bin % 256 < 31) carry the small
    keys, so the 32nd smallest per-thread minimum is a large key and the list overflows; the kernel must fall back to the round-based
    selection and still agree with the oracle's stable sort."""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    rng = np.random.default_rng(11)
    ncat, per = 8000, 40
    n = ncat * per
    cat = np.repeat(np.arange(ncat), per).astype(np.float64)
    rng.shuffle(cat)
    X = np.stack([cat, rng.standard_normal(n)], axis=1)
    dsp = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=400000 num_threads=0 categorical_feature=0"
    ds = capi.Dataset.from_mat(X, dsp)
    bins = ds.get_bins16()[:, 0].astype(np.int64)
    assert bins.max() > 7000
    low = ((bins % 256) < 31) & ((bins // 256) < 20) & (bins > 0)
    assert len(np.unique(bins[low])) > 512
    catnoise = rng.standard_normal(int(bins.max()) + 1) * 0.05            # distinct ctr per category, no exact ties among the candidates
    y = (np.where(low, -5.0, 5.0) + catnoise[bins] + 0.01 * rng.standard_normal(n)).astype(np.float32)
    ds.set_field("label", y)
    params = _params("regression", "min_data_per_group=10 cat_smooth=10 min_data_in_leaf=5")
    b = capi.Booster(ds, params)
    for _ in range(3):
        assert not b.update_one_iter()
    ods = O.OracleDataset(X, dsp)
    assert np.array_equal(ods.bins16()[:, 0], bins)
    ods.set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(3)
    ma, mb = parse_model(b.save_model_to_string()), parse_model(ob.model_string())
    compare_models(ma, mb)
    assert any((np.asarray(t["decision_type"]).astype(np.int64) & 1).any() for t in ma["trees"]), "no categorical split was made"
    np.testing.assert_allclose(b.get_scores(), ob.scores(), rtol=1e-9, atol=1e-9)
    b.free(); ds.free()
