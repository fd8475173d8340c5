"""Host-side logic of the reference's estimator layer, tested without a GPU: the TrainParams wire format, the
trainCore loop (early stopping, delegate learning-rate schedule), the driver rendezvous protocol, partitioning,
and the N>1 plumbing of bench.py under gloo with world_size 2."""
import os
import socket
import subprocess
import sys
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------- wire format (TrainParams.scala:47-179)
def test_classifier_param_string_is_byte_exact():
    from mmlspark_b200.lightgbm import LightGBMClassifier
    c = LightGBMClassifier()
    s = c.getTrainParams(2, {"label": np.array([0, 1])}).to_string()
    assert s == ("metric= boost_from_average=true is_pre_partition=True boosting_type=gbdt tree_learner=data_parallel top_k=20 "
                 "num_iterations=100 learning_rate=0.1 num_leaves=31 max_bin=255 bagging_fraction=1.0 pos_bagging_fraction=1.0 "
                 "neg_bagging_fraction=1.0 bagging_freq=0 bagging_seed=3 early_stopping_round=0 feature_fraction=1.0 max_depth=-1 "
                 "min_sum_hessian_in_leaf=0.001 num_machines=2 verbosity=-1 lambda_l1=0.0 lambda_l2=0.0 metric= min_gain_to_split=0.0 "
                 "max_delta_step=0.0 min_data_in_leaf=20 objective=binary  num_threads=0  is_unbalance=false")
    m = LightGBMClassifier(objective="multiclass", categoricalSlotIndexes=[1, 3], maxBinByFeature=[10, 20])
    sm = m.getTrainParams(1, {"label": np.array([0, 1, 2, 2])}).to_string()
    assert sm.endswith("num_class=3") and "categorical_feature=1,3 max_bin_by_feature=10,20 num_threads=0" in sm
    d = LightGBMClassifier(boostingType="dart", learningRate=1e-4).getTrainParams(1, {"label": np.array([0, 1])}).to_string()
    assert "drop_rate=0.1 max_drop=50 skip_drop=0.5 xgboost_dart_mode=false uniform_drop=false" in d and "learning_rate=1.0E-4" in d


def test_regressor_ranker_dataset_param_strings():
    from mmlspark_b200.lightgbm import LightGBMRanker, LightGBMRegressor, dataset_params

    class F:
        def getGradient(self, p, l): return p, p
    r = LightGBMRegressor(alpha=0.5, fobj=F()).getTrainParams(1, {}).to_string()
    assert r.startswith("alpha=0.5 tweedie_variance_power=1.5 boost_from_average=true is_pre_partition=True")
    assert "objective=" not in r                                  # omitted with a custom fobj (TrainParams.scala:173-179)
    k = LightGBMRanker(groupCol="q", labelGain=[0.0, 1.0, 3.0]).getTrainParams(4, {}).to_string()
    assert k.startswith("max_position=20 label_gain=0.0,1.0,3.0 eval_at=1,2,3,4,5 is_pre_partition=True") and "objective=lambdarank" in k
    assert dataset_params(255, 200000, 0) == "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"   # LightGBMBase.scala:265-272
    assert dataset_params(63, 1000, 4, [2, 5]).endswith("num_threads=4 categorical_feature=2,5")


def test_param_accessors_like_pyspark_wrappers():
    from mmlspark_b200.lightgbm import LightGBMClassifier
    c = LightGBMClassifier(learningRate=0.3, numIterations=100, numLeaves=31)       # docs/lightgbm.md:33-36
    assert c.getLearningRate() == 0.3 and c.setNumLeaves(5).getNumLeaves() == 5 and c.getMaxBin() == 255
    with pytest.raises(TypeError):
        LightGBMClassifier(notAParam=1)
    with pytest.raises(AttributeError):
        c.getNotAParam()


# ---------------------------------------------------------------- trainCore (TrainUtils.scala:92-159)
class FakeBooster:
    def __init__(self, valid_scores, names=("auc",), finish_at=None):
        self.valid_scores, self.names, self.finish_at = list(valid_scores), list(names), finish_at
        self.it, self.resets, self.train_evals = 0, [], 0

    def eval_names(self): return self.names
    def update_one_iter(self):
        self.it += 1
        return self.finish_at is not None and self.it > self.finish_at
    def get_eval(self, idx):
        if idx == 0:
            self.train_evals += 1
        return np.array([self.valid_scores[min(self.it - 1, len(self.valid_scores) - 1)]] * len(self.names))
    def reset_parameter(self, s): self.resets.append(s)


def _tp(**kw):
    from mmlspark_b200.lightgbm import LightGBMClassifier
    return LightGBMClassifier(**kw).getTrainParams(1, {"label": np.array([0, 1])})


def test_train_core_early_stopping_maximised_metric():
    from mmlspark_b200.lightgbm import train_core
    b = FakeBooster([0.6, 0.7, 0.8, 0.79, 0.78, 0.77, 0.9], names=("auc",))
    best = train_core(0, 0, _tp(numIterations=50, earlyStoppingRound=2), b, True)
    assert best == 2 and b.it == 5                                   # best at 0-based iter 2; stops when iters - best >= 2
    b = FakeBooster([0.5, 0.4, 0.3, 0.35, 0.36], names=("binary_logloss",))
    assert train_core(0, 0, _tp(numIterations=50, earlyStoppingRound=1), b, True) == 2 and b.it == 4      # minimised metric


def test_train_core_quirk_early_stopping_round_zero():
    """Appendix D: with earlyStoppingRound=0 (default) and a validation set the first non-improving iteration stops."""
    from mmlspark_b200.lightgbm import train_core
    b = FakeBooster([0.5, 0.6, 0.6, 0.9], names=("auc",))
    assert train_core(0, 0, _tp(numIterations=50), b, True) == 1 and b.it == 3
    b = FakeBooster([0.5, 0.6, 0.595, 0.9], names=("auc",))            # improvementTolerance compared on the signed difference
    assert train_core(0, 0, _tp(numIterations=4, improvementTolerance=-0.01), b, True) is None and b.it == 4


def test_train_core_stops_on_is_finished_and_runs_delegate():
    from mmlspark_b200.lightgbm import LightGBMDelegate, train_core
    calls = []

    class D(LightGBMDelegate):
        def getLearningRate(self, batchIndex, partitionId, curIters, trainParams, previousLearningRate):
            return 0.005 if curIters == 0 else previousLearningRate      # VerifyLightGBMClassifier.scala:497-510
        def afterTrainIteration(self, *a): calls.append(a[2])
    b = FakeBooster([0.1], finish_at=3)
    assert train_core(0, 0, _tp(numIterations=10, delegate=D(), isProvideTrainingMetric=True), b, False) is None
    assert b.it == 4 and calls == [0, 1, 2, 3] and b.resets == ["learning_rate=0.005"] and b.train_evals == 3

    class Boom(FakeBooster):
        def update_one_iter(self): raise RuntimeError("native failure")
    b = Boom([0.1])
    assert train_core(0, 0, _tp(numIterations=10), b, False) is None      # exception -> isFinished (TrainUtils.scala:82-88)


# ---------------------------------------------------------------- rendezvous (LightGBMBase.scala:392-430, TrainUtils.scala:193-363)
def test_driver_rendezvous_and_main_worker_election():
    from mmlspark_b200.lightgbm import DriverRendezvous
    from mmlspark_b200.lightgbm import train_utils as tu
    drv = DriverRendezvous(4, 0, 30.0)
    host, port = drv.start()
    out = {}

    def task(pid, empty):
        s, p = tu.find_open_port(23400, pid)
        try:
            out[pid] = (tu.get_network_init_nodes(host, port, p, empty), p)
        finally:
            s.close()
    ts = [threading.Thread(target=task, args=(i, i == 2)) for i in range(4)]      # partition 2 is empty -> "ignore"
    [t.start() for t in ts]; [t.join(30) for t in ts]
    drv.join(30)
    assert out[2][0] == "ignore"
    lists = {out[i][0] for i in (0, 1, 3)}
    assert len(lists) == 1
    nodes = lists.pop().split(",")
    assert len(nodes) == 3 and sorted(int(n.split(":")[1]) for n in nodes) == sorted(out[i][1] for i in (0, 1, 3))
    main_port = tu.get_main_worker_port(",".join(nodes))
    assert sum(out[i][1] == main_port for i in (0, 1, 3)) == 1               # exactly one task returns the booster


def test_find_open_port_skips_busy_ports():
    from mmlspark_b200.lightgbm import train_utils as tu
    a, pa = tu.find_open_port(23500, 0)
    b, pb = tu.find_open_port(23500, 0)
    assert pb > pa >= 23500
    a.close(); b.close()
    with pytest.raises(RuntimeError):
        tu.find_open_port(65000, 10, 100)


def test_ranker_partitions_keep_groups_whole_and_sorted():
    from mmlspark_b200.lightgbm import Frame, LightGBMRanker
    rng = np.random.default_rng(0)
    sizes = rng.integers(1, 30, 200)
    g = np.repeat(np.arange(200), sizes)
    perm = rng.permutation(len(g))
    df = Frame({"features": rng.standard_normal((len(g), 3))[perm], "label": np.zeros(len(g)), "q": g[perm]})
    r = LightGBMRanker(groupCol="q")
    sdf = r._preprocess(df)
    assert (np.diff(sdf["q"]) >= 0).all()
    parts = r._partitions(sdf, 4)
    seen = set()
    total = 0
    for sl in parts:
        q = set(sdf["q"][sl].tolist())
        assert not (q & seen)                                                  # no group straddles two ranks
        seen |= q
        total += sl.stop - sl.start
    assert total == len(g)
    with pytest.raises(ValueError):
        LightGBMRanker(groupCol="q")._preprocess(Frame({"q": np.array([0.5, 1.5])}))      # VerifyLightGBMRanker.scala:77-82


def test_frame_from_pandas_and_binary_output_shapes():
    import pandas as pd
    from mmlspark_b200.lightgbm import Frame, LightGBMBooster
    pdf = pd.DataFrame({"features": [np.array([1.0, 2.0]), np.array([3.0, 4.0])], "label": [0, 1]})
    f = Frame.of(pdf)
    assert f["features"].shape == (2, 2) and f.num_rows() == 2
    import json
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "oracle_golden.json")))["models"]["binary"]["model"]
    b = LightGBMBooster(g)                                                     # host-only: model load + predict need no GPU
    x = np.linspace(-1, 1, 10)
    raw, prob = b.score(x, True, True), b.score(x, False, True)
    assert raw.shape == (2,) and raw[0] == -raw[1] and abs(prob.sum() - 1) < 1e-12       # [-s, s] / [1-p, p] (LightGBMBooster.scala:547-563)
    assert abs(prob[1] - 1 / (1 + np.exp(-raw[1]))) < 1e-12


# ---------------------------------------------------------------- N>1 host plumbing under gloo, world_size 2
GLOO_SCRIPT = r'''
import os, sys, torch, torch.distributed as dist
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
N = 1001
n_local = N // world + (1 if rank < N % world else 0)
row_start = rank * (N // world) + min(rank, N % world)
t = torch.tensor([float(10 + rank), float(n_local)], dtype=torch.float64)
dist.all_reduce(t[:1], op=dist.ReduceOp.MAX)
s = torch.tensor([float(n_local)], dtype=torch.float64); dist.all_reduce(s, op=dist.ReduceOp.SUM)
dist.barrier()
base = int(os.environ["MASTER_PORT"]) + 512
machines = ",".join("127.0.0.1:%d" % (base + r) for r in range(world))
open(os.path.join(os.environ["OUT_DIR"], "rank%d.txt" % rank), "w").write(" ".join(str(x) for x in ["RANK", rank, "max", t[0].item(), "rows", int(s[0].item()), "start", row_start, "n", n_local, machines, base + rank]))
'''


def test_bench_multi_rank_plumbing_gloo(tmp_path):
    script = tmp_path / "g.py"
    script.write_text(GLOO_SCRIPT)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=300, env=dict(os.environ, OUT_DIR=str(tmp_path)))
    assert out.returncode == 0, out.stderr[-2000:]
    lines = sorted((tmp_path / ("rank%d.txt" % r)).read_text() for r in range(2))
    assert len(lines) == 2
    r0, r1 = lines[0].split(), lines[1].split()
    assert r0[3] == r1[3] == "11.0" and r0[5] == r1[5] == "1001"            # max over ranks, total rows
    assert (r0[7], r0[9]) == ("0", "501") and (r1[7], r1[9]) == ("501", "500")   # contiguous shards cover all rows
    assert r0[10] == r1[10] and int(r1[11]) == int(r0[11]) + 1              # same machine list, own listen port


def test_categorical_slot_names_and_slot_name_validation():
    """LightGBMBase.getCategoricalIndexes (:168-198): indexes united with the positions of the named slots;
    validateSlotNames (:218-232, 'Verify LightGBM Regressor with bad column names fails early')."""
    from mmlspark_b200.lightgbm import LightGBMClassifier, LightGBMRegressor
    est = LightGBMClassifier(slotNames=["a", "b", "c", "d"], categoricalSlotNames=["c", "a"], categoricalSlotIndexes=[3, 0])
    assert est.getCategoricalIndexes() == [3, 0, 2]
    tp = est.getTrainParams(1, {"label": np.array([0.0, 1.0])})
    assert "categorical_feature=3,0,2 " in tp.to_string()
    assert LightGBMRegressor(categoricalSlotIndexes=[1]).getCategoricalIndexes() == [1]
    assert LightGBMRegressor().getCategoricalIndexes() == []
    bad = LightGBMRegressor(slotNames=["ok", "b[a]d", 'q"uote', "fine:not"])
    with pytest.raises(ValueError) as ei:
        bad.validateSlotNames()
    assert str(ei.value) == 'Invalid slot names detected in features column: b[a]d,q"uote,fine:not'
    LightGBMRegressor(slotNames=["x_1", "y-2", "z 3"]).validateSlotNames()


def test_model_shap_accessors_dense_and_sparse_agree():
    """getFeatureShaps / getDenseFeatureShaps / getSparseFeatureShaps (LightGBMModelMethods.scala:25-46) on a loaded golden model:
    host predictor only, no GPU needed."""
    import json
    import os
    from mmlspark_b200.lightgbm import LightGBMRegressionModel
    here = os.path.dirname(os.path.abspath(__file__))
    text = json.load(open(os.path.join(here, "golden", "oracle_golden.json")))["models"]["regression"]["model"]
    m = LightGBMRegressionModel.loadNativeModelFromString(text)
    x = np.array([0.3, 0.0, 0.0, -1.2, 2.0, 0.0, 0.7, 0.0, 0.0, 1.1])
    dense = np.array(m.getFeatureShaps(x))
    assert len(dense) == 11 and np.allclose(dense, m.getDenseFeatureShaps(x))
    nz = np.nonzero(x)[0]
    sparse = np.array(m.getSparseFeatureShaps(10, nz, x[nz]))
    np.testing.assert_allclose(sparse, dense, rtol=0, atol=1e-12)
    np.testing.assert_allclose(dense.sum(), m.predict(x), rtol=0, atol=1e-12)          # contributions + expected value = prediction


@pytest.mark.parametrize("name", ["regression", "binary", "regression_categorical|categorical_feature=4", "regression_quantile"])
def test_feature_shap_equals_brute_force_shapley_values(name):
    """Independent known-answer test of the TreeSHAP predictor (C_API_PREDICT_CONTRIB, LightGBMBooster.featuresShap :412-423): the
    contributions of the host predictor equal Shapley values computed from their definition on golden models, incl. NaN rows,
    categorical splits and the expected-value slot."""
    import json
    import os
    from mmlspark_b200.lightgbm import LightGBMRegressionModel
    from mmlspark_b200.modeltext import parse_model
    from tree_walk_ref import brute_force_shap
    here = os.path.dirname(os.path.abspath(__file__))
    text = json.load(open(os.path.join(here, "golden", "oracle_golden.json")))["models"][name]["model"]
    trees = parse_model(text)["trees"]
    m = LightGBMRegressionModel.loadNativeModelFromString(text)
    F = m.getBoosterNumFeatures()
    rng = np.random.default_rng(5)
    rows = [rng.standard_normal(F) * 2 for _ in range(4)]
    rows[1][rng.integers(0, F, 2)] = np.nan
    rows[2][:] = 0.0
    if "categorical" in name:
        for r in rows:
            r[4] = float(rng.integers(0, 12))
    used = 0
    for x in rows:
        want = np.zeros(F + 1)
        for t in trees:
            phi, e = brute_force_shap(t, x)
            used = max(used, len(phi))
            for f, v in phi.items():
                want[f] += v
            want[F] += e
        got = np.array(m.getFeatureShaps(x))
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)
    assert used >= 3          # the trees really use several features
