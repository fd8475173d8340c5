"""Data-parallel training with several rank-threads of one process on ONE device: LGBM_NetworkInit sees every rank on the same GPU and
picks the same-device communicator (k_allreduce_same_device on the device's shared stream) instead of NCCL, which refuses that layout.
This is the layout of the reference's local mode whenever numTasks exceeds the GPU count.

The existing multi-rank scenarios run here unchanged with every rank on device 0: a fixture maps capi.set_device to device 0 and makes
the modules' GPU counts report enough GPUs, and their bars apply as they are (bins bit-exact, trees and leaves against the oracle's R-rank
emulation, ranks agreeing).  The tests are called through their module objects so pytest does not collect them twice."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import test_gpu_bundling as B
import test_gpu_estimators as E
import test_gpu_multi as M
import test_gpu_sparse_estimators as S
import test_gpu_wide as W
import test_gpu_xendcg_xentlambda as X
import tree_check as tc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL_NGPU = M._ngpu


@pytest.fixture
def one_device(monkeypatch):
    from mmlspark_b200 import capi
    real = capi.set_device
    monkeypatch.setattr(capi, "set_device", lambda ordinal: real(0))
    for m in (M, B, E, S, X):
        monkeypatch.setattr(m, "_ngpu", lambda: 16)
    return capi


def _cases(fn):
    return [c for mark in fn.pytestmark if mark.name == "parametrize" for c in mark.args[1]]


# ------------------------------------------------------------------------------------------------ the existing scenarios on one device
@pytest.mark.parametrize("objective,R", _cases(M.test_data_parallel_matches_oracle_emulation))
def test_multi_matches_oracle_emulation(built, one_device, objective, R):
    M.test_data_parallel_matches_oracle_emulation(built, objective, R)


def test_multi_rank_with_single_class(built, one_device):
    M.test_rank_with_single_class_does_not_hang(built)


@pytest.mark.parametrize("mode", _cases(M.test_data_parallel_row_sampling))
def test_multi_row_sampling(built, one_device, mode):
    M.test_data_parallel_row_sampling(built, mode)


def test_multi_push_rows_ingestion(built, one_device):
    M.test_data_parallel_push_rows_ingestion(built)


@pytest.mark.parametrize("fmt", _cases(B.test_two_ranks_bundled_equals_unbundled))
def test_bundling_two_ranks(built, one_device, fmt):
    B.test_two_ranks_bundled_equals_unbundled(built, fmt)


def test_xendcg_two_ranks(built, one_device):
    X.test_two_ranks_xendcg_seeds_each_ranks_queries_by_local_index(built)


def test_xentlambda_two_ranks(built, one_device):
    X.test_two_ranks_xentlambda_init_score_from_global_sums(built)


def test_estimator_two_tasks(built, one_device):
    E.test_two_tasks_two_gpus(built)


def test_sparse_estimator_two_tasks(built, one_device):
    S.test_two_tasks_sparse(built)


# ------------------------------------------------------------------------------------------------ helpers
def _regression_data(seed, n, F=20):
    rng = np.random.default_rng(seed)
    X_ = rng.standard_normal((n, F))
    y = (1.5 * X_[:, 0] + np.sin(2 * X_[:, 1]) + X_[:, 2] * X_[:, 3] + 0.3 * rng.standard_normal(n)).astype(np.float32)
    return X_, y


def _train_shards(X_, y, rank_rows, params, iters):
    """body for tree_check.on_ranks: rank r trains on its contiguous shard and returns its model, scores, GetInfo and memory info"""
    from mmlspark_b200 import capi
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        ds = capi.Dataset.from_mat(X_[sl], M.DS_PARAMS).set_field("label", y[sl])
        b = capi.Booster(ds, params)
        try:
            for _ in range(iters):
                if b.update_one_iter():
                    break
            return dict(model=b.save_model_to_string(), scores=b.get_scores(), info=b.get_info(), mem=b.get_memory_info())
        finally:
            b.free()
            ds.free()
    return body


# ------------------------------------------------------------------------------------------------ new scenarios
def test_wide_categorical_two_ranks_on_one_device(built):
    """the wide features' mapper records travel in the same-device all-gather, their histograms in the all-reduce"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    n = 100_000
    X_, s = W._data(6, n)
    y = (s > 0).astype(np.float32)
    rank_rows = [n // 2 + 500, n - n // 2 - 500]
    params = W._params("binary", "is_unbalance=false", machines=2)
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        ds = capi.Dataset.from_mat(X_[sl], W.DS).set_field("label", y[sl])
        b = capi.Booster(ds, params)
        for _ in range(6):
            b.update_one_iter()
        res = dict(model=b.save_model_to_string(), bins=ds.get_bins16(), info=b.get_info())
        b.free(); ds.free()
        return res

    res, errs = tc.on_ranks(2, 26000, body)
    assert not errs, errs
    ods = O.OracleDataset(X_, W.DS, rank_rows=rank_rows).set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(6)
    want = ods.bins16()
    for r in range(2):
        assert res[r]["info"]["reduce_mode"] == 3
        assert np.array_equal(res[r]["bins"], want[offs[r]:offs[r + 1]])
    assert res[0]["model"] == res[1]["model"]
    compare_models(parse_model(res[0]["model"]), parse_model(ob.model_string()))


def test_three_ranks_unequal_shards(built, one_device):
    """R = 3 on one device (rank-ordered double sums: a NCCL run may differ in the last bits, the oracle emulation bar holds); the last
    shard has fewer rows than min_data_in_leaf"""
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    n = 60_000
    X_, y = _regression_data(31, n, F=24)
    rank_rows = [n // 2, n - n // 2 - 7, 7]
    params = M._params("regression", 3)
    res = M.run_ranks(X_, y, rank_rows, params, 12, 26100)
    ods = O.OracleDataset(X_, M.DS_PARAMS, rank_rows=rank_rows).set_field("label", y)
    ob = O.OracleBooster(ods, params)
    ob.train(12)
    obins = ods.bins()
    offs = np.concatenate([[0], np.cumsum(rank_rows)])
    for r in range(3):
        assert np.array_equal(res[r]["bins"], obins[offs[r]:offs[r + 1]]), "rank %d bins differ" % r
        assert res[r]["model"] == res[0]["model"]
    compare_models(parse_model(res[0]["model"]), parse_model(ob.model_string()))
    np.testing.assert_allclose(np.concatenate([res[r]["scores"] for r in range(3)]), ob.scores(), rtol=1e-6, atol=1e-6)


def test_reduce_mode_is_same_device(built):
    """GetInfo reports world, rank and reduce mode 3, and both ranks hold the same model"""
    n = 40_000
    X_, y = _regression_data(41, n)
    rank_rows = [n // 2 + 99, n - n // 2 - 99]
    params = M._params("regression", 2)
    res, errs = tc.on_ranks(2, 26200, _train_shards(X_, y, rank_rows, params, 8))
    assert not errs, errs
    for r in range(2):
        assert res[r]["info"]["num_machines"] == 2 and res[r]["info"]["rank"] == r and res[r]["info"]["reduce_mode"] == 3
    assert res[1]["model"] == res[0]["model"]


def test_column_copy_with_four_ranks_on_one_device(built, monkeypatch):
    """each rank's partition column copy comes out of its 1/R share of the spare memory, and results do not depend on the copy"""
    n = 80_000
    X_, y = _regression_data(51, n)
    rank_rows = [n // 4] * 4
    params = M._params("regression", 4)
    res, errs = tc.on_ranks(4, 26300, _train_shards(X_, y, rank_rows, params, 6))
    assert not errs, errs
    monkeypatch.setenv("B200GBM_COLUMN_COPY", "0")
    off, errs = tc.on_ranks(4, 26310, _train_shards(X_, y, rank_rows, params, 6))
    assert not errs, errs
    for r in range(4):
        assert res[r]["model"] == res[0]["model"] and off[r]["model"] == res[0]["model"]
        assert off[r]["mem"]["partition_column_copy_bytes"] == 0
    copies = [res[r]["mem"]["partition_column_copy_bytes"] for r in range(4)]
    assert min(copies) > 0
    # the ranks decided on the same free memory F before allocating: 4 * copy <= F - reserve <= (free now + the copies made since)
    free_now = min(res[r]["mem"]["device_free_bytes"] for r in range(4))
    assert 4 * max(copies) <= free_now + sum(copies)


_INIT_ONE_RANK = """
import sys, time
sys.path.insert(0, %r)
from mmlspark_b200 import capi
capi.set_device(0)
t0 = time.time()
try:
    capi.network_init(%r, %d, 60, 2)
    capi.network_free()
    print("INIT-OK")
except capi.LightGBMError as e:
    print("INIT-FAILED %%.1f %%s" %% (time.time() - t0, e))
"""


def test_ranks_of_two_processes_on_one_device_are_rejected(built):
    """two processes on device 0 need CUDA IPC and a cross-process rendezvous: both ranks fail at once with the layout message"""
    machines = "127.0.0.1:26400,127.0.0.1:26401"
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    procs = [subprocess.Popen([sys.executable, "-c", _INIT_ONE_RANK % (ROOT, machines, 26400 + r)], cwd=ROOT, env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=180) for p in procs]
    for out, err in outs:
        line = [l for l in out.splitlines() if l.startswith("INIT-")]
        assert line and line[0].startswith("INIT-FAILED"), (out, err)
        secs = float(line[0].split()[1])
        assert secs < 30, line[0]
        assert "ranks 0,1 share CUDA device" in line[0] and "supported layouts" in line[0], line[0]


def test_a_rank_that_fails_releases_the_others(built):
    """rank 1 fails in BoosterCreate (a cross_entropy label outside [0, 1] on its shard only) and frees the network: rank 0 fails with
    'left the network' long before the timeout, and a single-rank training in the same process works afterwards"""
    from mmlspark_b200 import capi
    n = 20_000
    X_, _ = _regression_data(61, n)
    y = (np.random.default_rng(62).random(n)).astype(np.float32)
    y[n - 5] = 1.5
    params = M._params("cross_entropy", 2)
    t0 = time.time()
    _, errs = tc.on_ranks(2, 26500, _train_shards(X_, y, [n // 2, n - n // 2], params, 5), timeout=100)
    elapsed = time.time() - t0
    by_rank = dict(errs)
    assert "outside [0, 1]" in by_rank.get(1, ""), errs
    assert "left the network" in by_rank.get(0, ""), errs
    assert elapsed < 50, elapsed
    ds = capi.Dataset.from_mat(X_[: n // 2], M.DS_PARAMS).set_field("label", y[: n // 2])
    b = capi.Booster(ds, params.replace("num_machines=2", "num_machines=1"))
    for _ in range(3):
        b.update_one_iter()
    assert b.get_info()["num_machines"] == 1 and np.isfinite(b.get_scores()).all()
    b.free(); ds.free()


# ------------------------------------------------------------------------------------------------ with two or more GPUs
def test_same_device_model_equals_nccl_model(built):
    if REAL_NGPU() < 2:
        pytest.skip("needs 2 GPUs")
    n = 40_000
    X_, y = _regression_data(71, n)
    rank_rows = [n // 2 + 5, n - n // 2 - 5]
    params = M._params("regression", 2)
    same, errs = tc.on_ranks(2, 26600, _train_shards(X_, y, rank_rows, params, 10))
    assert not errs, errs
    nccl, errs = tc.on_ranks(2, 26610, _train_shards(X_, y, rank_rows, params, 10), device_of=lambda r: r)
    assert not errs, errs
    assert same[0]["info"]["reduce_mode"] == 3 and nccl[0]["info"]["reduce_mode"] == 0
    assert same[0]["model"] == nccl[0]["model"]


def test_three_ranks_on_two_devices_are_rejected(built):
    if REAL_NGPU() < 2:
        pytest.skip("needs 2 GPUs")
    _, errs = tc.on_ranks(3, 26700, lambda r: None, device_of=lambda r: r % 2, timeout=60)
    assert sorted(r for r, _ in errs) == [0, 1, 2], errs
    for _, e in errs:
        assert "ranks 0,2 share CUDA device" in e and "supported layouts" in e, e
