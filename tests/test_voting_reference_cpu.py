"""The NumPy restatement of the voting-parallel learner (voting_ref.py, grown by tree_ref.py) on its own: the vote rule on hand-made records, the local top-k
order, one rank as the serial learner, and shard-skewed data on which the vote decides the tree.  No GPU."""
import math

import numpy as np
import pytest

import split_scan_ref as ref
import tree_ref
import voting_ref as V

GRID = 1.0 / 1024


def test_vote_weights_gain_by_rows_and_keeps_each_features_best():
    # mean = 100 / 2 = 50: weights 2 * 60/50 = 2.4, 3 * 10/50 = 0.6, 1 * 100/50 = 2, 2.5 * 40/50 = 2
    records = [(7, 2.0, 30, 30), (4, 3.0, 5, 5), (9, 1.0, 50, 50), (4, 2.5, 20, 20)]
    assert V.vote(records, 100, 2, 3) == [7, 4, 9]
    # feature 4's best record is its 2.5 one (weight 2): it ties feature 9, and the smaller index comes first
    assert V.vote(records, 100, 2, 2) == [7, 4]
    # -inf gains and feature -1 never enter the vote, and fewer voted features than top_k is fine
    assert V.vote([(3, -math.inf, 0, 10), (-1, 5.0, 5, 5), (2, 0.5, 5, 5)], 20, 2, 3) == [2]


def test_vote_mean_is_fp32():
    """score_t mean = global count / R in fp32.  Two records one ulp apart: divided by the fp64 mean they tie (feature 0 would win on
    index), divided by the fp32 mean they stay apart (feature 1 wins)"""
    count, R = 21271165, 7
    lo, hi = 1.5414612202490918, 1.541461220249092
    m32, m64 = float(np.float32(count) / np.float32(R)), count / R
    assert lo / m64 == hi / m64 and lo / m32 < hi / m32
    assert V.vote([(0, lo, 1, 0), (1, hi, 1, 0)], count, R, 1) == [1]


def test_local_top_k_order():
    class S:
        def __init__(self, f, gain, lc, n):
            self.feature, self.gain, self.left_count, self.num_data = f, gain, lc, n
    scans = {f: S(f, gain, 3, 10) for f, gain in [(5, 1.0), (2, 1.0), (8, 2.0), (1, -math.inf)]}
    assert V.local_top_k(scans, 3) == [(8, 2.0, 3, 7), (2, 1.0, 3, 7), (5, 1.0, 3, 7)]
    assert V.local_top_k(scans, 10)[-1][0] == 5          # the -inf candidate sends no record


def _skewed_bins(seed, rank_rows, F=12, nbin=16):
    """bins [n][F] and grid (g, h): rank r's gradients step on feature r, every rank's on feature F-1 more weakly"""
    rng = np.random.default_rng(seed)
    R, n = len(rank_rows), int(sum(rank_rows))
    bins = rng.integers(0, nbin, (n, F))
    rank_of_row = np.repeat(np.arange(R), rank_rows)
    g = np.where(bins[:, F - 1] < nbin // 2, -0.7, 0.7)
    for r in range(R):
        on = rank_of_row == r
        g[on] += np.where(bins[on, r] < nbin // 2, -1.0, 1.0)
    g = np.round((g + rng.integers(-64, 65, n) * GRID) / GRID) * GRID
    h = rng.integers(512, 1537, n) * GRID
    feats = [ref.Feature(f, nbin) for f in range(F)]
    return bins, g, h, feats, rank_of_row


def test_one_rank_is_the_serial_learner():
    bins, g, h, feats, rank_of_row = _skewed_bins(1, [3000])
    p = ref.Params(min_data_in_leaf=20)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 8, voting=(rank_of_row, 1, 1))
    S = tree_ref.grow_tree(bins, g, h, feats, p, 8)
    for k in ("split_feature", "threshold_bin", "left_child", "right_child", "leaf_count", "leaf_value"):
        assert T[k] == S[k]


@pytest.mark.parametrize("R", [2, 3])
def test_skewed_shards_vote_for_their_own_features(R):
    """with top_k = 1 each rank sends its own feature: the shared feature F-1, which the serial (and data-parallel) learner splits the root
    on, is never voted at the root, so the trees differ; with top_k = R + 1 it is voted as every rank's second best; with top_k = F every locally splittable feature is voted and the root split is
    the serial one"""
    rank_rows = [2000 + 13 * r for r in range(R)]
    bins, g, h, feats, rank_of_row = _skewed_bins(10 + R, rank_rows)
    F = len(feats)
    p = ref.Params(min_data_in_leaf=20)
    S = tree_ref.grow_tree(bins, g, h, feats, p, 8)
    assert S["split_feature"][0] == F - 1
    T1 = tree_ref.grow_tree(bins, g, h, feats, p, 8, voting=(rank_of_row, R, 1))
    assert T1["voted"][0][1] is None and T1["voted"][0][0][0] in range(R)
    assert T1["split_feature"][0] in range(R) and T1["split_feature"] != S["split_feature"]
    for smaller, larger in T1["voted"]:
        assert len(smaller) <= 1 and (larger is None or len(larger) <= 1)
    T3 = tree_ref.grow_tree(bins, g, h, feats, p, 8, voting=(rank_of_row, R, R + 1))
    assert F - 1 in T3["voted"][0][0] and T3["split_feature"][0] == F - 1      # every rank's second best: the shared feature
    TF = tree_ref.grow_tree(bins, g, h, feats, p, 8, voting=(rank_of_row, R, F))
    assert TF["split_feature"][0] == S["split_feature"][0] and TF["threshold_bin"][0] == S["threshold_bin"][0]
    # counts of a voting tree are the hessian-rebuilt global counts of its splits, and they add up at every node
    for T in (T1, T3, TF):
        assert sum(T["leaf_count"]) == sum(rank_rows)


def test_local_config_divides_min_data_and_min_hessian():
    q = V.local_params(ref.Params(min_data_in_leaf=21, min_sum_hessian_in_leaf=1.5), 4)
    assert q.min_data_in_leaf == 5 and q.min_sum_hessian_in_leaf == 0.375
