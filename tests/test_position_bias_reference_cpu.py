"""The NumPy restatement of the ranking objectives' position factors (position_bias_ref.py) on hand-worked cases, and the ranker's
parameter string; no GPU needed."""
import numpy as np

import position_bias_ref as P


def test_two_positions_one_step():
    ids = np.array([0, 1, 0, 1])
    g = np.array([-1.0, 0.5, -1.0, 0.5], np.float32)
    h = np.array([0.5, 0.25, 0.5, 0.25], np.float32)
    b = P.update(np.zeros(2), ids, g, h, 0.1, 0.0)
    # position 0: d1 = 2, d2 = -1; position 1: d1 = -1, d2 = -0.5
    assert b[0] == (0.1 * 2.0) / (1.0 + 0.001)
    assert b[1] == (0.1 * -1.0) / (0.5 + 0.001)
    assert b[0] > 0 > b[1]


def test_regularisation_pulls_factors_toward_zero():
    ids = np.array([0, 0, 1, 1, 1])
    zero = np.zeros(5, np.float32)
    b0 = np.array([1.0, -2.0])
    b = P.update(b0, ids, zero, zero, 0.5, 1.0)
    # d1 = -b reg cnt, d2 = -reg cnt: b - 0.5 b cnt / (cnt + 0.001)
    assert b[0] == 1.0 + (0.5 * -(1.0 * 1.0 * 2.0)) / (2.0 + 0.001)
    assert b[1] == -2.0 + (0.5 * -(-2.0 * 1.0 * 3.0)) / (3.0 + 0.001)
    assert (np.abs(b) < np.abs(b0)).all() and (np.sign(b) == np.sign(b0)).all()
    assert (P.update(b0, ids, zero, zero, 0.5, 0.0) == b0).all()      # no gradient and no regularisation: nothing moves


def test_weighted_gradients_enter_the_sums():
    ids = np.array([0, 0])
    g = np.array([-1.0, -1.0], np.float32)
    h = np.array([1.0, 1.0], np.float32)
    w = np.array([2.0, 0.5], np.float32)
    b = P.update(np.zeros(1), ids, g * w, h * w, 1.0, 0.0)
    assert b[0] == 2.5 / (2.5 + 0.001)


def test_negative_and_sparse_position_values():
    values, (ids,) = P.position_ids([np.array([-7, 1000000, -7, 3, -2147483648], np.int32)])
    assert values.tolist() == [-2147483648, -7, 3, 1000000]
    assert ids.tolist() == [1, 3, 1, 2, 0]


def test_fixed_point_grid_and_order():
    assert P.exponent(np.float32(1.0)) == 34 and P.exponent(np.float32(0.75)) == 35 and P.exponent(np.float32(0)) == 0
    assert P.exponent(np.float32(np.inf)) == 0
    # at max |g| = 1 the grid is 2^-34: 2^-40 rounds to 0, 3 * 2^-35 rounds half to even
    g = np.array([1.0, 2.0 ** -40, 3 * 2.0 ** -35], np.float32)
    qg, qh, cnt = P.fixed_sums(np.zeros(3, np.int64), g, np.ones(3, np.float32), 1, 34, 34)
    assert qg[0] == 2 ** 34 + 0 + 2 and cnt[0] == 3 and qh[0] == 3 * 2 ** 34
    rng = np.random.default_rng(0)
    ids = rng.integers(0, 5, 1000)
    g, h = rng.standard_normal(1000).astype(np.float32), rng.random(1000).astype(np.float32)
    perm = rng.permutation(1000)
    a = P.update(np.zeros(5), ids, g, h, 0.1, 0.3)
    assert np.array_equal(a, P.update(np.zeros(5), ids[perm], g[perm], h[perm], 0.1, 0.3))


def test_ranks_equal_one_rank_with_an_id_missing_on_one_rank():
    pos = [np.array([1, 2, 1, 2], np.int32), np.array([2, 5, 5], np.int32)]
    values, ids = P.position_ids(pos)
    assert values.tolist() == [1, 2, 5]
    assert ids[0].tolist() == [0, 1, 0, 1] and ids[1].tolist() == [1, 2, 2]
    rng = np.random.default_rng(1)
    g = [rng.standard_normal(4).astype(np.float32), 8 * rng.standard_normal(3).astype(np.float32)]      # rank 1 sets the exponent
    h = [rng.random(4).astype(np.float32), rng.random(3).astype(np.float32)]
    b = rng.standard_normal(3)
    split = P.update(b, ids, g, h, 0.2, 0.1)
    one = P.update(b, np.concatenate(ids), np.concatenate(g), np.concatenate(h), 0.2, 0.1)
    assert np.array_equal(split, one)


def test_adjusted_scores_move_the_gradients():
    """a two-document query at equal scores: a factor that lifts the relevant document lowers its lambda's magnitude"""
    y = np.array([1.0, 0.0], np.float32)
    s = np.zeros(2)
    ids = np.array([0, 1])
    g0, _ = P.lambdarank(s, ids, np.zeros(2), y, None, [2], norm=False)
    g1, _ = P.lambdarank(s, ids, np.array([1.0, 0.0]), y, None, [2], norm=False)
    assert g0[0] < g1[0] < 0 and g0[1] > g1[1] > 0
    from test_gpu_gradients import reference_lambdarank
    assert np.array_equal(g1, reference_lambdarank(np.array([1.0, 0.0]), y, None, [2], 30, False)[0])


def test_ranker_parameter_string_only_changes_when_the_regularisation_is_set():
    from mmlspark_b200.lightgbm.params import TrainParams
    from mmlspark_b200.lightgbm.estimators import LightGBMRanker
    plain = TrainParams("ranker", LightGBMRanker().params_dict(), 1).to_string()
    with_col = TrainParams("ranker", LightGBMRanker(positionCol="pos").params_dict(), 1).to_string()
    assert plain == with_col and "position_bias" not in plain
    reg = TrainParams("ranker", LightGBMRanker(positionCol="pos", lambdarankPositionBiasRegularization=0.5).params_dict(), 1).to_string()
    assert reg == plain + "lambdarank_position_bias_regularization=0.5 "
