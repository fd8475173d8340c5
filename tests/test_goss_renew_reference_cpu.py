"""The GOSS, bagging and renewal restatements (goss_ref.py, tree_check.bags, renew_ref.py) on hand-worked cases, without a GPU."""
import numpy as np
import pytest

import goss_ref as G
import renew_ref as RN
import tree_check as tc


def lcg(x, steps):
    """LightGBM's Random, written out: the state after `steps` draws and the draws"""
    out = []
    for _ in range(steps):
        x = (214013 * x + 2531011) % 2 ** 32
        out.append(((x >> 16) & 0x7FFF) / 32768)
    return x, out


# ---------------------------------------------------------------------------------------------------------------- PercentileFun
def test_percentile_is_the_linear_quantile():
    rng = np.random.default_rng(0)
    for cnt in (2, 3, 5, 17, 400):
        v = rng.standard_normal(cnt)
        for alpha in (0.01, 0.3, 0.5, 0.77, 0.99):
            assert abs(RN.percentile(v, alpha) - np.quantile(v, alpha, method="linear")) <= 1e-12 * max(1.0, np.abs(v).max())


def test_percentile_hand_worked():
    assert RN.percentile([3.0, 1.0, 4.0, 2.0], 0.5) == 2.5            # fp = 1.5: 3 - (3 - 2) * 0.5
    assert RN.percentile([7.0], 0.3) == 7.0                           # one row
    assert RN.percentile([2.0, 6.0], 0.5) == 4.0
    assert RN.percentile([2.0, 6.0, 1.0], 0.25) == 1.5                # fp = 1.5 in the descending order 6, 2, 1
    assert RN.percentile([2.0, 6.0, 1.0], 0.0) == 1.0                 # pos = cnt: the smallest
    assert RN.percentile([2.0, 6.0, 1.0], 2.0) == 6.0                 # fp = -2, pos = -1 < 1: the largest
    assert RN.percentile([2.0, 6.0, 1.0], 1.0) == 6.0                 # fp = 0, pos = 1, bias 0


def test_quantile_alpha_is_float32():
    """11 rows at alpha 0.3: (cnt - 1)(1 - alpha) is 7.0 in double and 6.99999988 with alpha as float32"""
    v = np.arange(11, dtype=np.float64)[::-1].copy()
    a32 = RN.renew_alpha("quantile", 0.3)
    assert a32 == float(np.float32(0.3)) and RN.renew_alpha("regression_l1", 0.3) == 0.5
    assert (11 - 1) * (1.0 - 0.3) == 7.0 and (11 - 1) * (1.0 - a32) < 7.0
    assert RN.percentile(v, 0.3) == 3.0
    got = RN.percentile(v, a32)
    assert got != 3.0 and got == 4.0 - 1.0 * ((11 - 1) * (1.0 - a32) - 6)


def test_percentile_float32_labels():
    """the init score's label percentile: T = float32, v1 - v2 taken in float32"""
    y = np.array([3.0, 1e8], np.float32)         # d = 1e8, 3; fp = 0.7; 1e8 - 3 rounds to 1e8 in float32
    got = RN.percentile(y, 0.3, np.float32)
    assert isinstance(got, np.float32)
    assert got == np.float32(3e7) and np.float32(1e8 - (1e8 - 3.0) * (1 - 0.3)) == np.float32(30000002.0)


# ---------------------------------------------------------------------------------------------------------------- WeightedPercentileFun
@pytest.mark.parametrize("values, weights, want", [
    ([1.0, 2.0, 3.0], [10.0, 1.0, 1.0], 1.0),                 # cdf 10 11 12, threshold 6: pos 0
    ([3.0, 1.0, 2.0], [10.0, 1.0, 1.0], 3.0),                 # cdf 1 2 12: pos = cnt - 1
    ([1.0, 2.0, 3.0, 4.0], [1.0, 1.0, 2.0, 2.0], 1.5),        # cdf 1 2 4 6, threshold 3: pos 2, step 2 >= 1: (3 - 4) / 2 * (3 - 2) + 2
    ([1.0, 2.0, 3.0, 4.0], [1.0, 1.0, 0.5, 0.5], 2.0),        # cdf 1 2 2.5 3, threshold 1.5: pos 1, step 0.5 < 1: v2
    ([1.0, 2.0, 3.0, 4.0], [1.0, 1.0, 1.0, 1.0], 1.0),        # threshold 2 equals cdf[1]: upper_bound gives pos 2, (2 - 3) / 1 * 1 + 2
    ([5.0, 5.0, 1.0], [3.0, 1.0, 1.0], -5.0),                 # tied 5s in row order: cdf 1 4 5, pos 1, (2.5 - 4) / 1 * 4 + 1
    ([5.0, 5.0, 1.0], [1.0, 3.0, 1.0], 5.0),                  # the same rows in the other order: cdf 1 2 5, pos = cnt - 1
    ([4.0], [0.3], 4.0),
])
def test_weighted_percentile_hand_worked(values, weights, want):
    why = []
    assert RN.weighted_percentile(values, weights, 0.5, why=why) == want
    assert not why


def test_weighted_keeps_the_sign_of_zero():
    got = RN.weighted_percentile([0.0, -0.0], [1.0, 1.0], 0.5)         # -0.0 ties with +0.0: row order, cdf 1 2, pos 1
    assert got == 0.0 and np.signbit(got)
    got = RN.weighted_percentile([-0.0, 0.0], [1.0, 1.0], 0.5)
    assert got == 0.0 and not np.signbit(got)
    assert np.signbit(RN.percentile([-0.0, 0.0, 1.0], 0.5)) == np.signbit(np.float64(0.0))   # d = 1, +0.0, -0.0: d[1] is the later row


def test_weighted_undecided_threshold():
    why = []
    RN.weighted_percentile([1.0, 2.0, 3.0], [1.0, 2.0 ** -52, 1.0], 0.5, why=why)   # threshold 1 + 2^-53 rounds near cdf[0] = 1
    RN.weighted_percentile([1.0, 2.0, 3.0], [1.0, 1.0 + 2.0 ** -51, 1.0 + 2 ** -51], 0.5, why=why)
    assert why


def test_mape_weights():
    y = np.array([0.5, -3.0, 7.0, 1e6], np.float32)
    assert RN.mape_weights(y).tolist() == [1.0, np.float32(1 / 3.0), np.float32(1 / 7.0), np.float32(1e-6)]
    w = np.array([2.0, 2.0, 0.5, 1.0], np.float32)
    assert RN.mape_weights(y, w).dtype == np.float32 and RN.mape_weights(y, w)[1] == np.float32(np.float32(1 / 3.0) * 2)


def test_renew_averages_over_the_ranks_with_rows():
    label = np.array([1, 2, 3, 10, 20, 30, 7], np.float32)
    rank = np.array([0, 0, 0, 1, 1, 1, 1])
    leaves = [np.array([0, 1, 3, 4]), np.array([2, 5, 6]), np.array([], int), np.array([0, 1])]
    got = RN.renew(leaves, label, 0.0, 0.5, rank_of_row=rank, R=2)
    assert got == [(1.5 + 15.0) / 2, (3.0 + 18.5) / 2, 0.0, 1.5]
    assert RN.renew(leaves[:2], label, np.ones(7), 0.5) == [5.0, 6.0]


# ---------------------------------------------------------------------------------------------------------------- the cdf's summation order
def wide_leaf(seed=5, cnt=4000):
    """a leaf whose float32 weights span 1..1e7 (log-uniform): the block scan's adds round"""
    rng = np.random.default_rng(seed)
    return rng.standard_normal(cnt), (10.0 ** rng.uniform(0, 7, cnt)).astype(np.float32)


def test_wide_weights_discriminate():
    res, w = wide_leaf()
    order, cdf = RN.weighted_cdf(res, w)
    assert not np.array_equal(cdf, RN.block_scan_cdf(w[order]))
    threshold = cdf[-1] * 0.3
    pos = int(np.searchsorted(cdf, threshold, side="right"))
    sh = RN.block_scan_cdf(w[order])
    step, step_sh = cdf[pos + 1] - cdf[pos], sh[pos + 1] - sh[pos]
    v1, v2 = res[order[pos - 1]], res[order[pos]]
    emulated = (sh[-1] * 0.3 - sh[pos]) / step_sh * (v2 - v1) + v1
    assert int(np.searchsorted(sh, sh[-1] * 0.3, side="right")) == pos and step >= 1.0
    assert RN.weighted_percentile(res, w, 0.3) != emulated
    # weights in [0.5, 2] on the same rows: every add of either order is exact
    narrow = np.float32(0.5) + (np.round(np.random.default_rng(1).uniform(0, 1.5, len(w)) * 64) / 64).astype(np.float32)
    assert np.array_equal(RN.weighted_cdf(res, narrow)[1], RN.block_scan_cdf(narrow[order]))


# ---------------------------------------------------------------------------------------------------------------- GOSS
def test_goss_ties_at_the_threshold_are_kept():
    g = np.array([[5.0, 5.0, 1.0, 1.0]], np.float32)
    h = np.ones_like(g)
    # top_k = 1, other_k = 2, multiply = 3 / 2; both 5s are top; row 2 draws 0.00116 < 2/3, row 3 draws 0.2356 < (2 - 1) / (1 + 1)
    bag, g2, h2, st = G.draw(g, h, G.seeds(4, 0), 0.25, 0.5)
    assert bag.tolist() == [True] * 4
    assert g2.tolist() == [[5.0, 5.0, 1.5, 1.5]] and h2.tolist() == [[1.0, 1.0, 1.5, 1.5]]
    assert int(st[0]) == lcg(0, 2)[0]


def test_goss_threshold_uses_the_float32_class_sum():
    """(2^24, 1) and (2^24, 0) both sum to 2^24 in float32: a tie at the threshold, so both rows are top"""
    g = np.array([[2.0 ** 24, 2.0 ** 24, 1.0, 1.0], [1.0, 0.0, 0.0, 0.0]], np.float32)
    h = np.ones_like(g)
    flag, multiply, x = G.block_draw(g, h, np.uint64(0), 0.25, 0.25)
    assert flag[:2].tolist() == [1, 1] and multiply == np.float32(3.0)
    # rows 2, 3: other_k = 1, rest_need 1 over rest_all (2 - (1 - 2)) = 3, then (1 - taken) over 2
    d = lcg(0, 2)[1]
    assert flag[2] == (2 if d[0] < 1 / 3 else 0) and int(x) == lcg(0, 2)[0]


def test_goss_zero_block_and_tail_block():
    rng = np.random.default_rng(3)
    n = 2 * 1024 + 3
    g = (rng.integers(1, 50, (1, n)) / 8.0).astype(np.float32)
    g[0, :1024] = 0.0                                          # every tg is 0: every row is top, the state does not move
    h = np.ones_like(g)
    bag, g2, h2, st = G.draw(g, h, G.seeds(n, 9), 0.2, 0.1)
    assert bag[:1024].all() and int(st[0]) == 9
    assert np.array_equal(g2[:, :1024], g[:, :1024])
    # the 3-row tail: top_k = 1, other_k = 0 (multiply is inf): one top row, two draws at probability 0
    tail = slice(2048, n)
    assert bag[tail].sum() == 1 and bag[tail][np.argmax(g[0, tail])] and int(st[2]) == lcg(11, 2)[0]
    assert np.array_equal(g2[:, tail], g[:, tail])
    # the middle block: 204 top rows (no ties in a 1/8 grid of 49 values? ties are kept, so at least 204), about 102 sampled, ×8.039
    mid = slice(1024, 2048)
    m = np.float32(1024 - 204) / np.float32(102)
    amp = bag[mid] & (g2[0, mid] != g[0, mid])
    assert np.array_equal(g2[0, mid][amp], (g[0, mid][amp] * m).astype(np.float32))
    assert (g[0, mid][bag[mid] & ~amp] >= np.sort(g[0, mid])[::-1][203]).all()


def test_goss_state_carries():
    rng = np.random.default_rng(4)
    g = rng.standard_normal((1, 1024)).astype(np.float32)
    h = np.ones_like(g)
    b1, _, _, s1 = G.draw(g, h, G.seeds(1024, 3), 0.2, 0.1)
    b2, _, _, s2 = G.draw(g, h, s1, 0.2, 0.1)
    top = np.abs(g[0]) >= np.sort(np.abs(g[0]))[::-1][203]
    assert int(s1[0]) == lcg(3, 1024 - top.sum())[0] and int(s2[0]) == lcg(3, 2 * (1024 - top.sum()))[0]
    assert (b1 & top).sum() == (b2 & top).sum() == top.sum() and not np.array_equal(b1, b2)


def test_goss_warm_up():
    assert G.warm_up(1.0) == 1 and G.warm_up(0.3) == 3 and G.warm_up(0.1) == 10 and G.warm_up(0.7) == 1


# ---------------------------------------------------------------------------------------------------------------- bagging
def test_bags_freq_and_balanced():
    plain = tc.bags(3000, 4, 0.6, 3)
    every3 = tc.bags(3000, 7, 0.6, 3, freq=3)
    assert [b is every3[0] for b in every3[:3]] == [True] * 3 and every3[3] is every3[5]
    assert np.array_equal(every3[0], plain[0]) and np.array_equal(every3[3], plain[1]) and np.array_equal(every3[6], plain[2])
    label = (np.arange(3000) % 3 == 0).astype(np.float32)
    bal = tc.bags(3000, 2, 1.0, 3, label=label, pos=0.9, neg=0.3)
    x, d = lcg(3, 1024)
    want = [dj < (0.9 if label[j] > 0 else 0.3) for j, dj in enumerate(d)]
    assert bal[0][:1024].tolist() == want
    assert np.array_equal(tc.bags(3000, 2, 0.6, 3, label=label, pos=0.6, neg=0.6)[1], plain[1])
