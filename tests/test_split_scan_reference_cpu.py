"""Pins split_scan_ref.py, the NumPy restatement of LightGBM 3.2's split search that test_gpu_split_scan.py compares the engine with:
brute force over every threshold with partitions built directly from rows, and hand-worked cases for the rules a brute force does not
exercise by chance."""
import math

import numpy as np
import pytest

import split_scan_ref as ref
import tree_ref

GRID = 1.0 / 1024


def _brute(col, g, h, num_bin, missing_type, offset, p):
    n = len(col)
    sum_g, sum_h = math.fsum(g), math.fsum(h) + 2 * ref.K_EPS
    cf = n / sum_h
    bin_h = np.bincount(col, weights=h, minlength=num_bin)
    cnt = [ref.round_int(x * cf) for x in bin_h]
    shift = ref.leaf_gain(sum_g, sum_h, p, p.lambda_l2) + p.min_gain_to_split
    two_way = num_bin > 2 and missing_type == 2
    na = num_bin - 1
    out = []          # (gain, threshold, default_left) of evaluated candidates in scan order, per pass
    for reverse in (True, False) if two_way else (True,):
        if reverse:
            order = range(num_bin - 2 - (1 if two_way else 0), -1, -1)
            near = lambda t: (col > t) & ~((col == na) & two_way)                   # the side the reverse scan accumulates
            near_bins = lambda t: [b for b in range(t + 1, num_bin - (1 if two_way else 0))]
        else:
            order = range(0, num_bin - 1)
            near = lambda t: (col <= t) | ((col == 0) & (offset == 1))
            near_bins = None
        res = []
        for t in order:
            m = near(t)
            ng, nh = math.fsum(g[m]), math.fsum(h[m])
            if reverse:
                nc = sum(cnt[b] for b in near_bins(t))
                nh_e = ref.K_EPS + nh
            else:
                if offset == 1:
                    nc = n - sum(cnt[1:num_bin]) + sum(cnt[b] for b in range(1, t + 1))
                    stored_h = math.fsum(h[col >= 1])
                    nh_e = (sum_h - ref.K_EPS) - stored_h + math.fsum(h[(col >= 1) & (col <= t)])
                    ng = sum_g - math.fsum(g[col >= 1]) + math.fsum(g[(col >= 1) & (col <= t)])
                else:
                    nc = sum(cnt[b] for b in range(0, t + 1))
                    nh_e = ref.K_EPS + nh
            if nc < p.min_data_in_leaf or nh_e < p.min_sum_hessian_in_leaf:
                continue
            fc, fh = n - nc, sum_h - nh_e
            if fc < p.min_data_in_leaf or fh < p.min_sum_hessian_in_leaf:
                break
            gain = ref.leaf_gain(ng, nh_e, p, p.lambda_l2) + ref.leaf_gain(sum_g - ng, fh, p, p.lambda_l2)
            if gain > shift:
                res.append((gain, t, reverse and not (missing_type == 2 and not two_way)))
        out.append(res)
    best = None
    for res in out:
        pb = None
        for c in res:                       # first maximum in scan order
            if pb is None or c[0] > pb[0]:
                pb = c
        if pb is not None and (best is None or pb[0] > best[0]):
            best = pb
    return best


def _random_case(rng, num_bin, nan, neg):
    n = int(rng.integers(60, 400))
    col = rng.integers(0, num_bin, n)
    if not nan:
        col = np.minimum(col, num_bin - 1)
    g = rng.integers(-2048, 2049, n) * GRID
    h = rng.integers(256, 2048, n) * GRID
    if neg:
        h = np.where(rng.random(n) < 0.15, -h, h)
    return col, g, h


@pytest.mark.parametrize("seed", range(60))
def test_numerical_scan_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    num_bin = int(rng.choice([2, 3, 5, 9, 17]))
    nan = bool(rng.random() < 0.5)
    neg = bool(seed % 3 == 0)
    offset = int(nan and rng.random() < 0.5)
    col, g, h = _random_case(rng, num_bin, nan, neg)
    if offset:
        col = np.where(rng.random(len(col)) < 0.4, 0, col)
    p = ref.Params(min_data_in_leaf=int(rng.integers(1, 30)), min_sum_hessian_in_leaf=float(rng.choice([1e-3, 5.0])),
                   lambda_l1=float(rng.choice([0.0, 2.0])), lambda_l2=float(rng.choice([0.0, 3.0])), max_delta_step=float(rng.choice([0.0, 0.7])))
    mt = 2 if nan else 0
    hg = np.bincount(col, weights=g, minlength=num_bin)
    hh = np.bincount(col, weights=h, minlength=num_bin)
    sum_h = math.fsum(h)
    if not sum_h > 0:
        pytest.skip("leaf hessian sum must be positive")
    r = ref.find_best_numerical(hg, hh, num_bin, mt, offset, math.fsum(g), sum_h, len(col), p)
    b = _brute(col, g, h, num_bin, mt, offset, p)
    if b is None:
        assert r.gain == ref.NEG_INF and not r.splittable
    else:
        assert r.splittable and r.threshold == b[1] and r.default_left == b[2]
        assert r.win[0] == b[0]


@pytest.mark.parametrize("seed", range(30))
def test_categorical_scan_equals_brute_force(seed):
    """every prefix of the ctr order from either end (and every single bin for one-hot), evaluated by the upstream rules"""
    rng = np.random.default_rng(100 + seed)
    num_bin = int(rng.integers(3, 12))
    n = int(rng.integers(200, 600))
    col = rng.integers(0, num_bin, n)
    g = rng.integers(-2048, 2049, n) * GRID + (col % 3 - 1)
    h = np.ones(n)
    p = ref.Params(min_data_in_leaf=int(rng.integers(1, 20)), max_cat_to_onehot=int(rng.choice([4, 16])), cat_smooth=float(rng.choice([1.0, 10.0])),
                   cat_l2=float(rng.choice([0.0, 10.0])), min_data_per_group=int(rng.choice([1, 30, 100])), max_cat_threshold=int(rng.choice([2, 32])))
    hg = np.bincount(col, weights=g, minlength=num_bin)
    hh = np.bincount(col, weights=h, minlength=num_bin)
    r = ref.find_best_categorical(hg, hh, num_bin, math.fsum(g), math.fsum(h), n, p)
    sum_g, sum_h = math.fsum(g), n + 2 * ref.K_EPS
    shift = ref.leaf_gain(sum_g, sum_h, p, p.lambda_l2) + p.min_gain_to_split
    cnt = {b: int((col == b).sum()) for b in range(num_bin)}
    best = None
    if num_bin <= p.max_cat_to_onehot:
        for b in range(1, num_bin):
            m = col == b
            lg, lh = math.fsum(g[m]), float(m.sum())
            if cnt[b] < p.min_data_in_leaf or lh < p.min_sum_hessian_in_leaf or n - cnt[b] < p.min_data_in_leaf:
                continue
            gain = ref.leaf_gain(sum_g - lg, sum_h - lh - ref.K_EPS, p, p.lambda_l2) + ref.leaf_gain(lg, lh + ref.K_EPS, p, p.lambda_l2)
            if gain > shift and (best is None or gain > best[0]):
                best = (gain, (b,))
    else:
        l2 = p.lambda_l2 + p.cat_l2
        used = sorted((b for b in range(1, num_bin) if cnt[b] >= p.cat_smooth), key=lambda b: (hg[b] / (hh[b] + p.cat_smooth), b))
        k = min(p.max_cat_threshold, (len(used) + 1) // 2)
        for seq in (used, used[::-1]):
            grp_start = 0
            for i in range(min(len(used), k)):
                left = np.isin(col, seq[:i + 1])
                lc = int(left.sum())
                lg, lh = sum(hg[b] for b in seq[:i + 1]), ref.K_EPS
                for b in seq[:i + 1]:
                    lh += hh[b]
                if lc < p.min_data_in_leaf:
                    continue
                if n - lc < p.min_data_in_leaf or n - lc < p.min_data_per_group:
                    break
                if sum(cnt[b] for b in seq[grp_start:i + 1]) < p.min_data_per_group:
                    continue
                grp_start = i + 1
                gain = ref.leaf_gain(lg, lh, p, l2) + ref.leaf_gain(sum_g - lg, sum_h - lh, p, l2)
                if gain > shift and (best is None or gain > best[0]):
                    best = (gain, tuple(sorted(seq[:i + 1])))
    if best is None:
        assert not r.splittable
    else:
        assert r.splittable and r.cat_bins == best[1] and r.win[0] == best[0]


def test_offset_one_forward_pass_starts_from_the_implicit_bin_0():
    """most_freq_bin == 0: bin 0 is not stored; the forward pass starts with left = leaf total - stored bins (threshold 0 first)"""
    p = ref.Params(min_data_in_leaf=1, min_sum_hessian_in_leaf=0.0)
    hg = np.array([999.0, 2.0, 3.0, 4.0])       # bin 0's entry must be ignored
    hh = np.array([999.0, 1.0, 1.0, 1.0])
    sum_g, sum_h, n = -10.0 + 9.0, 4.0, 4        # implicit bin 0: g = -10, h = 1
    r = ref.find_best_numerical(hg, hh, 4, 2, 1, sum_g, sum_h, n, p)
    fwd = [c for c in r.candidates if c[5][0] == "fwd"]
    assert fwd[0][5] == ("fwd", 0) and fwd[0][1] == -10.0 and fwd[0][2] == (sum_h + 2 * ref.K_EPS - ref.K_EPS) - 3.0
    assert r.threshold == 0 and r.default_left is False          # {bin 0} vs {1, 2, NaN}: only the forward pass can separate NaN from bin 0


def test_break_hides_a_better_threshold():
    """negative hessians: the reverse scan breaks on the first threshold whose left side fails min_data_in_leaf and never reaches the
    far better threshold beyond it"""
    p = ref.Params(min_data_in_leaf=20)
    hh = np.array([100.0] * 8 + [-800.0, 1000.0])             # 100 rows per bin; rebuilt counts are exact (sum_h == num_data)
    hg = np.array([-100.0] * 8 + [200.0, 200.0])
    r = ref.find_best_numerical(hg, hh, 10, 0, 0, float(hg.sum()), float(hh.sum()), 1000, p)
    assert not r.splittable and r.candidates == []
    q = ref.Params(min_data_in_leaf=0, min_sum_hessian_in_leaf=-1e30, lambda_l2=1.0)     # nothing breaks: 7|8 is evaluated
    s = ref.find_best_numerical(hg, hh, 10, 0, 0, float(hg.sum()), float(hh.sum()), 1000, q)
    assert s.splittable and ("rev", 7) in [c[5] for c in s.candidates]


def test_min_data_per_group_skips_groups():
    """many-vs-many: a prefix is evaluated only once the bins added since the last evaluated prefix hold min_data_per_group rows"""
    p = ref.Params(min_data_in_leaf=1, cat_smooth=1.0, min_data_per_group=50, max_cat_threshold=8, cat_l2=0.0)
    sizes = [0, 30, 30, 30, 30, 30, 30, 30, 30]
    hh = np.array(sizes, float)
    hg = np.array([0, -60, -50, -40, -30, 30, 40, 50, 60], float)
    r = ref.find_best_categorical(hg, hh, 9, float(hg.sum()), float(hh.sum()), int(hh.sum()), p)
    tags = [c[5] for c in r.candidates]
    assert tags == [("dir+1", 1), ("dir+1", 3), ("dir-1", 1), ("dir-1", 3)]
    assert r.cat_bins in ((1, 2, 3, 4), (5, 6, 7, 8))


def test_max_delta_step_clipping_changes_the_winner():
    p0 = ref.Params(min_data_in_leaf=1, min_sum_hessian_in_leaf=0.0)
    p1 = ref.Params(min_data_in_leaf=1, min_sum_hessian_in_leaf=0.0, max_delta_step=0.5)
    hg = np.array([-20.0, -15.0, -15.0, 50.0])                 # threshold 0 isolates one bin with a large output (20 / 1)
    hh = np.array([1.0, 40.0, 40.0, 40.0])
    a = ref.find_best_numerical(hg, hh, 4, 0, 0, float(hg.sum()), float(hh.sum()), 121, p0)
    b = ref.find_best_numerical(hg, hh, 4, 0, 0, float(hg.sum()), float(hh.sum()), 121, p1)
    assert a.threshold == 0 and b.threshold == 2                # clipped to 0.5, bin 0's output is worth little


def test_undecided_flags_a_near_tie_and_a_count_at_half():
    p = ref.Params(min_data_in_leaf=1)
    bins = np.array([[0], [1], [2], [3]])
    T = tree_ref.grow_tree(bins, np.array([-1.0, 1.0, 1.0, -1.0 - GRID]), np.ones(4), [ref.Feature(0, 4)], p, 2)
    assert ref.undecided(T) == []
    bins2 = np.array([[0], [1]])
    T = tree_ref.grow_tree(bins2, np.array([-1.0, 1.0]), np.array([1.0, 3.0]), [ref.Feature(0, 2)], ref.Params(min_data_in_leaf=0), 2)
    assert any(".5 boundary" in w for w in ref.undecided(T))   # 2 rows, h = 1 and 3: rebuilt counts 0.5 and 1.5
