"""The per-node sampling restatement (bynode_ref.py, grown by tree_ref.py) on its own: which draws GetByNode takes and when, the sample size rule, both branches
of Random::Sample, the pool with a tree sample and under interaction constraints, the stream position across trees, the exact integer
form of the selection test the device uses, and the estimators' parameter string."""
import math

import numpy as np
import pytest

import bynode_ref as B
import extra_trees_ref as X3
import interaction_ref as I
import split_scan_ref as ref
import tree_ref


def _data(seed, n=4000, nf=6):
    rng = np.random.default_rng(seed)
    bins = np.stack([rng.integers(0, 12 + 3 * j, n) for j in range(nf)], axis=1)
    y = sum(np.sin(bins[:, j] / (2.0 + j)) * (1.0 - 0.1 * j) for j in range(nf)) + 0.3 * rng.standard_normal(n)
    g = np.round(-y * 1024) / 1024
    h = np.round(rng.uniform(0.5, 1.5, n) * 1024) / 1024
    feats = [ref.Feature(j, 12 + 3 * j) for j in range(nf)]
    return bins, g, h, feats


_SHAPE = ("split_feature", "threshold_bin", "default_left", "left_child", "right_child", "leaf_value", "leaf_count", "split_gain")


def test_bynode_one_draws_nothing():
    bins, g, h, feats = _data(1)
    p = ref.Params(min_data_in_leaf=20)
    s = B.ColSampler(feats, 1.0, 1.0)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 12, sampler=s)
    assert T["draws"] == 0 and s.rnd.x == 2
    plain = tree_ref.grow_tree(bins, g, h, feats, p, 12)
    for k in _SHAPE:
        assert T[k] == plain[k], k
    assert all(samp == set(range(6)) for rnd in T["node_rounds"] for _, samp in rnd)


def test_sample_size_rule():
    assert [B.get_cnt(n, 0.5) for n in (0, 1, 2, 3, 5, 256)] == [0, 1, 2, 2, 3, 128]
    assert [B.get_cnt(n, 0.1) for n in (1, 2, 5, 19, 20, 256)] == [1, 2, 2, 2, 2, 26]
    assert B.get_cnt(7, 1e-9) == 2 and B.get_cnt(7, 0.999) == 7


def test_both_sample_branches():
    """N=5: bynode 0.5 (K=3) takes Floyd's branch (K draws), 0.8 (K=4) the selection branch (N draws); 256 features: 0.5 selection, 0.1
    Floyd's"""
    assert not B.selection_branch(5, B.get_cnt(5, 0.5)) and B.sample_draws(5, 3) == 3
    assert B.selection_branch(5, B.get_cnt(5, 0.8)) and B.sample_draws(5, 4) == 5
    assert B.selection_branch(256, B.get_cnt(256, 0.5)) and not B.selection_branch(256, B.get_cnt(256, 0.1))
    assert B.sample_draws(5, 5) == 0 and B.sample_draws(5, 0) == 0
    for n, k in ((5, 3), (5, 4), (300, 150), (300, 30), (1000, 7)):
        r = B.CountingRandom(17)
        got = r.sample(n, k)
        assert len(got) == k and got == sorted(set(got)) and r.draws == B.sample_draws(n, k)


def test_each_round_samples_from_the_stream():
    """every round that runs draws once per leaf, the smaller leaf first, and the tree's draws are the sum of the samples' draws"""
    bins, g, h, feats = _data(2)
    p = ref.Params(min_data_in_leaf=20)
    s = B.ColSampler(feats, 1.0, 0.5)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 12, sampler=s)
    rounds = T["node_rounds"]
    assert len(rounds) == len(T["rounds"]) and [len(r) for r in rounds] == [len(r) for r in T["rounds"]]
    assert len(rounds[0]) == 1 and all(len(r) == 2 for r in rounds[1:])
    assert all(len(samp) == 3 for r in rounds for _, samp in r)
    assert T["draws"] == sum(len(r) for r in rounds) * B.sample_draws(6, 3)
    # every split feature was sampled by the leaf it split
    allowed = [samp for r in rounds for _, samp in r]
    assert all(any(f in a for a in allowed) for f in T["split_feature"])
    replay = X3.Random(2)
    for r in rounds:
        for _, samp in r:
            assert {i for i in replay.sample(6, 3)} == samp
    assert replay.x == s.rnd.x


def test_tree_sample_is_the_pool():
    """with feature_fraction < 1 the pool is the tree's sample, K comes from its size, and the tree draws interleave with the node draws"""
    bins, g, h, feats = _data(3, nf=8)
    p = ref.Params(min_data_in_leaf=20)
    s = B.ColSampler(feats, 0.6, 0.5)
    replay = X3.Random(2)
    cnt = B.get_cnt(8, 0.6)
    replay.sample(8, cnt)
    for _ in range(3):
        T = tree_ref.grow_tree(bins, g, h, feats, p, 8, sampler=s)
        tree = replay.sample(8, cnt)
        assert set(tree) == set(s.tree)
        for r in T["node_rounds"]:
            for _, samp in r:
                assert samp == {tree[i] for i in replay.sample(cnt, B.get_cnt(cnt, 0.5))}
        assert replay.x == s.rnd.x
    assert cnt == 5 and B.get_cnt(cnt, 0.5) == 3


def test_interaction_filters_the_pool_and_caps_k():
    """a leaf whose allowed pool is smaller than K samples all of it and draws nothing; the root samples K of the allowed features"""
    bins, g, h, feats = _data(4, nf=8)
    p = ref.Params(min_data_in_leaf=20)
    cons = [[0, 1, 2, 3, 4, 5, 6, 7], [0, 5]]
    s = B.ColSampler(feats, 1.0, 0.5)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 12, sampler=s, constraints=cons)
    sets = I.sets_of(cons, 8)
    saw_capped = False
    replay = X3.Random(2)
    for r in T["node_rounds"]:
        for mask, samp in r:
            pool = [f for f in range(8) if sets[f] & mask]
            k = min(B.get_cnt(8, 0.5), len(pool))
            assert samp == {pool[i] for i in replay.sample(len(pool), k)}
            saw_capped |= len(pool) < B.get_cnt(8, 0.5)
    assert replay.x == s.rnd.x
    small = B.ColSampler(feats, 1.0, 0.5)
    small.by_tree()
    assert small.by_node({0, 5}) == {0, 5} and small.rnd.draws == 0
    assert len(small.by_node({0, 1, 2, 5, 7})) == 4 and small.rnd.draws == B.sample_draws(5, 4)
    assert saw_capped or 5 not in T["split_feature"]


def test_stream_after_an_early_stop_and_depth_gated_rounds():
    """a tree that stops (no positive gain) takes no draws after its last round, and rounds that max_depth stops take none either"""
    bins, g, h, feats = _data(5)
    p = ref.Params(min_data_in_leaf=20, min_gain_to_split=40.0)
    s = B.ColSampler(feats, 1.0, 0.5)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 31, sampler=s)
    assert T["num_leaves"] < 31, "the case must stop early"
    assert T["draws"] == sum(len(r) for r in T["node_rounds"]) * B.sample_draws(6, 3)
    assert len(T["node_rounds"]) == T["num_leaves"], "one round per split, plus the round that found no gain"
    p = ref.Params(min_data_in_leaf=20)
    s = B.ColSampler(feats, 1.0, 0.5)
    T = tree_ref.grow_tree(bins, g, h, feats, p, 31, sampler=s, max_depth=2)
    assert T["num_leaves"] == 4
    assert len(T["node_rounds"]) == 2 and T["draws"] == 3 * B.sample_draws(6, 3)


@pytest.mark.parametrize("seed", range(5))
def test_selection_threshold_is_exact(seed):
    """the device's integer test c < k - floor(m (n - i) / 2^15) equals NextFloat() < (k - c) / (n - i) in fp64"""
    rng = np.random.default_rng(seed)
    for _ in range(20000):
        n = int(rng.integers(2, 1 << int(rng.integers(2, 31))))
        i = int(rng.integers(0, n))
        k = int(rng.integers(1, n + 1))
        c = int(rng.integers(0, min(k, i) + 1))
        m = int(rng.integers(0, 32768)) if rng.random() < 0.7 else (32768 * (k - c)) // (n - i) + int(rng.integers(-1, 2))
        m = min(max(m, 0), 32767)
        assert (m / 32768.0 < (k - c) / (n - i)) == (c < k - (m * (n - i) >> 15)), (n, i, k, c, m)


def test_floyd_resolution_without_order():
    """the device resolves Floyd's collisions from two facts (an earlier step drew the same value, or drew an earlier step's r that was
    taken); the result equals the sequential algorithm"""
    for seed in range(200):
        for n, k in ((5, 3), (40, 3), (300, 30), (2000, 150)):
            r = X3.Random(seed)
            vs = [(r._next() & 0x7fffffff) % (n - k + s) for s in range(k)]
            first = {}
            for s, v in enumerate(vs):
                first.setdefault(v, s)
            col = [first[v] < s for s, v in enumerate(vs)]
            changed = True
            while changed:
                changed = False
                for s, v in enumerate(vs):
                    if not col[s] and v >= n - k and col[v - (n - k)]:
                        col[s] = changed = True
            got = sorted(n - k + s if c else v for s, (v, c) in enumerate(zip(vs, col)))
            assert got == X3.Random(seed).sample(n, k), (seed, n, k)


def test_branch_choice_has_no_near_tie():
    """for k < 2^16 not a power of two, k log2(k) is never within 1e-12 relative of an integer n, so k > n / log2(k) is never that close
    to a tie and a log2 that is off by an ulp (about 1e-16 relative) picks the same branch as the host's; powers of two are exact"""
    for k in range(3, 1 << 16):
        if k & (k - 1):
            x = k * math.log2(k)
            assert abs(x - round(x)) > 1e-12 * x, k


def test_estimator_parameter_string():
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    df = Frame({"features": np.zeros((10, 5)), "label": np.zeros(10)})
    assert LightGBMRegressor(featureFractionByNode=0.5).getTrainParams(1, df).to_string().endswith("feature_fraction_bynode=0.5 ")
    assert "bynode" not in LightGBMRegressor().getTrainParams(1, df).to_string()
    assert "bynode" not in LightGBMRegressor(featureFractionByNode=1.0).getTrainParams(1, df).to_string()


@pytest.mark.parametrize("extra", [False, True])
def test_sampler_at_one_grows_the_unsampled_tree(extra):
    """a sampler at feature_fraction_bynode = 1 grows the tree of no sampler, with and without constraints and extra trees"""
    bins, g, h, feats = _data(6)
    p = ref.Params(min_data_in_leaf=20)
    for cons in (None, [[0, 1, 2], [2, 3, 4, 5]]):
        streams = (lambda: X3.Streams(feats, 7)) if extra else (lambda: None)
        T = tree_ref.grow_tree(bins, g, h, feats, p, 12, sampler=B.ColSampler(feats, 1.0, 1.0), constraints=cons, streams=streams())
        want = tree_ref.grow_tree(bins, g, h, feats, p, 12, constraints=cons, streams=streams())
        for k in _SHAPE + ("masks", "branches"):
            assert T[k] == want[k], (cons, k)
