"""The extra_trees restatement (extra_trees_ref.py) on its own: the streams' first draws, the filtered scans against a brute-force
evaluation of the drawn candidate, and the draw order of a grown tree."""
import numpy as np

import extra_trees_ref as X3
import split_scan_ref as ref
import tree_ref


def test_stream_matches_a_published_sequence():
    """LightGBM's Random is the LCG of the Microsoft C runtime's rand(): x = 214013 x + 2531011, rand() = (x >> 16) & 0x7fff.  After
    srand(1) that rand() is known to return 41, 18467, 6334, 26500, 19169, 15724, 11478, 29358, 26962, 24464; NextFloat reads the same
    15 bits, and NextInt the low 31 bits of the same states."""
    r = X3.Random(1)
    assert [int(r.next_float() * 32768) for _ in range(10)] == [41, 18467, 6334, 26500, 19169, 15724, 11478, 29358, 26962, 24464]
    a, b = X3.Random(1), X3.Random(1)
    for _ in range(10):
        hi = int(a.next_float() * 32768)
        lo31 = b.next_int(0, 2 ** 31)
        assert (lo31 >> 16) & 0x7fff == hi


def _hist(rng, num_bin, n=3000, nan=False):
    col = rng.integers(0, num_bin, n)
    g = np.round(rng.standard_normal(n) * 1024) / 1024 + (col > num_bin // 2) * 0.5
    h = rng.integers(512, 1537, n) / 1024
    return col, g, h


def test_numerical_scan_evaluates_only_the_drawn_threshold():
    rng = np.random.default_rng(1)
    p = ref.Params(min_data_in_leaf=20)
    hits = 0
    for num_bin, missing in ((20, 0), (20, 2), (9, 2), (60, 0)):
        col, g, h = _hist(rng, num_bin)
        hg = np.bincount(col, weights=g, minlength=num_bin)
        hh = np.bincount(col, weights=h, minlength=num_bin)
        full = ref.find_best_numerical(hg, hh, num_bin, missing, 0, g.sum(), h.sum(), len(g), p)
        for t in range(num_bin - 2):
            r = X3.find_best_numerical(hg, hh, num_bin, missing, 0, g.sum(), h.sum(), len(g), p, 0, t)
            mine = [c for c in full.candidates if c[5][1] == t and c[0] > full.shift]
            assert r.splittable == bool(mine)
            if mine:
                best = max(mine, key=lambda c: c[0])
                assert r.threshold == t and r.gain == best[0] - full.shift
                assert r.default_left == (best[5][0] == "rev")
                if full.win is not None and full.win[5] == best[5]:      # the drawn candidate is the full scan's winner
                    assert (r.left_count, r.left_g, r.left_h) == (full.left_count, full.left_g, full.left_h)
                    hits += 1
    assert hits > 0


def test_categorical_scans_evaluate_only_the_drawn_candidate():
    rng = np.random.default_rng(2)
    p = ref.Params(min_data_in_leaf=10, min_data_per_group=10, cat_smooth=5)
    for num_bin in (4, 30):
        col, g, h = _hist(rng, num_bin)
        hg = np.bincount(col, weights=g, minlength=num_bin)
        hh = np.bincount(col, weights=h, minlength=num_bin)
        rng_n = X3.categorical_range(hh, num_bin, h.sum(), len(g), p)
        assert rng_n > 0
        for t in range(rng_n):
            r = X3.find_best_categorical(hg, hh, num_bin, g.sum(), h.sum(), len(g), p, 0, t)
            if r.splittable:
                if num_bin <= p.max_cat_to_onehot:
                    assert r.cat_bins == (t + 1,)
                else:
                    assert len(r.cat_bins) == t + 1
                assert r.gain + r.shift in [c[0] for c in r.candidates]


def test_grow_tree_draw_order_and_seeds():
    """trees differ by seed, repeat with the same seed, and without streams the root splits where the full scans put it; the root
    split's threshold is the first draw of its feature's stream"""
    rng = np.random.default_rng(3)
    n = 4000
    bins = np.stack([rng.integers(0, 40, n), rng.integers(0, 25, n), rng.integers(0, 4, n)], axis=1)
    g = np.round((bins[:, 0] * 0.05 - (bins[:, 2] == 2) + rng.standard_normal(n)) * 1024) / 1024
    h = np.ones(n)
    feats = [ref.Feature(0, 40), ref.Feature(1, 25), ref.Feature(2, 4, is_cat=True)]
    p = ref.Params(min_data_in_leaf=20)
    def grow(seed):
        return tree_ref.grow_tree(bins, g, h, feats, p, 8, streams=None if seed is None else X3.Streams(feats, seed))

    T6 = grow(6)
    assert T6["split_feature"] == grow(6)["split_feature"]
    root = ref.best_of_leaf(tree_ref.scan_leaf(bins, g, h, np.arange(n), g.sum(), h.sum(), n, feats, {0: True, 1: True, 2: True}, p))
    plain = grow(None)
    assert (plain["split_feature"][0], plain["threshold_bin"][0]) == (root.feature, root.threshold)
    shapes = {tuple(zip(grow(s)["split_feature"], grow(s)["threshold_bin"])) for s in range(6, 12)}
    assert len(shapes) > 1
    f = T6["split_feature"][0]
    if f != 2:
        i = [x.real_index for x in feats].index(f)
        assert T6["threshold_bin"][0] == X3.Random(6 + i).next_int(0, feats[i].num_bin - 2)


def test_feature_fraction_sets():
    sets = X3.feature_fraction_sets(10, 0.5, 2, 4)
    assert all(len(s) == 5 for s in sets) and len({tuple(sorted(s)) for s in sets}) > 1
    assert X3.feature_fraction_sets(10, 1.0, 2, 2) == [set(range(10))] * 2
