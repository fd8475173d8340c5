"""Position-debiased ranking: lambdarank and rank_xendcg with a `position` field learn one score factor per display position
(csrc/objective.h, kernels.cuh k_position_bias_update) against the NumPy restatement position_bias_ref.py.

- Factors: after every iteration bit-identical to the restatement's update from the engine's own gradients of that iteration (read
  with B200GBM_BoosterGetGradients, which does not move them).
- Gradients: at the factors read back, B200GBM_BoosterGetGradients equals the restatement at the adjusted scores at the bars of
  test_gpu_gradients.py (lambdarank: bit-exact without the normalisation, 2 ulps with it) and test_gpu_xendcg_xentlambda.py.
- Trees: every tree equals tree_ref.grow_tree on the engine's gradients (plain, bagged, GOSS), as test_gpu_goss_renew.py checks.
- Unchanged paths, ranks, reset, refit, the field API, validation sets and the estimator."""
import numpy as np
import pytest

import goss_ref as G
import position_bias_ref as P
import split_scan_ref as ref
import tree_check as tc
import tree_ref
from test_gpu_gradients import _compare as _compare_lr
from xendcg_xentlambda_ref import xendcg_rands

pytestmark = pytest.mark.gpu

DSP = "max_bin=255 min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 min_data_in_leaf=20 verbosity=-1 metric= "


def _data(seed, nq=300, lo=5, hi=40, F=4):
    """features, graded labels from them, query sizes and display positions 0 .. size-1 in each query (shuffled)"""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(lo, hi, nq)
    n = int(sizes.sum())
    X = rng.standard_normal((n, F))
    y = np.clip(np.round(1.2 * X[:, 0] + 0.6 * X[:, 1] + 0.5 * rng.standard_normal(n) + 1.5), 0, 4).astype(np.float32)
    pos = np.concatenate([rng.permutation(c) for c in sizes]).astype(np.int32)
    return X, y, sizes, pos


def _booster(X, y, sizes, params, pos=None, w=None, init=None, reference=None):
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, DSP, reference=reference).set_field("label", y).set_field("group", np.asarray(sizes, np.int32))
    for name, a in (("position", pos), ("weight", w), ("init_score", init)):
        if a is not None:
            ds.set_field(name, a)
    return capi.Booster(ds, BASE + params), ds


def _xe_advance(rands, sizes):
    for q, c in enumerate(sizes):
        if c > 1:
            for _ in range(c):
                rands[q].next_float()


# ------------------------------------------------------------------------------------------------ the field
def test_position_field_round_trip_errors_and_clear(built):
    from mmlspark_b200 import capi
    X, y, sizes, pos = _data(1, nq=20)
    ds = capi.Dataset.from_mat(X, DSP).set_field("label", y)
    try:
        with pytest.raises(capi.LightGBMError, match="Field position is empty"):
            ds.get_field("position")
        odd = pos.copy()
        odd[::3] = -7 - np.arange(len(odd[::3]))
        ds.set_field("position", odd)
        got = ds.get_field("position")
        assert got.dtype == np.int32 and np.array_equal(got, odd)
        with pytest.raises(capi.LightGBMError, match="Length of position"):
            ds.set_field("position", odd[:-1])
        with pytest.raises(capi.LightGBMError, match="Input type error for position"):
            ds.set_field("position", odd.astype(np.float32))
        with pytest.raises(capi.LightGBMError, match="Input type error for position"):
            ds.set_field("position", odd.astype(np.float64))
        assert np.array_equal(ds.get_field("position"), odd)      # a failed set keeps the field
        ds.set_field("position", np.zeros(0, np.int32))
        with pytest.raises(capi.LightGBMError, match="Field position is empty"):
            ds.get_field("position")
    finally:
        ds.free()


# ------------------------------------------------------------------------------------------------ factors, iteration by iteration
FACTOR_CASES = [(o, reg, wt) for o in ("lambdarank", "rank_xendcg") for reg, wt in ((0.0, False), (0.7, False), (0.0, True), (0.3, True))]


@pytest.mark.parametrize("objective, reg, weighted", FACTOR_CASES)
def test_factors_bit_identical_every_iteration(built, objective, reg, weighted):
    X, y, sizes, pos = _data(10 + int(10 * reg) + weighted, nq=400)
    pos = (pos // 2) * 3 - 5          # negative and sparse values
    w = (0.25 + 2.0 * np.random.default_rng(3).random(len(y))).astype(np.float32) if weighted else None
    params = "objective=%s learning_rate=0.2" % objective
    if reg:
        params += " lambdarank_position_bias_regularization=%r" % reg
    b, ds = _booster(X, y, sizes, params, pos=pos, w=w)
    try:
        values, (ids,) = P.position_ids([pos])
        v0, f0 = b.position_bias()
        assert np.array_equal(v0, values) and (f0 == 0).all()
        f = f0
        for it in range(6):
            g, h = b.get_gradients()
            assert np.array_equal(b.position_bias()[1], f), "reading gradients moved the factors"
            want = P.update(f, ids, g, h, 0.2, reg)
            b.update_one_iter()
            v, f = b.position_bias()
            assert np.array_equal(v, values)
            assert np.array_equal(f, want), "iteration %d: factors %r, restatement %r" % (it, f[:5], want[:5])
        assert np.abs(f).max() > 0
    finally:
        b.free(); ds.free()


# ------------------------------------------------------------------------------------------------ gradients at the factors
@pytest.mark.parametrize("truncation, norm, gains_weights", [(1, False, False), (30, False, False), (30, True, False), (30, False, True),
                                                             (10, True, True)])
def test_lambdarank_gradients_at_the_factors(built, truncation, norm, gains_weights):
    X, y, sizes, pos = _data(20 + truncation + 2 * norm, nq=300)
    w, gain, extra = None, None, ""
    if gains_weights:
        w = (0.25 + 2.0 * np.random.default_rng(4).random(len(y))).astype(np.float32)
        w[::11] = 0.0
        gain, extra = [0, 1, 3, 7, 15], " label_gain=0,1,3,7,15"
    params = "objective=lambdarank learning_rate=0.3 lambdarank_truncation_level=%d lambdarank_norm=%s%s" % (truncation, str(norm).lower(), extra)
    b, ds = _booster(X, y, sizes, params, pos=pos, w=w)
    try:
        ids = P.position_ids([pos])[1][0]
        for _ in range(4):
            b.update_one_iter()
        s, (_, f) = b.get_scores(0), b.position_bias()
        assert np.abs(f).max() > 0
        g, h = b.get_gradients()
        rg, rh = P.lambdarank(s, ids, f, y, w, sizes, truncation, norm, label_gain=gain)
        bar = 2 if norm else 0
        _compare_lr(g, rg, bar, "grad"); _compare_lr(h, rh, bar, "hess")
        plain_g, _ = P.lambdarank(s, ids, np.zeros_like(f), y, w, sizes, truncation, norm, label_gain=gain)
        assert not np.array_equal(plain_g, rg)      # the factors matter
        assert np.array_equal(b.position_bias()[1], f)
    finally:
        b.free(); ds.free()


@pytest.mark.parametrize("weighted", [False, True])
def test_xendcg_gradients_at_the_factors(built, weighted):
    from test_gpu_xendcg_xentlambda import _compare as _compare_xe
    X, y, sizes, pos = _data(30 + weighted, nq=300)
    w = (0.5 + np.random.default_rng(5).random(len(y))).astype(np.float32) if weighted else None
    b, ds = _booster(X, y, sizes, "objective=rank_xendcg learning_rate=0.3", pos=pos, w=w)
    try:
        ids = P.position_ids([pos])[1][0]
        iters = 3
        for _ in range(iters):
            b.update_one_iter()
        s, (_, f) = b.get_scores(0), b.position_bias()
        g, h = b.get_gradients()
        rands = xendcg_rands(len(sizes))
        for _ in range(iters):
            _xe_advance(rands, sizes)
        rg, rh, scale = P.xendcg(s, ids, f, y, sizes, rands, w=w)
        _compare_xe(g, rg, "grad", scale=scale); _compare_xe(h, rh, "hess")
    finally:
        b.free(); ds.free()


# ------------------------------------------------------------------------------------------------ trees on the engine's gradients
@pytest.mark.parametrize("case", ["plain", "bagged", "goss"])
def test_trees_match_reference_on_own_gradients(built, case):
    from mmlspark_b200.modeltext import parse_model
    X, y, sizes, pos = _data(40, nq=350, lo=10, hi=40, F=3)
    X = np.round(X * 8) / 8
    n, iters, lr, nl = len(y), 5, 0.3, 8
    params = "objective=lambdarank learning_rate=%r num_leaves=%d boost_from_average=false %s" % (lr, nl, DSP)
    sample = lambda it, g, h: (np.ones(n, bool), g, h)      # noqa: E731
    if case == "bagged":
        params += " bagging_fraction=0.6 bagging_freq=1 bagging_seed=5"
        bags = tc.bags(n, iters, 0.6, 5)
        sample = lambda it, g, h: (bags[it], g, h)      # noqa: E731
    if case == "goss":
        params += " boosting=goss top_rate=0.3 other_rate=0.2"
        st = {"s": [G.seeds(n, 3)]}

        def sample(it, g, h):
            if it < G.warm_up(lr):
                return np.ones(n, bool), g, h
            bag, g2, h2, st["s"] = G.ranks_draw(g[None], h[None], st["s"], [n], 0.3, 0.2)
            return bag, g2[0], h2[0]
    b, ds = _booster(X, y, sizes, params.replace("num_leaves=15 ", ""), pos=pos)
    try:
        grads = []
        for _ in range(iters):
            grads.append(b.get_gradients())
            b.update_one_iter()
        model = b.save_model_to_string()
        assert np.abs(b.position_bias()[1]).max() > 0
    finally:
        b.free(); ds.free()
    feats, bins, ub, b2c = tc.dataset(X, (), 255)
    trees = parse_model(model)["trees"]
    assert len(trees) == iters
    for it in range(iters):
        bag, g, h = sample(it, *grads[it])
        rows = np.nonzero(bag)[0]
        T = tree_ref.grow_tree(bins[rows], tc.quantized(g)[rows], tc.quantized(h)[rows], feats, ref.Params(min_data_in_leaf=20), nl)
        why = ref.undecided(T)
        assert not why, "iteration %d does not discriminate:\n%s" % (it, "\n".join(why[:10]))
        tc.compare_tree(trees[it], T, ub, b2c, lr)


# ------------------------------------------------------------------------------------------------ unchanged paths
def _run(X, y, sizes, params, iters, pos=None, custom=None):
    b, ds = _booster(X, y, sizes, params, pos=pos)
    try:
        for it in range(iters):
            if custom is None:
                b.update_one_iter()
            else:
                b.update_one_iter_custom(*custom)
        return b.save_model_to_string(), b.get_scores(0), b.position_bias()
    finally:
        b.free(); ds.free()


@pytest.mark.parametrize("objective", ["regression", "binary"])
def test_field_is_ignored_by_other_objectives(built, objective):
    X, y, sizes, pos = _data(50)
    y = (y > 1.5).astype(np.float32) if objective == "binary" else y
    params = "objective=%s learning_rate=0.1" % objective
    m0, s0, _ = _run(X, y, sizes, params, 5)
    m1, s1, (v, f) = _run(X, y, sizes, params, 5, pos=pos)
    assert m0 == m1 and np.array_equal(s0, s1) and len(v) == 0 and len(f) == 0


def test_field_is_ignored_with_custom_gradients(built):
    X, y, sizes, pos = _data(51)
    rng = np.random.default_rng(51)
    g, h = rng.standard_normal(len(y)).astype(np.float32), (0.5 + rng.random(len(y))).astype(np.float32)
    m0, s0, _ = _run(X, y, sizes, "objective=lambdarank", 4, custom=(g, h))
    m1, s1, (v, f) = _run(X, y, sizes, "objective=lambdarank", 4, pos=pos, custom=(g, h))
    assert m0 == m1 and np.array_equal(s0, s1) and (f == 0).all()


@pytest.mark.parametrize("objective", ["lambdarank", "rank_xendcg"])
def test_regularisation_without_field_changes_nothing(built, objective):
    X, y, sizes, _ = _data(52)
    m0, s0, (v0, _) = _run(X, y, sizes, "objective=%s" % objective, 5)
    m1, s1, (v1, _) = _run(X, y, sizes, "objective=%s lambdarank_position_bias_regularization=0.5" % objective, 5)
    assert tc.trees(m0) == tc.trees(m1) and np.array_equal(s0, s1) and len(v0) == len(v1) == 0
    assert "position_bias" not in m0
    assert "[lambdarank_position_bias_regularization: 0.5]" in m1
    assert m1.replace("[lambdarank_position_bias_regularization: 0.5]\n", "") == m0


def test_factors_are_not_in_the_model_or_predictions(built):
    X, y, sizes, pos = _data(53)
    m, s, (_, f) = _run(X, y, sizes, "objective=lambdarank", 5, pos=pos)
    assert np.abs(f).max() > 0 and "position" not in m.split("\nparameters:")[0]
    from mmlspark_b200 import capi
    loaded = capi.Booster(model_str=m)
    try:
        np.testing.assert_array_equal(loaded.predict_device(X, capi.PREDICT_RAW_SCORE).reshape(-1), s)      # scores are raw: no factor added
        assert len(loaded.position_bias()[0]) == 0
    finally:
        loaded.free()


# ------------------------------------------------------------------------------------------------ click model
def _click_data(seed, nq, size=20):
    """relevance from features 0 and 1; the logged order puts documents by feature 2, which has nothing to do with relevance; a click
    happens with probability relevance / (1 + position)"""
    rng = np.random.default_rng(seed)
    n = nq * size
    X = rng.standard_normal((n, 4))
    rel = 1.0 / (1.0 + np.exp(-(1.5 * X[:, 0] + X[:, 1] - 0.5)))
    pos = np.concatenate([np.argsort(np.argsort(-X[q * size:(q + 1) * size, 2] + 0.3 * rng.standard_normal(size))) for q in range(nq)]).astype(np.int32)
    clicks = (rng.random(n) < rel / (1.0 + pos)).astype(np.float32)
    return X, clicks, np.full(nq, size), pos, rel


def _ndcg5(score, rel, size):
    grades = np.floor(rel * 5)
    out = []
    for q in range(len(score) // size):
        s, r = score[q * size:(q + 1) * size], grades[q * size:(q + 1) * size]
        disc = 1.0 / np.log2(np.arange(2, 7))
        dcg = ((2 ** r[np.argsort(-s, kind="stable")][:5] - 1) * disc).sum()
        ideal = ((2 ** np.sort(r)[::-1][:5] - 1) * disc).sum()
        out.append(dcg / ideal if ideal > 0 else 1.0)
    return float(np.mean(out))


@pytest.mark.parametrize("objective", ["lambdarank", "rank_xendcg"])
def test_click_model_factors_fall_with_position_and_help_ndcg(built, objective):
    from mmlspark_b200 import capi
    X, clicks, sizes, pos, _ = _click_data(70, 4000)
    Xt, _, _, _, rel_t = _click_data(71, 1000)
    params = "objective=%s learning_rate=0.1 num_leaves=15" % objective
    ndcg, f = {}, None
    for with_pos in (False, True):
        b, ds = _booster(X, clicks, sizes, params, pos=pos if with_pos else None)
        try:
            for _ in range(60):
                b.update_one_iter()
            pred = b.predict_device(Xt, capi.PREDICT_RAW_SCORE).reshape(-1)
            ndcg[with_pos] = _ndcg5(pred, rel_t, 20)
            if with_pos:
                v, f = b.position_bias()
                assert v.tolist() == list(range(20))
        finally:
            b.free(); ds.free()
    print("[position bias] %s NDCG@5 on true relevance: without %.4f, with %.4f; factors %s" % (objective, ndcg[False], ndcg[True], np.round(f, 3)))
    assert f[0] == f.max() and f[0] > f[1] > f[2]
    assert f[:5].mean() > f[5:10].mean() > f[10:].mean()
    assert ndcg[True] > ndcg[False]


# ------------------------------------------------------------------------------------------------ data-parallel ranks
def _without_counts(model):
    """the trees without their leaf and internal counts: the data-parallel learner prints counts estimated from the hessians (as LightGBM's
    does), so only those lines may differ from one rank over all rows"""
    keep = [ln for ln in tc.trees(model).split("\n") if not ln.startswith(("leaf_count=", "internal_count=", "tree_sizes="))]
    return "\n".join(keep)


@pytest.mark.parametrize("R", [2, 3])
def test_ranks_equal_one_rank(built, R):
    from mmlspark_b200 import capi
    X, y, sizes, pos = _data(80 + R, nq=300)
    pos = pos.copy()
    pos[3] = 1000        # present on rank 0 only
    qcut = np.linspace(0, len(sizes), R + 1).astype(int)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    # min_data_in_leaf=0: no split may hinge on an estimated count
    extra = "objective=lambdarank learning_rate=0.2 lambdarank_position_bias_regularization=0.1 min_data_in_leaf=0"
    params = BASE + extra + " tree_learner=data"

    def body(r):
        q0, q1 = qcut[r], qcut[r + 1]
        sl = slice(int(offs[q0]), int(offs[q1]))
        full = capi.Dataset.from_mat(X, DSP)
        ds = capi.Dataset.from_mat(X[sl], DSP, reference=full).set_field("label", y[sl]).set_field("group", np.asarray(sizes[q0:q1], np.int32))
        ds.set_field("position", pos[sl])
        b = capi.Booster(ds, params + " num_machines=%d" % R)
        try:
            fs = []
            for _ in range(5):
                b.update_one_iter()
                fs.append(b.position_bias())
            return b.save_model_to_string(), fs
        finally:
            b.free(); ds.free(); full.free()

    b, ds = _booster(X, y, sizes, extra, pos=pos)
    try:
        want = []
        for _ in range(5):
            b.update_one_iter()
            want.append(b.position_bias())
        want_model = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    res, errs = tc.on_ranks(R, 28400 + 10 * R, body)
    assert not errs, errs
    for model, fs in res:
        assert _without_counts(model) == _without_counts(want_model)
        for (v, f), (wv, wf) in zip(fs, want):
            assert np.array_equal(v, wv) and np.array_equal(f, wf)
    assert 1000 in want[0][0]


def test_ranks_disagreeing_on_the_field_all_fail(built):
    from mmlspark_b200 import capi
    X, y, sizes, pos = _data(85, nq=100)
    half = int(np.cumsum(sizes)[49])

    def body(r):
        sl = slice(0, half) if r == 0 else slice(half, len(y))
        s = sizes[:50] if r == 0 else sizes[50:]
        full = capi.Dataset.from_mat(X, DSP)
        ds = capi.Dataset.from_mat(X[sl], DSP, reference=full).set_field("label", y[sl]).set_field("group", np.asarray(s, np.int32))
        if r == 0:
            ds.set_field("position", pos[sl])
        try:
            capi.Booster(ds, BASE + "objective=lambdarank tree_learner=data num_machines=2").free()
        finally:
            ds.free(); full.free()

    _, errs = tc.on_ranks(2, 28500, body)
    assert sorted(r for r, _ in errs) == [0, 1] and all("position field" in e for _, e in errs), errs


# ------------------------------------------------------------------------------------------------ parameters: reset and checks
def test_reset_changes_only_later_updates(built):
    X, y, sizes, pos = _data(90, nq=300)
    b, ds = _booster(X, y, sizes, "objective=lambdarank learning_rate=0.2", pos=pos)
    try:
        ids = P.position_ids([pos])[1][0]
        f = b.position_bias()[1]
        lr, reg = 0.2, 0.0
        for it in range(6):
            if it == 2:
                b.reset_parameter("lambdarank_position_bias_regularization=2.5")
                reg = 2.5
            if it == 4:
                b.reset_parameter("learning_rate=0.05")
                lr = 0.05
            assert np.array_equal(b.position_bias()[1], f)      # a reset moves nothing by itself
            g, h = b.get_gradients()
            want = P.update(f, ids, g, h, lr, reg)
            b.update_one_iter()
            f = b.position_bias()[1]
            assert np.array_equal(f, want), "iteration %d" % it
        from mmlspark_b200 import capi
        with pytest.raises(capi.LightGBMError, match="lambdarank_position_bias_regularization should be >= 0"):
            b.reset_parameter("lambdarank_position_bias_regularization=-1")
        g, h = b.get_gradients()      # the rejected reset changed nothing: the update still uses 2.5
        want = P.update(f, ids, g, h, lr, reg)
        b.update_one_iter()
        assert np.array_equal(b.position_bias()[1], want)
    finally:
        b.free(); ds.free()


def _rank_dataset(capi, X, y, sizes, pos, r, nq0):
    cut = int(np.sum(sizes[:nq0]))
    sl, s = (slice(0, cut), sizes[:nq0]) if r == 0 else (slice(cut, len(y)), sizes[nq0:])
    full = capi.Dataset.from_mat(X, DSP)
    ds = capi.Dataset.from_mat(X[sl], DSP, reference=full).set_field("label", y[sl]).set_field("group", np.asarray(s, np.int32))
    ds.set_field("position", pos[sl])
    return ds, full


def test_negative_regularisation_fails_at_create_and_reset_on_every_rank(built):
    from mmlspark_b200 import capi
    X, y, sizes, pos = _data(91, nq=40)
    with pytest.raises(capi.LightGBMError, match="lambdarank_position_bias_regularization should be >= 0"):
        _booster(X, y, sizes, "objective=lambdarank lambdarank_position_bias_regularization=-0.5", pos=pos)
    params = BASE + "objective=lambdarank tree_learner=data num_machines=2"

    def create(r):
        ds, full = _rank_dataset(capi, X, y, sizes, pos, r, 20)
        try:
            capi.Booster(ds, params + " lambdarank_position_bias_regularization=-1").free()
        finally:
            ds.free(); full.free()

    _, errs = tc.on_ranks(2, 28600, create)
    assert sorted(r for r, _ in errs) == [0, 1] and all("should be >= 0" in e for _, e in errs), errs

    def reset(r):
        ds, full = _rank_dataset(capi, X, y, sizes, pos, r, 20)
        b = capi.Booster(ds, params)
        try:
            b.update_one_iter()
            try:
                b.reset_parameter("lambdarank_position_bias_regularization=-1")
                err = ""
            except capi.LightGBMError as e:
                err = str(e)
            b.update_one_iter()      # the ranks still train together
            return err, b.position_bias()[1]
        finally:
            b.free(); ds.free(); full.free()

    res, errs = tc.on_ranks(2, 28610, reset)
    assert not errs, errs
    assert all("should be >= 0" in e for e, _ in res) and np.array_equal(res[0][1], res[1][1])


# ------------------------------------------------------------------------------------------------ refit
def test_refit_moves_the_factors_as_the_restatement(built):
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    X, y, sizes, pos = _data(95, nq=300)
    params = "objective=lambdarank learning_rate=0.2 lambdarank_norm=false refit_decay_rate=0.5"
    old, ds0 = _booster(X, y, sizes, params, pos=pos)
    try:
        for _ in range(3):
            old.update_one_iter()
        model = old.save_model_to_string()
    finally:
        old.free(); ds0.free()
    old = capi.Booster(model_str=model)
    try:
        leaf = old.predict_device(X, capi.PREDICT_LEAF_INDEX).astype(np.int32)
        b, ds = _booster(X, y, sizes, params, pos=pos)
        try:
            b.merge(old)
            b.refit(leaf)
            got = b.position_bias()[1]
            refit_trees = parse_model(b.save_model_to_string())["trees"]
        finally:
            b.free(); ds.free()
    finally:
        old.free()
    ids = P.position_ids([pos])[1][0]
    s, f = np.zeros(len(y)), np.zeros(len(got))
    for m in range(3):      # per tree: the gradients at the current scores move the factors, then the refit tree joins the scores
        g, h = P.lambdarank(s, ids, f, y, None, sizes, 30, False)
        f = P.update(f, ids, g, h, 0.2, 0.0)
        s = s + refit_trees[m]["leaf_value"][leaf[:, m]]
    assert np.array_equal(got, f)
    assert np.abs(got).max() > 0


# ------------------------------------------------------------------------------------------------ validation sets
def test_validation_position_changes_no_metric(built):
    from mmlspark_b200 import capi
    X, y, sizes, pos = _data(100, nq=300)
    Xv, yv, sv, pv = _data(101, nq=100)
    evals = []
    for vpos in (None, pv):
        b, ds = _booster(X, y, sizes, "objective=lambdarank metric=ndcg,map eval_at=1,3,5", pos=pos)
        vds = capi.Dataset.from_mat(Xv, DSP, reference=ds).set_field("label", yv).set_field("group", np.asarray(sv, np.int32))
        if vpos is not None:
            vds.set_field("position", vpos)
        try:
            b.add_valid(vds)
            out = []
            for _ in range(4):
                b.update_one_iter()
                out.append((b.get_eval(0), b.get_eval(1)))
            evals.append(out)
        finally:
            b.free(); vds.free(); ds.free()
    for (t0, v0), (t1, v1) in zip(*evals):
        assert np.array_equal(t0, t1) and np.array_equal(v0, v1)


# ------------------------------------------------------------------------------------------------ estimator
def test_ranker_estimator_with_position_col(built):
    from mmlspark_b200.lightgbm import Frame, LightGBMRanker
    from mmlspark_b200.lightgbm.params import TrainParams
    X, y, sizes, pos = _data(110, nq=300)
    q = np.repeat(np.arange(len(sizes)), sizes)
    df = Frame({"features": X, "label": y.astype(np.float64), "query": q, "pos": pos})
    kw = dict(groupCol="query", positionCol="pos", numIterations=8, minDataInLeaf=5, lambdarankPositionBiasRegularization=0.25)
    one = LightGBMRanker(numTasks=1, **kw).fit(df).getNativeModel()
    four = LightGBMRanker(numTasks=4, useSingleDatasetMode=True, defaultListenPort=28700, **kw).fit(df).getNativeModel()
    assert tc.trees(one) == tc.trees(four)
    assert "[lambdarank_position_bias_regularization: 0.25]" in one
    # the C-API run with the estimator's parameter string and the same dataset fields
    est = LightGBMRanker(numTasks=1, **kw)
    tp = TrainParams("ranker", est.params_dict(), 1).to_string()
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0")
    ds.set_field("label", y).set_field("group", np.asarray(sizes, np.int32)).set_field("position", pos)
    b = capi.Booster(ds, tp)
    try:
        for _ in range(8):
            b.update_one_iter()
        assert tc.trees(b.save_model_to_string()) == tc.trees(one)
    finally:
        b.free(); ds.free()
    plain = LightGBMRanker(numTasks=1, groupCol="query", numIterations=8, minDataInLeaf=5).fit(df).getNativeModel()
    assert tc.trees(plain) != tc.trees(one)
