"""The NumPy restatement of quantised training (quant_ref): the levels' bounds, stochastic rounding's mean and key determinism, round half
away from zero, the packed word's decode and the flush cap C(B), and the estimators' parameter string."""
import numpy as np
import pytest

import quant_ref as Q


@pytest.mark.parametrize("B", [2, 3, 4, 16, 63])
@pytest.mark.parametrize("stochastic", [True, False])
def test_levels_within_bounds(B, stochastic):
    rng = np.random.default_rng(B)
    g = rng.standard_normal(20000).astype(np.float32)
    h = (rng.standard_normal(20000) * 3).astype(np.float32)      # negative hessians too: the rule is symmetric
    qg, qh, s_g, s_h = Q.quantize(g, h, B, stochastic, 1, 7)
    assert np.abs(qg).max() == B // 2 and np.abs(qh).max() == B      # the maxima reach the limits
    assert qg.min() < 0 < qg.max() and qh.min() < 0 < qh.max()
    assert s_g == float(np.abs(g).max()) / (B // 2) and s_h == float(np.abs(h).max()) / B
    # a level is within one step of the value
    assert np.all(np.abs(qg - g / s_g) < 1) and np.all(np.abs(qh - h / s_h) < 1)


def test_zero_column_gives_scale_one_and_zero_levels():
    z = np.zeros(100, np.float32)
    qg, qh, s_g, s_h = Q.quantize(z, z, 4, True, 1, 0)
    assert (s_g, s_h) == (1.0, 1.0) and not qg.any() and not qh.any()


def test_constant_hessian_is_the_count_plane():
    g = np.linspace(-1, 1, 101, dtype=np.float32)
    qg, qh, s_g, s_h = Q.quantize(g, None, 4, False, 1, 0, const_hessian=True)
    assert s_h == 1.0 and np.all(qh == 1)


@pytest.mark.parametrize("x", [0.3, -0.3, 1.7, -1.25])
def test_stochastic_rounding_is_unbiased(x):
    """the mean of q s over many rows of the same value is the value: within 5 standard errors of a Bernoulli level choice"""
    n = 200000
    g = np.full(n, x, np.float32)
    g[0] = 2.0                                                      # max |g| = 2: s_g = 1 at B = 4
    qg, _, s_g, _ = Q.quantize(g, np.ones(n, np.float32), 4, True, 3, 11)
    frac = abs(float(np.float32(x))) % 1.0
    se = np.sqrt(frac * (1 - frac) / (n - 1))
    assert abs(qg[1:].mean() * s_g - float(np.float32(x))) < 5 * se
    assert set(np.unique(qg[1:])) == {np.trunc(x), np.trunc(x) + np.sign(x)}


def test_draws_are_determined_by_their_key():
    rows = np.arange(1000)
    u = Q.uniform(1, 5, rows, 0)
    assert np.array_equal(u, Q.uniform(1, 5, rows, 0))
    assert np.array_equal(u[500:], Q.uniform(1, 5, rows[500:], 0))      # a row's draw does not depend on the others
    for other in (Q.uniform(2, 5, rows, 0), Q.uniform(1, 6, rows, 0), Q.uniform(1, 5, rows, 1)):
        assert np.mean(u == other) < 0.01
    assert u.min() >= 0.0 and u.max() < 1.0 and abs(u.mean() - 0.5) < 0.05


def test_round_half_away_from_zero():
    # s_g = 1 at B = 4 (max |g| = 2): v = g exactly
    g = np.array([2.0, 0.5, -0.5, 1.5, -1.5, 0.49999997, -0.49999997, 0.0], np.float32)
    qg, _, s_g, _ = Q.quantize(g, np.ones_like(g), 4, False, 1, 0)
    assert s_g == 1.0
    assert qg.tolist() == [2, 1, -1, 2, -2, 0, 0, 0]


@pytest.mark.parametrize("B,count_plane,C", [(2, False, 16383), (4, False, 8191), (4, True, 16383), (16, False, 2047), (63, False, 520),
                                             (63, True, 1057)])
def test_flush_cap(B, count_plane, C):
    assert Q.flush_cap(B, count_plane) == C
    assert C >= 512          # K4's row chunks are whole 512-row stages
    lim_g, lim_h = B // 2, (1 if count_plane else B)
    # C additions at the field limits, either sign, decode exactly; the sums of C + 1 can leave a field
    for sg in (1, -1):
        for sh in (1, -1):
            w = (Q.pack(sg * lim_g, sh * lim_h) * C) & 0xFFFFFFFF
            assert Q.unpack(w) == (sg * lim_g * C, sh * lim_h * C)
    assert max(lim_g, lim_h) * (C + 1) > 32767


def test_packed_sums_decode():
    rng = np.random.default_rng(0)
    B = 16
    qg, qh = rng.integers(-8, 9, 2047), rng.integers(-16, 17, 2047)
    w = int(np.sum(Q.pack(qg, qh))) & 0xFFFFFFFF
    assert Q.unpack(w) == (qg.sum(), qh.sum())
    assert Q.flush_cap(B) == 2047


def test_estimator_parameter_string():
    from mmlspark_b200.lightgbm import Frame, LightGBMClassifier
    df = Frame({"features": np.zeros((10, 5)), "label": np.zeros(10)})
    s = LightGBMClassifier(useQuantizedGrad=True, numGradQuantBins=8).getTrainParams(1, df).to_string()
    assert "use_quantized_grad=true num_grad_quant_bins=8 quant_train_renew_leaf=false stochastic_rounding=true " in s
    default = LightGBMClassifier().getTrainParams(1, df).to_string()
    for key in ("use_quantized_grad", "num_grad_quant_bins", "quant_train_renew_leaf", "stochastic_rounding"):
        assert key not in default
    assert LightGBMClassifier(numGradQuantBins=8).getTrainParams(1, df).to_string() == default
