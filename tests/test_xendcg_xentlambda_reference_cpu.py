"""Pins of the NumPy restatement of rank_xendcg and cross_entropy_lambda (tests/xendcg_xentlambda_ref.py) that the GPU tests hold the
kernels to: the random stream against a published sequence, the jump-ahead table k_grad_xendcg reads against sequential draws, when
the per-query states advance, and the cross_entropy_lambda gradient, hessian and init score against the loss they differentiate."""
import numpy as np

import xendcg_xentlambda_ref as R


def test_lcg_is_the_msvc_rand_stream():
    # the same LCG and output bits as the MSVC C runtime's rand() after srand(1): 41, 18467, 6334, 26500, 19169
    r = R.Lcg(1)
    assert [int(r.next_float() * 32768) for _ in range(5)] == [41, 18467, 6334, 26500, 19169]


def test_jump_table_equals_sequential_draws():
    """k_grad_xendcg's table: x_{j+1} = mul[j] x0 + add[j] (mod 2^32), built as Objective::Init builds it, beyond 20,000 draws"""
    m = 25_000
    mul, add = np.zeros(m, np.uint64), np.zeros(m, np.uint64)
    a, c = 1, 0
    for j in range(m):
        a, c = (a * 214013) & 0xFFFFFFFF, (c * 214013 + 2531011) & 0xFFFFFFFF
        mul[j], add[j] = a, c
    for x0 in (5, 7, 123456, 0xFFFFFFFF):
        r = R.Lcg(x0)
        seq = np.array([r.next_float() for _ in range(m)], np.float32)
        x = (mul * np.uint64(x0) + add) & np.uint64(0xFFFFFFFF)
        jumped = (((x >> np.uint64(16)) & np.uint64(0x7FFF)).astype(np.float32) / np.float32(32768.0))
        assert np.array_equal(seq, jumped)
        assert r.x == int(x[-1])


def _queries(rng, sizes):
    n = int(np.sum(sizes))
    return 3.0 * rng.standard_normal(n), rng.integers(0, 5, n).astype(np.float32)


def test_states_advance_by_query_size_and_single_documents_draw_nothing():
    rng = np.random.default_rng(3)
    sizes = np.array([1, 2, 1, 100, 7, 1, 3000])
    s, y = _queries(rng, sizes)
    rands = R.xendcg_rands(len(sizes), seed=5)
    for it in range(3):
        g, h, _ = R.xendcg_gradients(s, y, sizes, rands)
        for q, cnt in enumerate(sizes):
            fresh = R.Lcg(5 + q)
            for _ in range((it + 1) * cnt if cnt > 1 else 0):
                fresh.next_float()
            assert rands[q].x == fresh.x, "query %d after %d iterations" % (q, it + 1)
        single = np.repeat(sizes == 1, sizes)
        assert not g[single].any() and not h[single].any()


def test_xendcg_iterations_differ_and_seeds_differ():
    rng = np.random.default_rng(4)
    sizes = np.array([20, 30, 40])
    s, y = _queries(rng, sizes)
    rands = R.xendcg_rands(3, seed=5)
    g1, _, _ = R.xendcg_gradients(s, y, sizes, rands)
    g2, h2, _ = R.xendcg_gradients(s, y, sizes, rands)
    g7, h7, _ = R.xendcg_gradients(s, y, sizes, R.xendcg_rands(3, seed=7))
    assert not np.array_equal(g1, g2) and not np.array_equal(g1, g7)
    assert np.array_equal(h2, h7)                     # the hessian rho (1 - rho) draws nothing
    # the first-order term is the softmax cross-entropy gradient rho - phi / sum(phi): it sums to zero over a query, and the
    # higher-order terms are small against it for these scores
    assert abs(float(np.sum(g1[:20], dtype=np.float64))) < 1e-2


def _xentlambda_loss(s, y, w):
    z = 1.0 - np.exp(-w * np.log1p(np.exp(s)))
    return -(y * np.log(z) + (1.0 - y) * np.log(1.0 - z))


def test_xentlambda_gradient_is_the_derivative_of_its_loss():
    rng = np.random.default_rng(5)
    n = 2000
    s = rng.uniform(-4.0, 4.0, n)
    y = rng.random(n).astype(np.float32)
    w = (0.2 + 3.0 * rng.random(n)).astype(np.float32)
    g, h = R.xentlambda_gradients(s, y, w)
    y64, w64, e = y.astype(np.float64), w.astype(np.float64), 1e-4
    fd_g = (_xentlambda_loss(s + e, y64, w64) - _xentlambda_loss(s - e, y64, w64)) / (2 * e)
    L = [_xentlambda_loss(s + k * 1e-3, y64, w64) for k in (-2, -1, 0, 1, 2)]      # five-point second difference
    fd_h = (-L[0] + 16 * L[1] - 30 * L[2] + 16 * L[3] - L[4]) / (12 * 1e-6)
    np.testing.assert_allclose(g, fd_g, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(h, fd_h, rtol=1e-3, atol=1e-3)
    # unit weights: the link is the plain sigmoid, and the weighted formulas reduce to the unweighted ones
    g1, h1 = R.xentlambda_gradients(s, y, np.ones(n, np.float32))
    g0, h0 = R.xentlambda_gradients(s, y)
    np.testing.assert_allclose(g1, g0, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(h1, h0, rtol=1e-5, atol=1e-6)


def test_xentlambda_init_score_inverts_the_output_transform():
    rng = np.random.default_rng(6)
    y = rng.random(1000).astype(np.float32)
    w = (0.5 + rng.random(1000)).astype(np.float32)
    havg = float((y.astype(np.float64) * w).sum() / w.astype(np.float64).sum())
    np.testing.assert_allclose(np.log1p(np.exp(R.xentlambda_init_score(y, w))), havg, rtol=1e-12)


def test_metrics_at_known_points():
    y = np.array([0.0, 0.25, 0.5, 1.0], np.float32)
    p = y.astype(np.float64)
    assert abs(R.metric_kldiv(p, y)) < 1e-12                     # KL(y || y) = 0
    np.testing.assert_allclose(R.metric_kldiv(np.full(4, 0.5), y), np.mean(np.log(2.0) + R.yent_loss(y.astype(np.float64))), rtol=1e-12)
    # cross_entropy_lambda: p = -log(1 - q) makes 1 - exp(-p) = q, and the weight scales p
    q = np.array([0.1, 0.3, 0.6, 0.9])
    np.testing.assert_allclose(R.metric_xentlambda(-np.log1p(-q), y), np.mean(R.xent_loss(y.astype(np.float64), q)), rtol=1e-12)
    w = np.full(4, 2.0, np.float32)
    np.testing.assert_allclose(R.metric_xentlambda(-np.log1p(-q) / 2, y, w), np.mean(R.xent_loss(y.astype(np.float64), q)), rtol=1e-12)
