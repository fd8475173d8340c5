"""NumPy restatement of quantised training's discretisation (use_quantized_grad; kernels.cuh k_set_quant_scale, d_quant_uniform,
d_discretize, k_quantize_discrete) and of the packed K4 plane's flush cap (hist_kernel.cuh packed_flush_cap).

Per tree, with B = num_grad_quant_bins: s_g = max|g| / floor(B/2) and s_h = max|h| / B in fp64 from the fp32 maxima (a zero maximum
gives 1; constant hessians keep s_h = 1 and q_h = 1).  v = x / s; with stochastic rounding q = trunc(v + sign(v) u), else v rounded half
away from zero as trunc(v), plus sign(v) when |v - trunc(v)| >= 0.5; q is clamped to [-floor(B/2), floor(B/2)] for g and [-B, B] for h.
u in [0, 1) is the top 53 bits of splitmix64 chained over (data_random_seed, tree index, 2 row + (0 for g, 1 for h))."""
import numpy as np

M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def mix64(z):
    """splitmix64's finaliser on uint64 arrays (wrapping arithmetic)"""
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def uniform(seed, tree, rows, which):
    """the draws u in [0, 1) of rows (rank-local) of one tree; which: 0 for g, 1 for h"""
    z = mix64(np.uint64(seed & 0xFFFFFFFF))
    z = mix64(z ^ np.uint64(tree & 0xFFFFFFFF))
    z = mix64(z ^ (np.uint64(2) * np.asarray(rows, np.uint64) + np.uint64(which)))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def scales(g, h, B, const_hessian=False):
    """(s_g, s_h) from the fp32 maxima"""
    mg = np.float32(np.max(np.abs(np.asarray(g, np.float32)))) if len(g) else np.float32(0)
    s_g = float(mg) / (B // 2) if mg > 0 and np.isfinite(mg) else 1.0
    if const_hessian:
        return s_g, 1.0
    mh = np.float32(np.max(np.abs(np.asarray(h, np.float32)))) if len(h) else np.float32(0)
    return s_g, (float(mh) / B if mh > 0 and np.isfinite(mh) else 1.0)


def discretize(x, s, lim, stochastic, u=None):
    v = np.asarray(x, np.float32).astype(np.float64) / s
    if stochastic:
        q = np.trunc(v + np.sign(v) * u)
    else:
        q = np.trunc(v)
        q = q + np.where(np.abs(v - q) >= 0.5, np.sign(v), 0.0)
    return np.clip(q, -lim, lim).astype(np.int64)


def levels(g, h, B, stochastic, seed, tree, s_g, s_h, rows, const_hessian=False):
    """(q_g, q_h) of some rows at given scales: rows are the rank-local row ids that key the draws (a rank's scales come from the
    maxima over every rank's rows)"""
    qg = discretize(g, s_g, B // 2, stochastic, uniform(seed, tree, rows, 0) if stochastic else None)
    qh = np.ones(len(g), np.int64) if const_hessian else discretize(h, s_h, B, stochastic, uniform(seed, tree, rows, 1) if stochastic else None)
    return qg, qh


def quantize(g, h, B, stochastic, seed, tree, const_hessian=False):
    """(q_g, q_h, s_g, s_h) of one tree's rows on one rank, as k_quantize_discrete writes them"""
    s_g, s_h = scales(g, h, B, const_hessian)
    qg, qh = levels(g, h, B, stochastic, seed, tree, s_g, s_h, np.arange(len(g)), const_hessian)
    return qg, qh, s_g, s_h


def flush_cap(B, count_plane=False):
    """additions a packed cell takes before a 16-bit field could leave [-32767, 32767]"""
    return 32767 // max(B // 2, 1 if count_plane else B)


def pack(qg, qh):
    """the packed 32-bit word of one addition, and the decode of a (wrapped) sum of them"""
    return (np.asarray(qg, np.int64) * 65536 + np.asarray(qh, np.int64)) & 0xFFFFFFFF


def unpack(w):
    w = np.asarray(w, np.int64) & 0xFFFFFFFF
    h = ((w & 0xFFFF) ^ 0x8000) - 0x8000
    w32 = np.where(w >= 2 ** 31, w - 2 ** 32, w)
    return (w32 - h) >> 16, h
