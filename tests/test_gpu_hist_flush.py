"""K4 flushes its 32-bit shared-memory sub-histogram only when the per-block bin-count bound says a cell could pass 2^14 additions.
These tests compare every cell of Dataset.histogram with NumPy on data where a CTA that skipped a needed flush would return a wrong
histogram:

* one column has nearly every row in one bin, so a CTA's range of a tile puts far more than 2^14 rows into one (column, bin) cell;
* every gradient and hessian has low fixed-point bits 2^18 - 2^11 (the values carry bits down to 2^-22 and quantise at 2^33), so
  the 18-bit low field of a cell wraps its 32-bit accumulator at 16514 additions.  Before comparing, each test checks in NumPy,
  with the kernel's own split of the rows into CTA windows, that the skewed cell of some window takes more additions than that: a
  K4 that flushed only at tile changes and after its last item, or whose bound were too small or read from the wrong tile or rows,
  would fail.  The values are exact in float64, so the comparison is exact.

Cases: the skew over all rows of a column in the second tile, and the skew over the second half of the rows of a column in the first
tile (a window that starts on uniform rows must flush in time); the whole row range, every 2nd row (an index list, bounded through
its first and last row ids), a sparse shuffled row list (sorted before K4) and a list that repeats rows (bounded by row counts)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS = "max_bin=255 is_pre_partition=True num_threads=0 enable_bundle=false"
N, F = 3_000_000, 36                 # two tiles of 32 storage columns (feature f is column f)
SKEWED = {"skew_all": 33, "skew_second_half": 3}
D = 2.0 ** -15 - 2.0 ** -22
G = np.array([2 + D, 3 + D, -(2 + 2.0 ** -22), -(3 + 2.0 ** -22)], dtype=np.float32)     # |g| < 4: quantised at 2^33
H = np.array([2 + D, 3 + D], dtype=np.float32)
LO = 2 ** 18 - 2 ** 11               # low fixed-point field of every value above
K_LO_BITS, K_FLUSH_ROWS, K_STAGE_ROWS = 18, 1 << 14, 512
WRAP = -(-2 ** 32 // LO)             # additions of LO that wrap a 32-bit accumulator: 16514


def _q(v):
    return np.rint(v.astype(np.float64) * 2.0 ** 33).astype(np.int64)


def _data(case):
    rng = np.random.default_rng(11)
    X = rng.integers(0, 200, (N, F), dtype=np.uint8).astype(np.float32)
    rows = np.arange(0 if case == "skew_all" else N // 2, N)
    X[rows[rows % 64 != 0], SKEWED[case]] = 0.0
    return X


@pytest.fixture(scope="module", params=sorted(SKEWED))
def dataset(request, built):
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(_data(request.param), DS)
    yield request.param, ds, ds.get_bins()
    ds.free()


def _rows(kind):
    if kind == "all":
        return None
    if kind == "every_2nd":
        return np.arange(0, N, 2, dtype=np.int32)
    rng = np.random.default_rng(5)
    if kind == "sparse_shuffled":
        r = np.nonzero(rng.random(N) < 0.05)[0].astype(np.int32)
        rng.shuffle(r)
        return r
    return np.repeat(np.arange(0, N, 2, dtype=np.int32), 2)      # "duplicates"


def _sm_count():
    """multiprocessor count of device 0 through the driver API (K4's grid size)"""
    import ctypes
    cu = ctypes.CDLL("libcuda.so.1")
    dev, sms = ctypes.c_int(), ctypes.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(ctypes.byref(sms), 16, dev) == 0      # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return sms.value


def _windows(count, num_tiles, grid):
    """(tile, first, end) list positions of every CTA's items of every tile, split as k4_hist_build_ws splits them"""
    rpi = -(-count * num_tiles // (4 * grid))
    rpi = min(max(-(-rpi // K_STAGE_ROWS) * K_STAGE_ROWS, K_STAGE_ROWS), K_FLUSH_ROWS)
    chunks = -(-count // rpi)
    items = chunks * num_tiles
    for b in range(grid):
        i0, i1 = items * b // grid, items * (b + 1) // grid
        for t in range(num_tiles):
            lo, hi = max(i0, t * chunks), min(i1, (t + 1) * chunks)
            if lo < hi:
                yield t, (lo - t * chunks) * rpi, min((hi - t * chunks) * rpi, count)


@pytest.mark.parametrize("kind", ["all", "every_2nd", "sparse_shuffled", "duplicates"])
def test_histogram_exact_with_skewed_cells(dataset, kind):
    case, ds, bins = dataset
    assert np.all(_q(G) & (2 ** K_LO_BITS - 1) == LO) and np.all(_q(H) & (2 ** K_LO_BITS - 1) == LO)
    assert K_FLUSH_ROWS * LO < 2 ** 32 <= WRAP * LO                   # 2^14 additions fit in the field, WRAP do not
    i = np.arange(N)
    g, h = G[i % 4], H[(i // 4) % 2]
    idx = _rows(kind)
    rows = i if idx is None else np.sort(idx)            # the order K4 sees
    f = SKEWED[case]
    if kind != "sparse_shuffled":                       # a sparse leaf spreads its rows too thin to overflow a window
        grid = _sm_count()                              # one K4 CTA per SM
        most = max(np.bincount(bins[rows[p0:p1], f], minlength=256).max()
                   for t, p0, p1 in _windows(len(rows), 2, grid) if t == f // 32)
        assert most >= WRAP, "no CTA window would overflow without a flush: the test would not see a missing one"
    Hk = ds.histogram(g, h, idx)
    for u in range(F):
        b = bins[rows, u]
        want_g = np.bincount(b, weights=g[rows].astype(np.float64), minlength=256)
        want_h = np.bincount(b, weights=h[rows].astype(np.float64), minlength=256)
        assert np.array_equal(Hk[u, :, 0], want_g), "feature %d: gradient sums differ" % u
        assert np.array_equal(Hk[u, :, 1], want_h), "feature %d: hessian sums differ" % u
