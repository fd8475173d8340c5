"""Dataset construction checks shared by the three ingestion paths (LGBM_DatasetCreateFromMat, LGBM_DatasetCreateFromCSR and
LGBM_DatasetCreateFromSampledColumn + LGBM_DatasetPushRows): the same bin parameters are rejected with the same message on every
path that finds bins, a reference dataset with another column count is rejected, and a rejected row push leaves the dataset usable."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BASE_PARAMS = "is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
DS_PARAMS = "max_bin=255 " + BASE_PARAMS


def _matrix(rng, n, F):
    X = rng.standard_normal((n, F))
    X[:, 1] = np.where(rng.random(n) < 0.5, 0.0, X[:, 1])
    return X


def _csr(X):
    stored = X != 0
    indptr = np.concatenate([[0], np.cumsum(stored.sum(axis=1))]).astype(np.int32)
    return indptr, np.nonzero(stored)[1].astype(np.int32), X[stored]


@pytest.mark.parametrize("bad,message", [
    ("max_bin=255 zero_as_missing=true", "zero_as_missing=true is not supported by this build"),
    ("max_bin=1", "max_bin should be >= 2"),
    ("max_bin=16384", "max_bin >= 16384 is not supported"),
], ids=["zero_as_missing", "max_bin_1", "max_bin_16384"])
def test_bin_parameters_rejected_on_every_path(built, bad, message):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(11)
    n, F = 3000, 6
    X = _matrix(rng, n, F)
    indptr, indices, data = _csr(X)
    params = BASE_PARAMS + " " + bad
    paths = {
        "from_mat": lambda: capi.Dataset.from_mat(X, params),
        "from_csr": lambda: capi.Dataset.from_csr(indptr, indices, data, F, params),
        "from_sampled_columns": lambda: capi.Dataset.from_sampled_columns(X[capi.sample_indices(n, 200000, 1)], n, params),
    }
    for name, create in paths.items():
        with pytest.raises(capi.LightGBMError) as e:
            create()
        assert str(e.value) == message, name


def test_reference_with_other_column_count_rejected(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(12)
    X = _matrix(rng, 3000, 6)
    ds = capi.Dataset.from_mat(X, DS_PARAMS)
    Xv = _matrix(rng, 500, 7)
    with pytest.raises(capi.LightGBMError, match="different number of features"):
        capi.Dataset.from_mat(Xv, DS_PARAMS, reference=ds)
    with pytest.raises(capi.LightGBMError, match="different number of features"):
        capi.Dataset.from_csr(*_csr(Xv), 7, DS_PARAMS, reference=ds)
    ds.free()


def test_rejected_push_rows_leaves_dataset_usable(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(13)
    n, F = 5000, 6
    X = _matrix(rng, n, F)
    sample = X[capi.sample_indices(n, 200000, 1)]
    ds = capi.Dataset.from_sampled_columns(sample, n, DS_PARAMS)
    assert ds.ingest_ms() == 0.0
    for start_row in (-1, 1, n):
        with pytest.raises(capi.LightGBMError, match="row block out of range"):
            ds.push_rows(X, start_row)
    ds.push_rows(X, 0)
    assert ds.ingest_ms() > 0.0
    fresh = capi.Dataset.from_sampled_columns(sample, n, DS_PARAMS)
    fresh.push_rows(X, 0)
    for f in range(F):
        assert ds.feature_info(f) == fresh.feature_info(f)
    assert np.array_equal(ds.get_bins(), fresh.get_bins())
    ds.free(); fresh.free()
