"""Objective checks of LGBM_BoosterCreate: the configurations and training labels each objective rejects (with their messages), the
objective string of the model header and whether the booster trains with a constant hessian."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=7 learning_rate=0.1 min_data_in_leaf=20 verbosity=-1 "
N, F = 2000, 5


def _labels(objective, rng, x):
    if objective == "binary":
        return (x > 0).astype(np.float32)
    if objective in ("multiclass", "multiclassova"):
        return np.digitize(x, [-0.5, 0.5]).astype(np.float32)
    if objective == "cross_entropy":
        return (1.0 / (1.0 + np.exp(-x))).astype(np.float32)
    if objective in ("poisson", "gamma", "tweedie"):
        return np.exp(0.5 * x).astype(np.float32)
    if objective == "lambdarank":
        return np.clip(np.round(x + 1.5), 0, 4).astype(np.float32)
    return (2.0 * x + 0.1 * rng.standard_normal(len(x))).astype(np.float32)


def _dataset(objective, seed, label=None, weight=None, group=True):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, F))
    y = _labels(objective, rng, X[:, 0] + 0.5 * X[:, 1]) if label is None else label(X)
    ds = capi.Dataset.from_mat(X, DS_PARAMS)
    ds.set_field("label", y.astype(np.float32))
    if weight is not None:
        ds.set_field("weight", weight(rng).astype(np.float32))
    if objective == "lambdarank" and group:
        ds.set_field("group", np.full(N // 20, 20, dtype=np.int32))
    return ds


REJECTIONS = {
    "quantile_alpha_0": ("quantile", "alpha=0", {}, "Check failed: alpha_ > 0 && alpha_ < 1"),
    "quantile_alpha_1": ("quantile", "alpha=1", {}, "Check failed: alpha_ > 0 && alpha_ < 1"),
    "multiclass_num_class_1": ("multiclass", "num_class=1", {},
                               "Number of classes should be specified and greater than 1 for multiclass training"),
    "multiclassova_num_class_1": ("multiclassova", "num_class=1", {},
                                  "Number of classes should be specified and greater than 1 for multiclass training"),
    "multiclass_label_num_class": ("multiclass", "num_class=3", {"label": lambda X: np.where(X[:, 0] > 1.0, 3, 0)},
                                   "Label must be in [0, 3), but found 3 in label"),
    "multiclassova_label_negative": ("multiclassova", "num_class=3", {"label": lambda X: np.where(X[:, 0] > 1.0, -1, 1)},
                                     "Label must be in [0, 3), but found -1 in label"),
    "poisson_label_negative": ("poisson", "", {"label": lambda X: X[:, 0]}, "[poisson]: at least one target label is negative"),
    "gamma_label_negative": ("gamma", "", {"label": lambda X: X[:, 0]}, "[gamma]: at least one target label is negative"),
    "tweedie_label_negative": ("tweedie", "", {"label": lambda X: X[:, 0]}, "[tweedie]: at least one target label is negative"),
    "cross_entropy_label_1_5": ("cross_entropy", "", {"label": lambda X: np.where(X[:, 0] > 1.0, 1.5, 0.5)},
                                "[cross_entropy]: does not tolerate label 1.500000 outside [0, 1]"),
    "cross_entropy_weight_negative": ("cross_entropy", "", {"weight": lambda rng: np.where(rng.random(N) < 0.01, -1.0, 1.0)},
                                      "[cross_entropy]: at least one weight is negative"),
    "cross_entropy_weights_zero": ("cross_entropy", "", {"weight": lambda rng: np.zeros(N)}, "[cross_entropy]: sum of weights is zero"),
    "lambdarank_no_group": ("lambdarank", "", {"group": False}, "Ranking tasks require query information"),
    "lambdarank_label_beyond_gain": ("lambdarank", "label_gain=0,1,3", {}, "Label excel the max range 3 for lambdarank"),
    "lambdarank_truncation_0": ("lambdarank", "lambdarank_truncation_level=0", {}, "lambdarank_truncation_level should be in [1, 180]"),
}


@pytest.mark.parametrize("case", list(REJECTIONS))
def test_objective_rejects(built, case):
    from mmlspark_b200 import capi
    objective, extra, fields, message = REJECTIONS[case]
    ds = _dataset(objective, 31, **fields)
    with pytest.raises(capi.LightGBMError) as e:
        capi.Booster(ds, BASE + "objective=%s %s" % (objective, extra))
    assert message in str(e.value)
    ds.free()


HEADERS = {
    "regression": ("", "regression"),
    "huber": ("", "huber"),
    "fair": ("", "fair"),
    "poisson": ("", "poisson"),
    "gamma": ("", "gamma"),
    "tweedie": ("", "tweedie"),
    "regression_l1": ("", "regression_l1"),
    "quantile": ("alpha=0.3", "quantile"),
    "mape": ("", "mape"),
    "binary": ("", "binary sigmoid:1"),
    "multiclass": ("num_class=3", "multiclass num_class:3"),
    "multiclassova": ("num_class=3", "multiclassova num_class:3 sigmoid:1"),
    "cross_entropy": ("", "cross_entropy"),
    "lambdarank": ("", "lambdarank"),
}
CONSTANT_HESSIAN = ("regression", "regression_l1", "quantile", "mape")


@pytest.mark.parametrize("objective", list(HEADERS))
def test_objective_header_and_constant_hessian(built, objective):
    from mmlspark_b200 import capi
    extra, header = HEADERS[objective]
    ds = _dataset(objective, 32)
    b = capi.Booster(ds, BASE + "objective=%s %s" % (objective, extra))
    b.update_one_iter()
    lines = b.save_model_to_string().splitlines()
    assert [ln for ln in lines if ln.startswith("objective=")] == ["objective=" + header]
    assert b.get_info()["constant_hessian"] == (objective in CONSTANT_HESSIAN)
    b.free(); ds.free()


@pytest.mark.parametrize("objective", CONSTANT_HESSIAN)
@pytest.mark.parametrize("variant", ["weighted", "goss"])
def test_weights_and_goss_make_the_hessian_vary(built, objective, variant):
    from mmlspark_b200 import capi
    weight = (lambda rng: 0.5 + rng.random(N)) if variant == "weighted" else None
    ds = _dataset(objective, 33, weight=weight)
    boosting = "boosting_type=goss" if variant == "goss" else ""
    b = capi.Booster(ds, BASE + "objective=%s %s" % (objective, boosting))
    b.update_one_iter()
    assert not b.get_info()["constant_hessian"]
    b.free(); ds.free()
