"""C-ABI checks that need no GPU: the library loads, exports every symbol include/*.h declares, follows the
reference's error convention, and its host-side parts (model text, single-row predictor, TreeSHAP, ChunkedArray)
behave like the reference's tests expect.  Compute entries must FAIL loudly without a GPU (no CPU fallback)."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "oracle_golden.json")))


@pytest.fixture(scope="module")
def capi(built):
    from mmlspark_b200 import capi
    capi.load()
    return capi


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "b200gbm_c_api.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b((?:LGBM|B200GBM)_[A-Za-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol(capi):
    lib = capi.load()
    names = _declared_symbols()
    assert len(names) >= 60
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, "declared in include/b200gbm_c_api.h but not exported: %s" % missing
    # the subset MMLSpark calls through SWIG (SURVEY.md §8b)
    for n in ["LGBM_GetLastError", "LGBM_NetworkInit", "LGBM_NetworkFree", "LGBM_DatasetCreateFromMat", "LGBM_DatasetCreateFromCSR",
              "LGBM_DatasetSetField", "LGBM_DatasetGetField", "LGBM_DatasetGetNumData", "LGBM_DatasetGetNumFeature",
              "LGBM_DatasetSetFeatureNames", "LGBM_DatasetFree", "LGBM_BoosterCreate", "LGBM_BoosterLoadModelFromString",
              "LGBM_BoosterMerge", "LGBM_BoosterAddValidData", "LGBM_BoosterFree", "LGBM_BoosterUpdateOneIter",
              "LGBM_BoosterUpdateOneIterCustom", "LGBM_BoosterResetParameter", "LGBM_BoosterGetEvalNames", "LGBM_BoosterGetEval",
              "LGBM_BoosterGetPredict", "LGBM_BoosterGetNumClasses", "LGBM_BoosterNumModelPerIteration", "LGBM_BoosterNumberOfTotalModel",
              "LGBM_BoosterGetNumFeature", "LGBM_BoosterFeatureImportance", "LGBM_BoosterSaveModelToString", "LGBM_BoosterDumpModel",
              "LGBM_BoosterPredictForMatSingle", "LGBM_BoosterPredictForCSRSingle"]:
        assert n in names


def _has_gpu():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout.count("GPU ") > 0
    except Exception:
        return False


def test_compute_entries_fail_loudly_without_gpu(capi):
    if _has_gpu():
        pytest.skip("a GPU is present")
    with pytest.raises(capi.LightGBMError) as e:
        capi.Dataset.from_mat(np.zeros((10, 3)), "max_bin=255")
    assert "no CUDA device" in str(e.value) and "no CPU fallback" in str(e.value)
    h = C.c_void_p()
    rc = capi.load().LGBM_DatasetCreateFromMat(None, 1, 10, 3, 1, b"", None, C.byref(h))
    assert rc == -1 and capi.load().LGBM_GetLastError()          # -1 + message convention (LightGBMUtils.scala:22-27)


def test_error_convention_bad_model_string(capi):
    with pytest.raises(capi.LightGBMError):
        capi.Booster(model_str="this is not a model")
    with pytest.raises(capi.LightGBMError) as e:
        capi.Booster(model_str="tree\nversion=v3\nnum_class=1\n")
    assert "label_index" in str(e.value) or "specify" in str(e.value)


@pytest.mark.parametrize("name", ["regression", "binary", "multiclass"])
def test_model_text_roundtrip_and_single_row_predict(capi, name):
    """verifySaveBooster (VerifyLightGBMClassifier.scala:712-755): load -> save -> load gives identical predictions; the
    native predictor agrees with the oracle's predictions stored beside the golden model."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "golden", "make_golden.py"))
    mg = importlib.util.module_from_spec(spec); spec.loader.exec_module(mg)
    X, _ = mg.dataset(123, 2000, 10)
    g = GOLDEN["models"][name]
    b = capi.Booster(model_str=g["model"])
    K = 3 if name == "multiclass" else 1
    assert b.num_model_per_iteration() == K and b.num_total_model() == 5 * K and b.num_feature() == 10
    assert b.num_classes() == (3 if name == "multiclass" else 1) and b.current_iteration() == 5
    raw = np.stack([b.predict_for_mat_single(X[i], capi.PREDICT_RAW_SCORE) for i in range(8)])
    np.testing.assert_allclose(raw, np.array(g["raw_pred_first8"]), rtol=1e-12, atol=1e-12)
    s2 = b.save_model_to_string()
    b2 = capi.Booster(model_str=s2)
    assert b2.save_model_to_string() == s2
    np.testing.assert_array_equal(b2.predict_for_mat(X[:200], capi.PREDICT_RAW_SCORE), b.predict_for_mat(X[:200], capi.PREDICT_RAW_SCORE))
    from mmlspark_b200.modeltext import parse_model, compare_models
    compare_models(parse_model(s2), parse_model(g["model"]), value_tol=1e-15)
    # normal prediction = objective transform of raw
    p = b.predict_for_mat(X[:50])
    r = b.predict_for_mat(X[:50], capi.PREDICT_RAW_SCORE)
    if name == "binary":
        np.testing.assert_allclose(p, 1 / (1 + np.exp(-r)), rtol=1e-12)
    elif name == "multiclass":
        e = np.exp(r - r.max(axis=1, keepdims=True))
        np.testing.assert_allclose(p, e / e.sum(axis=1, keepdims=True), rtol=1e-12)
        np.testing.assert_allclose(p.sum(axis=1), 1.0, atol=1e-12)        # VerifyLightGBMClassifier.scala:91-99
    else:
        np.testing.assert_array_equal(p, r)
    # start_iteration / num_iteration (VerifyLightGBMClassifier.scala:385-397)
    r2 = b.predict_for_mat(X[:50], capi.PREDICT_RAW_SCORE, 0, 2)
    r3 = b.predict_for_mat(X[:50], capi.PREDICT_RAW_SCORE, 2, -1)
    np.testing.assert_allclose(r2 + r3, r, rtol=1e-12, atol=1e-12)
    # CSR single row == dense single row
    row = X[3].copy(); row[np.isnan(row)] = 0.0
    nz = np.nonzero(row)[0]
    np.testing.assert_allclose(b.predict_for_csr_single(nz, row[nz], 10, capi.PREDICT_RAW_SCORE), b.predict_for_mat_single(row, capi.PREDICT_RAW_SCORE))


def test_leaf_index_and_shap_properties(capi):
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "golden", "make_golden.py"))
    mg = importlib.util.module_from_spec(spec); spec.loader.exec_module(mg)
    X, _ = mg.dataset(123, 2000, 10)
    b = capi.Booster(model_str=GOLDEN["models"]["binary"]["model"])
    leaves = b.predict_for_mat(X[:100], capi.PREDICT_LEAF_INDEX)
    assert leaves.shape == (100, 5) and (leaves == np.round(leaves)).all() and leaves.min() >= 0 and leaves.max() < 7   # :512-535
    shap = b.predict_for_mat(X[:100], capi.PREDICT_CONTRIB)
    assert shap.shape == (100, 11)                                                                                           # :537-567
    raw = b.predict_for_mat(X[:100], capi.PREDICT_RAW_SCORE)[:, 0]
    np.testing.assert_allclose(shap.sum(axis=1), raw, rtol=1e-9, atol=1e-9)     # predict == sum(shap)  (VerifyLightGBMRanker.scala:124)
    mc = capi.Booster(model_str=GOLDEN["models"]["multiclass"]["model"])
    shap3 = mc.predict_for_mat(X[:20], capi.PREDICT_CONTRIB)
    assert shap3.shape == (20, 33)
    np.testing.assert_allclose(shap3.reshape(20, 3, 11).sum(axis=2), mc.predict_for_mat(X[:20], capi.PREDICT_RAW_SCORE), rtol=1e-9, atol=1e-9)


def test_feature_importance_dump_and_merge(capi):
    g = GOLDEN["models"]["regression"]["model"]
    b = capi.Booster(model_str=g)
    split = b.feature_importance("split")
    gain = b.feature_importance("gain")
    from mmlspark_b200.modeltext import parse_model
    m = parse_model(g)
    want = np.zeros(10)
    for t in m["trees"]:
        for f, gn in zip(t["split_feature"], t["split_gain"]):
            if gn > 0:
                want[f] += 1
    np.testing.assert_array_equal(split, want)
    assert (gain[want > 0] > 0).all() and (gain[want == 0] == 0).all()
    dump = json.loads(b.dump_model())
    assert dump["num_class"] == 1 and len(dump["tree_info"]) == 5 and dump["tree_info"][0]["num_leaves"] == m["trees"][0]["num_leaves"]
    # LGBM_BoosterMerge: other's trees come first (GBDT::MergeFrom)
    a, o = capi.Booster(model_str=g), capi.Booster(model_str=g)
    a.merge(o)
    assert a.num_total_model() == 10
    x = np.linspace(-1, 1, 10)
    np.testing.assert_allclose(a.predict_for_mat_single(x, capi.PREDICT_RAW_SCORE), 2 * b.predict_for_mat_single(x, capi.PREDICT_RAW_SCORE), rtol=1e-12)


def test_gradients_of_a_loaded_model_fail_loudly(capi):
    """B200GBM_BoosterGetGradients needs training data: a booster loaded from a model string has none."""
    b = capi.Booster(model_str=GOLDEN["models"]["regression"]["model"])
    g, h = np.zeros(1, np.float32), np.zeros(1, np.float32)
    with pytest.raises(capi.LightGBMError, match="model string"):
        capi.check(capi.load().B200GBM_BoosterGetGradients(b.handle, capi._ptr(g), capi._ptr(h)))
    with pytest.raises(capi.LightGBMError, match="model string"):
        b.get_gradients()


def test_save_model_small_buffer_protocol(capi):
    """saveToString passes a 10 000-byte buffer and retries with out_len (LightGBMBooster.scala:269-274)."""
    g = GOLDEN["models"]["binary"]["model"]
    b = capi.Booster(model_str=g)
    lib = capi.load()
    n = C.c_int64(0)
    buf = C.create_string_buffer(16)
    assert lib.LGBM_BoosterSaveModelToString(b.handle, 0, -1, 0, C.c_int64(16), C.byref(n), buf) == 0
    assert n.value > 16
    buf = C.create_string_buffer(n.value)
    assert lib.LGBM_BoosterSaveModelToString(b.handle, 0, -1, 0, C.c_int64(n.value), C.byref(n), buf) == 0
    assert buf.value.decode() == b.save_model_to_string(buffer_len=50)


def test_chunked_array_semantics(capi):
    """SwigUtils.scala:22-90 — add / counts / getitem / coalesce / release."""
    for code, dt in ((capi.DTYPE_FLOAT32, np.float32), (capi.DTYPE_FLOAT64, np.float64), (capi.DTYPE_INT32, np.int32)):
        ca = capi.ChunkedArray(code, 4)
        vals = np.arange(11).astype(dt)
        for v in vals[:6]:
            ca.add(float(v))
        ca.add_many(vals[6:])
        assert ca.get_add_count() == 11 and ca.get_chunks_count() == 3 and ca.get_last_chunk_add_count() == 3
        assert ca.getitem(1, 2, -1.0) == 6 and ca.getitem(2, 3, -1.0) == -1.0 and ca.getitem(9, 0, -7.0) == -7.0
        np.testing.assert_array_equal(ca.coalesce(), vals)
        ca.release()
        assert ca.get_add_count() == 0
        ca.free()
    with pytest.raises(capi.LightGBMError):
        capi.ChunkedArray(capi.DTYPE_FLOAT32, 0)


def test_sample_indices_matches_lcg(capi):
    from oracle import oracle as O
    for n, k in ((1000, 10), (5000, 4000), (300000, 200000)):
        np.testing.assert_array_equal(capi.sample_indices(n, k, 1), O.random_sample(1, n, k))


def test_jni_shim_compiles_and_links(built, tmp_path):
    """jvm/b200gbm_jni.c (INTEGRATION.md) against a stand-in jni.h and the real libb200gbm.so: every native the reference's Scala
    code reaches through com.microsoft.ml.lightgbm.lightgbmlib (grep of lightgbm/src/main/scala, SURVEY.md §8b) is defined and
    every C symbol it forwards to resolves (-Wl,--no-undefined)."""
    import shutil
    import subprocess
    import __graft_entry__ as g
    cc = shutil.which("gcc")
    if cc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "lib_lightgbm_swig.so")
    cmd = [cc, "-shared", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(root, "jvm", "stub"), "-I" + os.path.join(root, "include"),
           os.path.join(root, "jvm", "b200gbm_jni.c"), "-L" + os.path.dirname(g.LIB), "-lb200gbm", "-Wl,--no-undefined", "-o", out]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    syms = subprocess.run(["nm", "-D", "--defined-only", out], check=True, capture_output=True, text=True).stdout
    used_by_reference = [
        "LGBM_GetLastError", "LGBM_NetworkInit", "LGBM_NetworkFree", "LGBM_DatasetCreateFromMat", "LGBM_DatasetCreateFromCSR", "LGBM_DatasetSetField",
        "LGBM_DatasetGetField", "LGBM_DatasetGetNumData", "LGBM_DatasetGetNumFeature", "LGBM_DatasetSetFeatureNames", "LGBM_DatasetFree", "LGBM_BoosterCreate",
        "LGBM_BoosterLoadModelFromString", "LGBM_BoosterMerge", "LGBM_BoosterAddValidData", "LGBM_BoosterFree", "LGBM_BoosterUpdateOneIter",
        "LGBM_BoosterUpdateOneIterCustom", "LGBM_BoosterResetParameter", "LGBM_BoosterGetEvalNamesSWIG", "LGBM_BoosterGetEval", "LGBM_BoosterGetPredict",
        "LGBM_BoosterGetNumClasses", "LGBM_BoosterNumModelPerIteration", "LGBM_BoosterNumberOfTotalModel", "LGBM_BoosterGetNumFeature",
        "LGBM_BoosterFeatureImportance", "LGBM_BoosterSaveModelToStringSWIG", "LGBM_BoosterDumpModelSWIG", "LGBM_BoosterPredictForMatSingle",
        "LGBM_BoosterPredictForCSRSingle", "StringArrayHandle_get_strings", "StringArrayHandle_free", "new_intp", "delete_intp", "intp_value",
        "new_int32_tp", "int32_tp_value", "new_int64_tp", "int64_tp_assign", "int64_tp_value", "delete_int64_tp", "new_voidpp", "voidpp_handle", "voidpp_value",
        "new_intArray", "delete_intArray", "intArray_getitem", "intArray_setitem", "new_floatArray", "delete_floatArray", "floatArray_setitem",
        "new_doubleArray", "delete_doubleArray", "doubleArray_getitem", "doubleArray_setitem", "int_to_voidp_ptr", "float_to_voidp_ptr", "double_to_voidp_ptr",
        "new_floatChunkedArray", "delete_floatChunkedArray", "floatChunkedArray_add", "floatChunkedArray_get_add_count", "floatChunkedArray_get_chunks_count",
        "floatChunkedArray_get_last_chunk_add_count", "floatChunkedArray_getitem", "floatChunkedArray_coalesce_to", "floatChunkedArray_release",
        "new_doubleChunkedArray", "doubleChunkedArray_add", "doubleChunkedArray_coalesce_to", "doubleChunkedArray_release", "new_int32ChunkedArray"]
    for name in used_by_reference:
        mangled = "Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_" + name.replace("_", "_1")
        assert mangled in syms, name
