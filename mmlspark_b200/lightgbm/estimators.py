"""LightGBMClassifier / LightGBMRegressor / LightGBMRanker estimators and their models — the host-side mirror of
lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/{LightGBMBase,LightGBMClassifier,LightGBMRegressor,
LightGBMRanker,LightGBMModelMethods}.scala and booster/LightGBMBooster.scala, driving the b200gbm engine through the
C ABI.  There is no JVM/Spark in this environment, so a "DataFrame" is a `Frame` (dict of numpy columns, the
features column being a 2-D array or a scipy.sparse matrix) or a pandas DataFrame; a Spark partition is a contiguous row block and a Spark
task is a rank-thread bound to one GPU (SURVEY.md fact 8: in local mode all tasks are threads of one JVM)."""
import logging
import os
import threading

import numpy as np

from .. import capi
from . import train_utils as tu
from .params import COMMON_DEFAULTS, Params, TrainParams, dataset_params

log = logging.getLogger("mmlspark_b200.lightgbm")


def _is_sparse(x):
    """A scipy.sparse matrix or array (told apart without importing scipy)."""
    return not isinstance(x, np.ndarray) and hasattr(x, "tocsr") and hasattr(x, "nnz")


def _canonical_csr(x):
    """CSR with sorted, distinct indices per row: scipy's meaning of repeated entries (their sum) in every path that reads them."""
    m = x.tocsr()
    if not m.has_canonical_format:
        m = m.copy()
        m.sum_duplicates()
    return m


def _to_sparse(X):
    """Dense rows to CSR the way Spark's DenseVector.toSparse does: every value != 0 is kept, NaN included."""
    import scipy.sparse as sp
    X = np.asarray(X, dtype=np.float64)
    keep = X != 0
    indptr = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
    return sp.csr_matrix((X[keep], np.nonzero(keep)[1].astype(np.int32), indptr), shape=X.shape)


def resolve_matrix_type(matrix_type, features):
    """The features column as the fit will read it, sparse or dense (SharedState.scala:28-36; DatasetAggregator.scala:142-150).
    auto: as given (in a column of one kind the reference's vote over the first 10 rows always picks that kind); sparse: dense rows go
    through toSparse; dense: sparse rows are densified."""
    if matrix_type not in ("auto", "sparse", "dense"):
        raise ValueError("Invalid parameter matrix type specified: %s" % matrix_type)
    if _is_sparse(features):
        m = _canonical_csr(features)
        return m.toarray() if matrix_type == "dense" else m
    return _to_sparse(features) if matrix_type == "sparse" else features


def _row_features(x):
    return x if _is_sparse(x) else np.asarray(x, dtype=np.float64)


def _batch_features(col):
    return _canonical_csr(col) if _is_sparse(col) else np.ascontiguousarray(col, dtype=np.float64)


class Frame(dict):
    """Minimal columnar frame: column name -> numpy array.  The features column is [n_rows, n_features], a 2-D array of dense rows
    or a scipy.sparse matrix of sparse rows."""

    @classmethod
    def of(cls, data):
        if isinstance(data, Frame):
            return data
        if isinstance(data, dict):
            return cls({k: v if _is_sparse(v) else np.asarray(v) for k, v in data.items()})
        try:
            import pandas as pd
            if isinstance(data, pd.DataFrame):
                out = cls()
                for c in data.columns:
                    col = data[c]
                    if col.dtype == object and len(col) and hasattr(col.iloc[0], "__len__"):
                        out[c] = np.stack([np.asarray(v, dtype=np.float64) for v in col.values])
                    else:
                        out[c] = col.values
                return out
        except ImportError:
            pass
        raise TypeError("expected Frame, dict or pandas.DataFrame")

    def num_rows(self):
        if not self:
            return 0
        v = next(iter(self.values()))
        return v.shape[0] if _is_sparse(v) else len(v)

    def rows(self, sl):
        """Rows by slice, boolean mask or index array."""
        return Frame({k: v.tocsr()[sl] if _is_sparse(v) else v[sl] for k, v in self.items()})

    def with_column(self, name, values):
        out = Frame(self)
        out[name] = values
        return out


class LightGBMBooster:
    """booster/LightGBMBooster.scala: the model string plus a lazily created native handle used for prediction."""

    def __init__(self, model_str):
        self.modelStr = model_str
        self._native = None
        self._lock = threading.Lock()
        self.bestIteration = -1
        self.startIteration = 0
        self.numIterations = -1

    def _handle(self):
        with self._lock:
            if self._native is None:
                self._native = capi.Booster(model_str=self.modelStr)   # BoosterHandler(model) (:41-48)
            return self._native

    def setBestIteration(self, it):          # :444-447
        self.bestIteration = it
        self.numIterations = it

    def setStartIteration(self, v): self.startIteration = v
    def setNumIterations(self, v): self.numIterations = v

    @property
    def numClasses(self): return self._handle().num_classes()
    @property
    def numFeatures(self): return self._handle().num_feature()
    @property
    def numTotalModel(self): return self._handle().num_total_model()
    @property
    def numModelPerIteration(self): return self._handle().num_model_per_iteration()
    @property
    def numTotalIterations(self): return self.numTotalModel // max(self.numModelPerIteration, 1)

    def _pred_to_array(self, classification, pred, raw):       # predToArray (:547-563)
        if classification and self.numClasses == 1:
            p = float(pred[0])
            return np.array([-p, p]) if raw else np.array([1 - p, p])
        return np.asarray(pred[:self.numClasses], dtype=np.float64)

    def _predict_row(self, features, kind):
        """One row: dense through LGBM_BoosterPredictForMatSingle, a one-row scipy.sparse matrix through
        LGBM_BoosterPredictForCSRSingle (the SparseVector branch, :510-526)."""
        if _is_sparse(features):
            m = _canonical_csr(features)
            if m.shape[0] != 1:
                raise ValueError("expected one sparse row, got %d" % m.shape[0])
            return self._handle().predict_for_csr_single(m.indices, m.data, m.shape[1], kind, self.startIteration, self.numIterations)
        return self._handle().predict_for_mat_single(features, kind, self.startIteration, self.numIterations)

    def predict_batch(self, X, kind):
        """Many rows on the GPU: a 2-D array through predict_device, a scipy.sparse matrix through predict_csr_device."""
        h = self._handle()
        if _is_sparse(X):
            return h.predict_csr_device(X, predict_type=kind, start_iteration=self.startIteration, num_iteration=self.numIterations)
        return h.predict_device(X, kind, self.startIteration, self.numIterations)

    def score(self, features, raw, classification):             # :390-398
        kind = capi.PREDICT_RAW_SCORE if raw else capi.PREDICT_NORMAL
        out = self._predict_row(features, kind)
        return self._pred_to_array(classification, out, raw)

    def predictLeaf(self, features):                            # :400-410
        return self._predict_row(features, capi.PREDICT_LEAF_INDEX)

    def featuresShap(self, features):                           # :412-423
        return self._predict_row(features, capi.PREDICT_CONTRIB)

    def score_batch(self, X, raw, classification):
        """transform(): one batched GPU prediction instead of the reference's per-row UDF (SURVEY §8f-2); same values as score()."""
        kind = capi.PREDICT_RAW_SCORE if raw else capi.PREDICT_NORMAL
        out = self.predict_batch(X, kind)
        if classification and self.numClasses == 1:
            p = out[:, 0]
            return np.stack([-p, p], axis=1) if raw else np.stack([1 - p, p], axis=1)
        return out

    def getFeatureImportances(self, importanceType="split"):    # :491-498
        return self._handle().feature_importance(importanceType).tolist()

    def saveNativeModel(self, filename, overwrite=True):        # :449-463 (single text file; lines re-joined with \n on load)
        if not filename:
            raise ValueError("filename should not be empty or null.")
        if os.path.exists(filename) and not overwrite:
            raise IOError("file exists: " + filename)
        with open(filename, "w") as f:
            f.write(self.modelStr)

    def dumpModel(self):
        return self._handle().dump_model()


class _ModelBase(Params):
    _defaults = dict(featuresCol="features", predictionCol="prediction", leafPredictionCol="", featuresShapCol="", startIteration=0,
                     numIterations=-1)

    def __init__(self, booster=None, **kw):
        super().__init__(**kw)
        self.booster = booster

    def getModel(self): return self.booster
    def getLightGBMBooster(self): return self.booster
    def saveNativeModel(self, filename, overwrite=True): self.booster.saveNativeModel(filename, overwrite)
    def getNativeModel(self): return self.booster.modelStr
    def getFeatureImportances(self, importance_type="split"): return self.booster.getFeatureImportances(importance_type)
    def getFeatureShaps(self, vector): return self.booster.featuresShap(_row_features(vector)).tolist()
    def getDenseFeatureShaps(self, features): return self.getFeatureShaps(features)          # LightGBMModelMethods.scala:33-36

    def getSparseFeatureShaps(self, size, indices, values):                                  # LightGBMModelMethods.scala:38-46
        """SHAP values of a sparse vector (size, indices, values) through LGBM_BoosterPredictForCSRSingle."""
        return self.booster._handle().predict_for_csr_single(np.asarray(indices, dtype=np.int32), np.asarray(values, dtype=np.float64), int(size),
                                                             capi.PREDICT_CONTRIB, self.booster.startIteration, self.booster.numIterations).tolist()
    def getBoosterBestIteration(self): return self.booster.bestIteration
    def getBoosterNumTotalIterations(self): return self.booster.numTotalIterations
    def getBoosterNumTotalModel(self): return self.booster.numTotalModel
    def getBoosterNumFeatures(self): return self.booster.numFeatures
    def getBoosterNumClasses(self): return self.booster.numClasses

    def _update_booster_params(self):          # updateBoosterParamsBeforePredict (LightGBMModelMethods.scala)
        self.booster.setStartIteration(self.get("startIteration"))
        self.booster.setNumIterations(self.get("numIterations"))

    def _extra_columns(self, out, X):
        if self.get("leafPredictionCol"):
            out = out.with_column(self.get("leafPredictionCol"), self.booster.predict_batch(X, capi.PREDICT_LEAF_INDEX))
        if self.get("featuresShapCol"):
            # batched TreeSHAP on the GPU (k_predict_contrib); same values as the per-row featuresShap() the reference's UDF calls
            out = out.with_column(self.get("featuresShapCol"), self.booster.predict_batch(X, capi.PREDICT_CONTRIB))
        return out

    @classmethod
    def loadNativeModelFromString(cls, model, **kw):
        return cls(LightGBMBooster(model), **kw)

    @classmethod
    def loadNativeModelFromFile(cls, filename, **kw):
        with open(filename) as f:
            return cls(LightGBMBooster(f.read()), **kw)


class LightGBMClassificationModel(_ModelBase):
    """LightGBMClassifier.scala:93-184"""
    _defaults = dict(_ModelBase._defaults, probabilityCol="probability", rawPredictionCol="rawPrediction", thresholds=None, actualNumClasses=2)

    @property
    def numClasses(self): return self.get("actualNumClasses")

    def transform(self, data):
        df = Frame.of(data)
        self._update_booster_params()
        X = _batch_features(df[self.get("featuresCol")])
        out = df
        raw = prob = None
        if self.get("rawPredictionCol"):
            raw = self.booster.score_batch(X, True, True)
            out = out.with_column(self.get("rawPredictionCol"), raw)
        if self.get("probabilityCol"):
            prob = self.booster.score_batch(X, False, True)
            out = out.with_column(self.get("probabilityCol"), prob)
        if self.get("predictionCol"):
            if prob is None and raw is None:
                raw = self.booster.score_batch(X, True, True)
            base = prob if prob is not None else raw
            th = self.get("thresholds")
            if th is not None and prob is not None:
                if len(th) != base.shape[1]:
                    raise ValueError("transform() called with non-matching numClasses and thresholds.length")
                pred = np.argmax(base / np.asarray(th, dtype=np.float64), axis=1)
            else:
                pred = np.argmax(base, axis=1)
            out = out.with_column(self.get("predictionCol"), pred.astype(np.float64))
        return self._extra_columns(out, X)


class LightGBMRegressionModel(_ModelBase):
    """LightGBMRegressor.scala:85-150"""

    def transform(self, data):
        df = Frame.of(data)
        self._update_booster_params()
        X = _batch_features(df[self.get("featuresCol")])
        out = df.with_column(self.get("predictionCol"), self.booster.score_batch(X, False, False)[:, 0])
        return self._extra_columns(out, X)

    def predict(self, features):
        self._update_booster_params()
        return float(self.booster.score(_row_features(features), False, False)[0])


class LightGBMRankerModel(LightGBMRegressionModel):
    """LightGBMRanker.scala:112-177"""


class LightGBMBase(Params):
    """LightGBMBase.scala — train / innerTrain / trainLightGBM."""
    _kind = None
    _model_cls = None

    def getTrainParams(self, numTasks, frame):
        raise NotImplementedError

    def _num_devices(self):
        try:
            import subprocess
            out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
            return max(1, len([l for l in out.splitlines() if l.startswith("GPU ")]))
        except Exception:
            return 1

    def getCategoricalIndexes(self):             # LightGBMBase.getCategoricalIndexes (:168-198)
        """categoricalSlotIndexes united with the positions of categoricalSlotNames in slotNames (first occurrences kept, like
        Scala's union.distinct).  A Frame carries no ML attribute metadata, so names can only be resolved through slotNames."""
        names = list(self.get("slotNames") or ())
        by_name = [names.index(c) if c in names else -1 for c in (self.get("categoricalSlotNames") or ())] if names else []
        out = []
        for i in list(self.get("categoricalSlotIndexes") or ()) + by_name:
            if i not in out:
                out.append(int(i))
        return out

    def validateSlotNames(self):                 # LightGBMBase.validateSlotNames (:218-232)
        bad = [n for n in (self.get("slotNames") or ()) if any(ch in n for ch in '",:[]{}')]
        if bad:
            raise ValueError("Invalid slot names detected in features column: " + ",".join(bad))

    def fit(self, data):                         # train (:43-66)
        df = Frame.of(data)
        self.validateSlotNames()
        nb = self.get("numBatches")
        if nb and nb > 0:
            n = df.num_rows()
            perm = np.random.default_rng(0).permutation(n)
            model = None
            for bi, part in enumerate(np.array_split(perm, nb)):
                if model is not None:
                    self.setModelString(model.booster.modelStr)
                batch = df.rows(np.sort(part))
                d = self.get("delegate")
                if d is not None:
                    d.beforeTrainBatch(bi, batch, model)
                model = self._inner_train(batch, bi)
                if d is not None:
                    d.afterTrainBatch(bi, batch, model)
            return model
        return self._inner_train(df, 0)

    def _partitions(self, df, num_tasks):
        """coalesce(numTasks): contiguous row blocks (rows never move after this, is_pre_partition=True)."""
        n = df.num_rows()
        bounds = np.linspace(0, n, num_tasks + 1).astype(np.int64)
        return [slice(int(bounds[i]), int(bounds[i + 1])) for i in range(num_tasks)]

    def _inner_train(self, df, batch_index):     # innerTrain (:440-489)
        num_tasks = self.get("numTasks") if self.get("numTasks") > 0 else self._num_devices()
        fcol = self.get("featuresCol")
        df = df.with_column(fcol, resolve_matrix_type(self.get("matrixType"), df[fcol]))      # once per fit, train and validation alike
        vcol = self.get("validationIndicatorCol")
        valid = None
        if vcol and vcol in df:
            mask = np.asarray(df[vcol]).astype(bool)
            # the reference runs preprocessData (the ranker's sortWithinPartitions(groupCol)) on the validation frame too
            # (LightGBMBase.scala:465-468): without it count_cardinality(valid[groupCol]) would fragment shuffled query groups
            valid = self._preprocess(df.rows(mask))
            df = df.rows(~mask)
        df = self._preprocess(df)
        parts = self._partitions(df, num_tasks)
        train_params = self.getTrainParams(num_tasks, df)
        log.info("LightGBM parameters: %s", train_params.to_string())
        driver = tu.DriverRendezvous(num_tasks, self.get("driverListenPort"), self.get("timeout"))
        host, port = driver.start()
        results, errors = [None] * num_tasks, []
        single = bool(self.get("useSingleDatasetMode"))

        def task(pid):
            try:
                # single-dataset mode: the tasks of one device train as one rank over their partitions, in pid order.  The reference
                # gathers those rows on the executor behind latches (SharedState); in this in-process mirror the main task reads its
                # group's partitions from the frame directly, so no task waits for another.
                rows = self._device_group(pid, parts, num_tasks) if single else [pid]
                part_frames = [df.rows(parts[q]) for q in rows]
                results[pid] = self._train_lightgbm(batch_index, pid, part_frames, valid, train_params, host, port, num_tasks)
            except Exception as e:   # noqa
                log.exception("task %d failed", pid)
                errors.append(e)

        threads = [threading.Thread(target=task, args=(i,)) for i in range(num_tasks)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        driver.join(self.get("timeout"))
        if errors:
            raise errors[0]
        boosters = [r for r in results if r is not None]
        if not boosters:
            raise RuntimeError("no task returned a booster")
        return self.getModel(train_params, boosters[0])   # .reduce((b1, _) => b1)

    def _preprocess(self, df):
        return df

    def _device_group(self, pid, parts, num_tasks):
        """Single-dataset mode: the partitions task pid trains on.  The tasks of one device (pid % number of devices) form a group whose
        main task is the lowest pid with a non-empty partition; it gets the group's non-empty partitions in pid order, every other task
        none (it reports "ignore" like a disabled worker of the reference, LightGBMBase.trainLightGBM)."""
        ndev = self._num_devices()
        group = [q for q in range(num_tasks) if q % ndev == pid % ndev and parts[q].stop > parts[q].start]
        return group if group and group[0] == pid else []

    def _make_dataset(self, part, params_str, reference=None):
        """One dataset from a frame, or from a list of frames that count as one in order: a device group's partitions in single-dataset
        mode (their feature matrices go to the library as they are, never concatenated here)."""
        parts = part if isinstance(part, list) else [part]
        Xs = [p[self.get("featuresCol")] for p in parts]
        if len(Xs) > 1 and _is_sparse(Xs[0]):
            ds = capi.Dataset.from_csrs(Xs, Xs[0].shape[1], params_str, reference=reference)
        elif len(Xs) > 1:
            ds = capi.Dataset.from_mats([np.ascontiguousarray(X, dtype=np.float64) for X in Xs], params_str, reference=reference)
        elif _is_sparse(Xs[0]):      # CSR from resolve_matrix_type
            X = Xs[0]
            ds = capi.Dataset.from_csr(X.indptr, X.indices, X.data, X.shape[1], params_str, reference=reference)
        else:
            ds = capi.Dataset.from_mat(np.ascontiguousarray(Xs[0], dtype=np.float64), params_str, reference=reference)

        def column(name, dtype):
            return np.concatenate([np.asarray(p[name], dtype=dtype) for p in parts])

        ds.set_field("label", column(self.get("labelCol"), np.float32))       # narrowed to f32 (DatasetAggregator.scala:89-92)
        if self.get("weightCol"):
            ds.set_field("weight", column(self.get("weightCol"), np.float32))
        if self.get("initScoreCol"):
            init = column(self.get("initScoreCol"), np.float64)
            ds.set_field("init_score", init.T.reshape(-1) if init.ndim == 2 else init)    # class-major at the C ABI (Appendix D)
        gcol = self.get("groupCol") if "groupCol" in self._defaults else None
        if gcol:      # partitions never split a query, so the parts' runs are the runs of their concatenation
            ds.set_field("group", np.asarray([c for p in parts for c in tu.count_cardinality(p[gcol].tolist())], dtype=np.int32))
        pcol = self.get("positionCol") if "positionCol" in self._defaults else None
        if pcol:      # display positions of the ranker's rows: the ranking objectives learn one score factor per position
            ds.set_field("position", column(pcol, np.int32))
        names = list(self.get("slotNames"))
        if names:
            ds.set_feature_names(names)
        return ds

    def _train_lightgbm(self, batch_index, pid, parts, valid, train_params, driver_host, driver_port, num_tasks):
        """trainLightGBM (:337-382) + translate (:292-335) for one rank-thread: its partition, or in single-dataset mode its device
        group's partitions (none for a task that is not the group's main task)."""
        capi.set_device(pid % self._num_devices())
        parts = [p for p in parts if p.num_rows() > 0]
        empty = not parts
        sock, local_port = tu.find_open_port(self.get("defaultListenPort"), pid)
        try:
            nodes = tu.get_network_init_nodes(driver_host, driver_port, local_port, empty)
        finally:
            sock.close()
        if empty:
            return None                                   # "ignore" protocol for empty partitions and non-main tasks
        use_net = len(nodes.split(",")) > 1
        try:
            if use_net:
                tu.network_init(nodes, local_port)
            ds_params = dataset_params(self.get("maxBin"), self.get("binSampleCount"), self.get("numThreads"), train_params.categoricalFeatures)
            train_ds = self._make_dataset(parts if len(parts) > 1 else parts[0], ds_params)
            valid_ds = None
            try:
                # built once per rank; in single-dataset mode the validation rows stay apart from the training rows (the reference's
                # SharedState.merge would hand both the same shared aggregate)
                if valid is not None and valid.num_rows() > 0:
                    valid_ds = self._make_dataset(valid, ds_params, reference=train_ds)
                booster = tu.create_booster(train_params, train_ds, valid_ds)
                try:
                    best = tu.train_core(batch_index, pid, train_params, booster, valid_ds is not None,
                                         train_label=np.concatenate([np.asarray(p[self.get("labelCol")], dtype=np.float32) for p in parts]))
                    if tu.get_main_worker_port(nodes) == local_port:      # getReturnBooster (:355-363)
                        mb = LightGBMBooster(booster.save_model_to_string())
                        if best is not None:
                            mb.setBestIteration(best)
                        return mb
                    return None
                finally:
                    booster.free()
            finally:
                if valid_ds is not None:
                    valid_ds.free()
                train_ds.free()
        finally:
            if use_net:
                capi.network_free()


_CLS_DEFAULTS = dict(COMMON_DEFAULTS, objective="binary", isUnbalance=False, probabilityCol="probability", rawPredictionCol="rawPrediction", thresholds=None)
_REG_DEFAULTS = dict(COMMON_DEFAULTS, objective="regression", alpha=0.9, tweedieVariancePower=1.5)
# positionCol / lambdarankPositionBiasRegularization: LightGBM 4.1's unbiased lambdarank (the dataset's position field and
# lambdarank_position_bias_regularization); the reference has no such parameters
_RNK_DEFAULTS = dict(COMMON_DEFAULTS, objective="lambdarank", maxPosition=20, labelGain=(), evalAt=(1, 2, 3, 4, 5), groupCol=None,
                     positionCol=None, lambdarankPositionBiasRegularization=0.0)


class LightGBMClassifier(LightGBMBase):
    """LightGBMClassifier.scala:26-88"""
    _defaults = _CLS_DEFAULTS
    _kind = "classifier"

    def getTrainParams(self, numTasks, frame):
        labels = np.asarray(frame[self.get("labelCol")])
        num_class = int(labels.max()) + 1 if self.get("objective") != "binary" else 2      # getNumClasses
        return TrainParams("classifier", self.params_dict(), numTasks, self.getCategoricalIndexes(), num_class, self.get("slotNames"))

    def getModel(self, train_params, booster):
        m = LightGBMClassificationModel(booster, featuresCol=self.get("featuresCol"), predictionCol=self.get("predictionCol"),
                                        probabilityCol=self.get("probabilityCol"), rawPredictionCol=self.get("rawPredictionCol"),
                                        leafPredictionCol=self.get("leafPredictionCol"), featuresShapCol=self.get("featuresShapCol"),
                                        actualNumClasses=train_params.numClass, numIterations=booster.bestIteration)
        if self.get("thresholds") is not None:
            m.setThresholds(self.get("thresholds"))
        return m


class LightGBMRegressor(LightGBMBase):
    """LightGBMRegressor.scala:39-83"""
    _defaults = _REG_DEFAULTS
    _kind = "regressor"

    def getTrainParams(self, numTasks, frame):
        return TrainParams("regressor", self.params_dict(), numTasks, self.getCategoricalIndexes(), 1, self.get("slotNames"))

    def getModel(self, train_params, booster):
        return LightGBMRegressionModel(booster, featuresCol=self.get("featuresCol"), predictionCol=self.get("predictionCol"),
                                       leafPredictionCol=self.get("leafPredictionCol"), featuresShapCol=self.get("featuresShapCol"),
                                       numIterations=booster.bestIteration)


class LightGBMRanker(LightGBMBase):
    """LightGBMRanker.scala:27-110"""
    _defaults = _RNK_DEFAULTS
    _kind = "ranker"

    def getTrainParams(self, numTasks, frame):
        return TrainParams("ranker", self.params_dict(), numTasks, self.getCategoricalIndexes(), 1, self.get("slotNames"))

    def _partitions(self, df, num_tasks):
        """repartition by grouping column: whole query groups stay on one rank (LightGBMRanker.scala:93-108)."""
        g = np.asarray(df[self.get("groupCol")])
        n = len(g)
        starts = np.concatenate([[0], np.nonzero(g[1:] != g[:-1])[0] + 1, [n]])
        target = np.linspace(0, n, num_tasks + 1)
        cuts = [0]
        for t in target[1:-1]:
            cuts.append(int(starts[np.searchsorted(starts, t, side="left")]) if len(starts) else 0)
        cuts.append(n)
        cuts = np.maximum.accumulate(np.array(cuts))
        return [slice(int(cuts[i]), int(cuts[i + 1])) for i in range(num_tasks)]

    def _preprocess(self, df):
        """sortWithinPartitions(groupCol) — here: one stable sort by group id before partitioning."""
        g = np.asarray(df[self.get("groupCol")])
        is_text = g.dtype.kind in "US" or (g.dtype.kind == "O" and all(isinstance(v, str) for v in g.tolist()))
        if g.dtype.kind not in "iu" and not is_text:      # int, long and string query columns are accepted (VerifyLightGBMRanker.scala:60-82)
            raise ValueError("group column must be of type int, long or string")
        order = np.argsort(g, kind="stable")
        return df.rows(order)

    def getModel(self, train_params, booster):
        return LightGBMRankerModel(booster, featuresCol=self.get("featuresCol"), predictionCol=self.get("predictionCol"),
                                   leafPredictionCol=self.get("leafPredictionCol"), featuresShapCol=self.get("featuresShapCol"),
                                   numIterations=booster.bestIteration)
