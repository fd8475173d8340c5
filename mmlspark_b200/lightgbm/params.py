"""Param surface + TrainParams wire format of the reference's LightGBM estimators.

Mirrors lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/params/LightGBMParams.scala (names, defaults)
and params/TrainParams.scala:47-179 (the exact `key=value` string handed to LGBM_BoosterCreate).  The Python
API keeps the generated PySpark wrappers' shape: camelCase keyword constructor, setX/getX per Param
(SURVEY.md B.4)."""
import math

# name -> default   (LightGBMParams.scala line numbers in comments)
COMMON_DEFAULTS = dict(
    parallelism="data_parallel",       # :16-18
    topK=20,                            # :23-27
    defaultListenPort=12400,            # :32-38
    driverListenPort=0,                 # :40-46
    timeout=1200.0,                     # :48-49
    useBarrierExecutionMode=False,      # :54-56
    useSingleDatasetMode=False,         # :61-64
    numBatches=0,                       # :69-71
    repartitionByGroupingColumn=True,   # :76-78
    numTasks=0,                         # :83-86
    chunkSize=10000,                    # :91-95
    matrixType="auto",                  # :100-103
    numThreads=0,                       # :108-110
    earlyStoppingRound=0,               # :119-120
    improvementTolerance=0.0,           # :125-127
    maxBin=255,                         # :136-137
    binSampleCount=200000,              # :142-143
    dropRate=0.1, maxDrop=50, skipDrop=0.5, xgboostDartMode=False, uniformDrop=False,   # :152-182
    slotNames=(), categoricalSlotIndexes=(), categoricalSlotNames=(),                   # :191-213
    baggingFraction=1.0, posBaggingFraction=1.0, negBaggingFraction=1.0, featureFraction=1.0,   # :219-238
    leafPredictionCol="", featuresShapCol="",                                           # :247-256
    objective="regression",             # :296-300
    fobj=None,                          # :305
    numIterations=100, learningRate=0.1, numLeaves=31, baggingFreq=0, baggingSeed=3, maxDepth=-1,   # :318-350
    minSumHessianInLeaf=1e-3,           # :355-356
    modelString="",                     # :361-362
    verbosity=-1,                       # :367-369
    boostFromAverage=True,              # :374-376
    boostingType="gbdt",                # :381-385
    lambdaL1=0.0, lambdaL2=0.0,         # :390-397
    isProvideTrainingMetric=False,      # :402-404
    metric="",                          # :409-438
    minGainToSplit=0.0, maxDeltaStep=0.0, maxBinByFeature=(), minDataInLeaf=20,         # :443-466
    extraTrees=False, extraSeed=6,      # LightGBM 3.2's extra_trees / extra_seed (not a param of the reference's estimators)
    monotoneConstraints=(), monotoneConstraintsMethod="basic", monotonePenalty=0.0,      # monotone_constraints (per feature -1/0/1) etc.
    interactionConstraints=(),          # interaction_constraints: lists of feature indices; a branch splits on features of one list only
    featureFractionByNode=1.0,          # feature_fraction_bynode: the share of the tree's features each leaf's split is chosen from
    pathSmooth=0.0,                     # path_smooth: smooths every split gain and leaf output toward the parent leaf's output
    forcedSplitsFilename="",            # forcedsplits_filename: a JSON file of splits every tree starts with (no spaces in the path)
    # LightGBM 4's quantised training: use_quantized_grad, num_grad_quant_bins, quant_train_renew_leaf, stochastic_rounding
    useQuantizedGrad=False, numGradQuantBins=4, quantTrainRenewLeaf=False, stochasticRounding=True,
    delegate=None,
    # column params (core/contracts/Params.scala:93-208 + Spark ML)
    featuresCol="features", labelCol="label", predictionCol="prediction", weightCol=None, initScoreCol=None,
    validationIndicatorCol=None,
    startIteration=0,
)


def scala_double(x):
    """java.lang.Double.toString: shortest round-trip digits; plain decimal in [1e-3, 1e7), else d.dddE[-]n."""
    from decimal import Decimal
    x = float(x)
    if x != x:
        return "NaN"
    if math.isinf(x):
        return "Infinity" if x > 0 else "-Infinity"
    if x == 0:
        return "0.0" if math.copysign(1, x) > 0 else "-0.0"
    d = Decimal(repr(x)).normalize()
    sign, digits, exp = d.as_tuple()
    ds = "".join(str(k) for k in digits)
    sci = len(ds) + exp - 1
    neg = "-" if sign else ""
    if 1e-3 <= abs(x) < 1e7:
        s = format(abs(d), "f")
        if "." not in s:
            s += ".0"
        return neg + s
    return "%s%s.%sE%d" % (neg, ds[0], ds[1:] or "0", sci)


def scala_bool(b):
    return "true" if b else "false"


class ObjectiveParams:
    """params/TrainParams.scala:173-179"""

    def __init__(self, objective, fobj=None):
        self.objective, self.fobj = objective, fobj

    def to_string(self):
        return "objective=%s " % self.objective if self.fobj is None else ""


class TrainParams:
    """params/TrainParams.scala:10-63.  `kind` in {classifier, regressor, ranker}."""

    def __init__(self, kind, p, numMachines, categoricalFeatures=(), numClass=1, featureNames=()):
        self.kind = kind
        self.p = dict(p)
        self.numMachines = numMachines
        self.categoricalFeatures = list(categoricalFeatures)
        self.numClass = numClass
        self.featureNames = list(featureNames)
        self.objectiveParams = ObjectiveParams(p["objective"], p.get("fobj"))
        for k in ("numIterations", "learningRate", "earlyStoppingRound", "improvementTolerance", "isProvideTrainingMetric", "delegate"):
            setattr(self, k, p[k])
        self.modelString = p["modelString"] or None

    def _base(self):
        p = self.p
        s = ("is_pre_partition=True boosting_type=%s tree_learner=%s top_k=%d " % (p["boostingType"], p["parallelism"], p["topK"]) +
             "num_iterations=%d learning_rate=%s num_leaves=%d " % (p["numIterations"], scala_double(p["learningRate"]), p["numLeaves"]) +
             "max_bin=%d bagging_fraction=%s pos_bagging_fraction=%s " % (p["maxBin"], scala_double(p["baggingFraction"]), scala_double(p["posBaggingFraction"])) +
             "neg_bagging_fraction=%s bagging_freq=%d " % (scala_double(p["negBaggingFraction"]), p["baggingFreq"]) +
             "bagging_seed=%d early_stopping_round=%d " % (p["baggingSeed"], p["earlyStoppingRound"]) +
             "feature_fraction=%s max_depth=%d min_sum_hessian_in_leaf=%s " % (scala_double(p["featureFraction"]), p["maxDepth"], scala_double(p["minSumHessianInLeaf"])) +
             "num_machines=%d verbosity=%d " % (self.numMachines, p["verbosity"]) +
             "lambda_l1=%s lambda_l2=%s metric=%s min_gain_to_split=%s " % (scala_double(p["lambdaL1"]), scala_double(p["lambdaL2"]), p["metric"], scala_double(p["minGainToSplit"])) +
             "max_delta_step=%s min_data_in_leaf=%d %s " % (scala_double(p["maxDeltaStep"]), p["minDataInLeaf"], self.objectiveParams.to_string()))
        if self.categoricalFeatures:
            s += "categorical_feature=%s " % ",".join(str(i) for i in self.categoricalFeatures)
        if p["maxBinByFeature"]:
            s += "max_bin_by_feature=%s " % ",".join(str(i) for i in p["maxBinByFeature"])
        if p["boostingType"] == "dart":
            s += ("drop_rate=%s max_drop=%d skip_drop=%s xgboost_dart_mode=%s uniform_drop=%s  " % (
                scala_double(p["dropRate"]), p["maxDrop"], scala_double(p["skipDrop"]), scala_bool(p["xgboostDartMode"]), scala_bool(p["uniformDrop"])))
        s += "num_threads=%d " % p["numThreads"]
        if p["extraTrees"]:      # only when set, so every other parameter string stays as the reference builds it
            s += "extra_trees=true extra_seed=%d " % p["extraSeed"]
        if len(p["monotoneConstraints"]) > 0:      # only when given, so every other parameter string stays as the reference builds it
            s += "monotone_constraints=%s monotone_constraints_method=%s monotone_penalty=%s " % (
                ",".join(str(int(c)) for c in p["monotoneConstraints"]), p["monotoneConstraintsMethod"], scala_double(p["monotonePenalty"]))
        if len(p["interactionConstraints"]) > 0:      # only when given, so every other parameter string stays as the reference builds it
            s += "interaction_constraints=%s " % ",".join("[%s]" % ",".join(str(int(f)) for f in c) for c in p["interactionConstraints"])
        if p["featureFractionByNode"] != 1.0:      # only when set, so every other parameter string stays as the reference builds it
            s += "feature_fraction_bynode=%s " % scala_double(p["featureFractionByNode"])
        if p["pathSmooth"] != 0.0:      # only when set, so every other parameter string stays as the reference builds it
            s += "path_smooth=%s " % scala_double(p["pathSmooth"])
        if p["forcedSplitsFilename"]:      # only when set, so every other parameter string stays as the reference builds it
            s += "forcedsplits_filename=%s " % p["forcedSplitsFilename"]
        if p["useQuantizedGrad"]:      # only when set, so every other parameter string stays as the reference builds it
            s += "use_quantized_grad=true num_grad_quant_bins=%d quant_train_renew_leaf=%s stochastic_rounding=%s " % (
                p["numGradQuantBins"], scala_bool(p["quantTrainRenewLeaf"]), scala_bool(p["stochasticRounding"]))
        return s

    def to_string(self):
        p = self.p
        if self.kind == "classifier":      # :83-88
            extra = "num_class=%d" % self.numClass if p["objective"] != "binary" else "is_unbalance=%s" % scala_bool(p["isUnbalance"])
            return "metric=%s boost_from_average=%s %s %s" % (p["metric"], scala_bool(p["boostFromAverage"]), self._base(), extra)
        if self.kind == "regressor":       # :108-111
            return "alpha=%s tweedie_variance_power=%s boost_from_average=%s %s" % (
                scala_double(p["alpha"]), scala_double(p["tweedieVariancePower"]), scala_bool(p["boostFromAverage"]), self._base())
        lg = "label_gain=%s" % ",".join(scala_double(x) for x in p["labelGain"]) if p["labelGain"] else ""   # :131-137
        ea = "eval_at=%s" % ",".join(str(i) for i in p["evalAt"]) if p["evalAt"] else ""
        s = "max_position=%d %s %s %s" % (p["maxPosition"], lg, ea, self._base())
        if p.get("lambdarankPositionBiasRegularization", 0.0) != 0.0:      # only when set, so every other parameter string stays as it was
            s += "lambdarank_position_bias_regularization=%s " % scala_double(p["lambdarankPositionBiasRegularization"])
        return s

    __str__ = to_string


def dataset_params(max_bin, bin_sample_count, num_threads, categorical=()):
    """LightGBMBase.getDatasetParams (LightGBMBase.scala:265-272)"""
    s = "max_bin=%d is_pre_partition=True bin_construct_sample_cnt=%d num_threads=%d" % (max_bin, bin_sample_count, num_threads)
    if categorical:
        s += " categorical_feature=" + ",".join(str(i) for i in categorical)
    return s


class Params:
    """camelCase keyword params with setX/getX, like the generated PySpark wrappers (Wrappable.scala:311-378)."""
    _defaults = {}

    def __init__(self, **kwargs):
        self._values = {}
        self.setParams(**kwargs)

    def setParams(self, **kwargs):
        for k, v in kwargs.items():
            if k not in self._defaults:
                raise TypeError("%s has no param %r" % (type(self).__name__, k))
            self._values[k] = v
        return self

    def get(self, name):
        return self._values.get(name, self._defaults[name])

    def isSet(self, name):
        return name in self._values

    def _param_of_accessor(self, suffix):
        # setNumLeaves -> numLeaves; acronym setters like setXGBoostDartMode -> xgboostDartMode (LightGBMParams.scala:176-180)
        name = suffix[0].lower() + suffix[1:]
        if name in self._defaults:
            return name
        low = suffix.lower()
        for k in self._defaults:
            if k.lower() == low:
                return k
        return None

    def __getattr__(self, item):
        if item.startswith("_"):
            raise AttributeError(item)
        if item.startswith("set") and len(item) > 3:
            name = self._param_of_accessor(item[3:])
            if name is not None:
                def setter(value, _n=name):
                    self._values[_n] = value
                    return self
                return setter
        if item.startswith("get") and len(item) > 3:
            name = self._param_of_accessor(item[3:])
            if name is not None:
                return lambda _n=name: self.get(_n)
        raise AttributeError(item)

    def params_dict(self):
        d = dict(self._defaults)
        d.update(self._values)
        return d
