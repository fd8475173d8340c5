"""Helpers the tree-by-tree GPU tests share: data and parameter builders, runs on custom or the engine's own gradients, rank-threads on
one device, and one check of an engine tree against tree_ref.grow_tree's.

The runs on custom gradients keep gradients and hessians on a 2^-10 grid with few enough rows that K4's fixed-point histograms equal
NumPy's fp64 ones bit for bit, so only the scans, the draws, the samples and the pick are under test.  Every tree of such a run is grown
from the same custom (g, h): the trees differ only by the state that carries from tree to tree (the extra-trees streams, the ColSampler
stream).  Bar (compare_tree): identical structure (feature, threshold bin, default direction, category set, which leaf splits, counts),
split_gain as printed (%g), leaf weights within 4 fp64 ulps (-O3 contracts to FMA), internal weights as printed, internal values as
printed and leaf values within 4 ulps or, where a run shrinks them by the learning rate, internal values within %g's precision (1e-5
relative) and leaf values within 1e-12 relative.  Every tree must be decided on the reference side first (split_scan_ref.undecided):
a case whose winner could flip with the last bits of a gain or a count at a .5 boundary fails instead of passing by luck."""
import threading

import numpy as np

import bynode_ref as B
import extra_trees_ref as X3
import interaction_ref as I
import split_scan_ref as ref
import tree_ref

GRID = 1.0 / 1024
DS = "min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0"


def grid(rng, lo, hi, n):
    """values on the 2^-10 grid in [lo, hi]"""
    return rng.integers(int(lo * 1024), int(hi * 1024) + 1, n) * GRID


def data(seed, n=6000, cat=False, wide=False, const_h=False):
    """numerical features (one with NaN), optionally a one-hot (3 categories) and a many-vs-many (40 categories) categorical feature, or
    two numerical features of ~500 bins and a categorical one of 600 categories (max_bin=511)"""
    rng = np.random.default_rng(seed)
    cols = [rng.integers(0, 60, n).astype(np.float64), rng.standard_normal(n), rng.integers(0, 9, n).astype(np.float64)]
    cols[1][rng.random(n) < 0.15] = np.nan
    if cat:
        cols += [rng.integers(0, 3, n).astype(np.float64), rng.integers(0, 40, n).astype(np.float64)]
    if wide:
        cols += [rng.integers(0, 500, n).astype(np.float64), rng.standard_normal(n), rng.integers(0, 600, n).astype(np.float64)]
    X = np.stack(cols, axis=1)
    y = 0.02 * X[:, 0] + np.nan_to_num(X[:, 1]) + (X[:, 2] > 4)
    if cat:
        y += 0.8 * (X[:, 3] == 1) + 0.05 * (X[:, 4] % 7)
    if wide:
        w = 5 if cat else 3
        y += 0.004 * X[:, w] + 4.0 * (X[:, w + 2] % 3 == 0)
    g = np.round((-y + 0.3 * rng.standard_normal(n)) / GRID) * GRID
    h = np.ones(n) if const_h else grid(rng, 0.5, 1.5, n)
    cats = ([3, 4] if cat else []) + ([7 if cat else 5] if wide else [])
    return X, g, h, cats


def monotone_data(n, seed):
    rng = np.random.default_rng(seed)
    # a few hundred distinct values per constrained feature, so that a sweep over all of them stays small
    X = np.stack([rng.integers(-150, 150, n) / 50.0, rng.integers(-100, 100, n) / 50.0, rng.integers(0, 50, n).astype(np.float64),
                  rng.standard_normal(n), rng.standard_normal(n)], axis=1)
    X[rng.random(n) < 0.05, 0] = np.nan
    # against the constraints in places, so an unconstrained model breaks them
    z = np.sin(2 * np.nan_to_num(X[:, 0])) + 0.8 * np.nan_to_num(X[:, 0]) - np.cos(2 * X[:, 1]) - 0.6 * X[:, 1] \
        + 0.03 * X[:, 2] + 0.3 * np.sin(X[:, 2]) + X[:, 3] * X[:, 4] + 0.3 * rng.standard_normal(n)
    return X, z


# objective and boosting options, trees per iteration, label of monotone_data's z, rows
CASES = {
    "regression": ("objective=regression", 1, lambda z: z, 50000),
    "binary": ("objective=binary", 1, lambda z: (z > np.median(z)).astype(float), 50000),
    "multiclass": ("objective=multiclass num_class=3", 3, lambda z: np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])).astype(float), 30000),
    "lambdarank": ("objective=lambdarank", 1, lambda z: np.digitize(z, np.quantile(z, [0.5, 0.8, 0.95])).astype(float), 20000),
    "goss": ("objective=regression boosting=goss", 1, lambda z: z, 50000),
    "dart": ("objective=regression boosting=dart drop_rate=0.3", 1, lambda z: z, 30000),
    "rf": ("objective=regression boosting=rf bagging_fraction=0.7 bagging_freq=1 feature_fraction=0.8", 1, lambda z: z, 50000),
    "bagging": ("objective=regression bagging_fraction=0.6 bagging_freq=1 feature_fraction=0.8", 1, lambda z: z, 200000),
}


def params(num_leaves, extra, cats=(), max_bin=255):
    p = ("objective=regression boost_from_average=false learning_rate=1 verbosity=-1 num_leaves=%d min_data_in_leaf=20 max_bin=%d %s %s"
         % (num_leaves, max_bin, DS, extra))
    if cats:
        p += " categorical_feature=" + ",".join(str(c) for c in cats)
    return p


def ds_params(cats, max_bin):
    return DS + " max_bin=%d" % max_bin + (" categorical_feature=" + ",".join(str(c) for c in cats) if cats else "")


def mc(mono):
    return "monotone_constraints=" + ",".join(str(m) for m in mono)


def ic(cons):
    return "interaction_constraints=" + ",".join("[%s]" % ",".join(str(f) for f in c) for c in cons)


def features(ds, F, cats):
    infos = [ds.feature_info(f) for f in range(F)]
    return [ref.Feature(f, infos[f]["num_bin"], infos[f]["missing_type"], int(infos[f]["most_freq_bin"] == 0), f in cats)
            for f in range(F) if not infos[f]["is_trivial"]]


def dataset(X, cats, max_bin, extra=""):
    """what the restatement needs of X's dataset (built with ds_params and `extra`): (features, bins, upper bounds, bin-to-category
    lists)"""
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, ds_params(cats, max_bin) + " " + extra).set_field("label", np.zeros(len(X), np.float32))
    try:
        feats = features(ds, X.shape[1], cats)
        return (feats, ds.get_bins16(), {f.real_index: ds.upper_bounds(f.real_index) for f in feats},
                {f.real_index: ds.bin_to_cat(f.real_index) for f in feats if f.is_cat})
    finally:
        ds.free()


def run(X, g, h, params, iters, ds_params, reset=None, label=None):
    """the model text of `iters` trees on the same custom (g, h); reset = (after tree k, parameter string) calls ResetParameter; label:
    the dataset's labels (zeros by default; multiclass needs every class present, or no class trains)"""
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, ds_params).set_field("label", np.zeros(len(X), np.float32) if label is None else np.asarray(label, np.float32))
    b = capi.Booster(ds, params)
    try:
        for k in range(iters):
            b.update_one_iter_custom(g.astype(np.float32), h.astype(np.float32))
            if reset is not None and reset[0] == k:
                b.reset_parameter(reset[1])
        return b.save_model_to_string()
    finally:
        b.free(); ds.free()


def trees(model):
    return model.split("\nparameters:")[0]


def split_features(model):
    from mmlspark_b200.modeltext import parse_model
    return {int(f) for t in parse_model(model)["trees"] for f in t["split_feature"]} if "split_feature=" in model else set()


def paths_inside(model, cons):
    """the number of root-to-leaf paths of the model that leave every set of `cons`"""
    from mmlspark_b200.modeltext import parse_model
    bad = 0
    for t in parse_model(model)["trees"]:
        for path in I.leaf_paths(t):
            bad += not any(set(path) <= set(c) for c in cons)
    return bad


def ulps(a, b):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) / np.spacing(np.maximum(np.abs(a), np.abs(b)) + 1e-300)


def compare_tree(t, T, ub, b2c, lr=None):
    """the engine's tree t (parse_model) against tree_ref's T at the bar above; ub / b2c: the dataset's upper bounds and bin-to-category
    lists per real feature; lr: the learning rate that shrank t's leaf values"""
    assert t["num_leaves"] == T["num_leaves"], "num_leaves %d vs reference %d" % (t["num_leaves"], T["num_leaves"])
    nl = T["num_leaves"]
    if nl > 1:
        assert t["split_feature"].tolist() == T["split_feature"], (t["split_feature"], T["split_feature"])
        assert t["left_child"].tolist() == T["left_child"] and t["right_child"].tolist() == T["right_child"]
        for i in range(nl - 1):
            f, dt = T["split_feature"][i], int(t["decision_type"][i])
            assert bool(dt & 1) == T["is_cat"][i], "node %d: categorical flag" % i
            if T["is_cat"][i]:
                k = int(t["threshold"][i])
                words = t["cat_threshold"][t["cat_boundaries"][k]:t["cat_boundaries"][k + 1]]
                cats = {32 * w + j for w, word in enumerate(words) for j in range(32) if (int(word) >> j) & 1}
                got = {b for b, c in enumerate(b2c[f]) if b > 0 and c in cats}
                assert got == set(T["cat_bins"][i]), "node %d: category bins %s vs reference %s" % (i, sorted(got), sorted(T["cat_bins"][i]))
            else:
                hit = np.nonzero(ub[f] == t["threshold"][i])[0]
                assert len(hit) == 1, "node %d: threshold %r is not exactly one upper bound" % (i, t["threshold"][i])
                assert hit[0] == T["threshold_bin"][i], "node %d: threshold bin %d vs reference %d" % (i, hit[0], T["threshold_bin"][i])
                assert bool(dt & 2) == T["default_left"][i], "node %d: default_left" % i
            assert t["split_gain"][i] == float("%g" % T["split_gain"][i]), "node %d: split_gain %r vs %g" % (i, t["split_gain"][i], T["split_gain"][i])
        assert t["leaf_count"].tolist() == T["leaf_count"] and t["internal_count"].tolist() == T["internal_count"]
        assert (ulps(t["leaf_weight"], T["leaf_weight"]) <= 4).all(), (t["leaf_weight"], T["leaf_weight"])
        assert t["internal_weight"].tolist() == [float("%g" % v) for v in T["internal_weight"]], (t["internal_weight"], T["internal_weight"])
        if lr is None:
            assert t["internal_value"].tolist() == [float("%g" % v) for v in T["internal_value"]], (t["internal_value"], T["internal_value"])
        else:       # shrunk as the leaf values are, then printed with %g's 6 digits
            np.testing.assert_allclose(t["internal_value"], np.asarray(T["internal_value"]) * lr, rtol=1e-5, atol=1e-300)
    if lr is None:
        assert (ulps(t["leaf_value"], T["leaf_value"]) <= 4).all(), (t["leaf_value"], T["leaf_value"])
    else:
        np.testing.assert_allclose(t["leaf_value"], np.asarray(T["leaf_value"]) * lr, rtol=1e-12, atol=1e-300)


def check_run(X, g, h, cats, num_leaves, iters, max_bin=255, extra="", extra_seed=None, fraction=1.0, mono=None, penalty=0.0, cons=None,
              bynode=None, max_depth=-1, reset=None, dropped=()):
    """`iters` iterations on the same custom (g, h), every tree against tree_ref.grow_tree with the same options, carried from tree to
    tree; returns the model text and the restated trees.
    - extra: more parameters, the split-scan ones (split_scan_ref.Params) also the restatement's; extra_seed: extra_trees on;
      fraction: feature_fraction; mono, penalty: monotone constraints; cons: interaction constraints (every path of the model must stay
      inside one set); bynode: feature_fraction_bynode; max_depth.
    - reset = (after tree k, parameter string) calls ResetParameter: it re-seeds every extra-trees stream, and a monotone_constraints
      list in it replaces `mono`.
    - dropped: the iterations whose tree has one leaf, which the booster does not keep (GBDT::TrainOneIter)."""
    from mmlspark_b200.modeltext import parse_model
    opts = extra
    if extra_seed is not None:
        opts += " extra_trees=true extra_seed=%d" % extra_seed
    if fraction < 1.0:
        opts += " feature_fraction=%r" % fraction
    if mono is not None:
        opts += " %s monotone_penalty=%r" % (mc(mono), penalty)
    if cons is not None:
        opts += " " + ic(cons)
    if bynode is not None:
        opts += " feature_fraction_bynode=%r" % bynode
    if max_depth > 0:
        opts += " max_depth=%d" % max_depth
    model = run(X, g, h, params(num_leaves, opts, cats, max_bin), iters, ds_params(cats, max_bin), reset)
    feats, bins, ub, b2c = dataset(X, cats, max_bin)
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(min_data_in_leaf=20, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS})
    trees = parse_model(model)["trees"] if "Tree=" in model else []
    assert len(trees) == iters - len(dropped)
    kept = iter(trees)
    sampler = B.ColSampler(feats, fraction, bynode) if bynode is not None else None
    used = X3.feature_fraction_sets(len(feats), fraction, 2, iters)
    streams = X3.Streams(feats, extra_seed) if extra_seed is not None else None
    Ts = []
    for k in range(iters):
        if reset is not None and k == reset[0] + 1:
            streams = X3.Streams(feats, extra_seed) if extra_seed is not None else None
            kv = dict(tok.split("=", 1) for tok in reset[1].split())
            if "monotone_constraints" in kv:
                mono = [int(m) for m in kv["monotone_constraints"].split(",")]
        T = tree_ref.grow_tree(bins, g, h, feats, p, num_leaves, used=None if sampler is not None else {feats[i].real_index for i in used[k]},
                               streams=streams, mono=mono, penalty=penalty, constraints=cons, sampler=sampler, max_depth=max_depth)
        why = ref.undecided(T)
        assert not why, "tree %d does not discriminate:\n%s" % (k, "\n".join(why[:10]))
        Ts.append(T)
        if k in dropped:
            assert T["num_leaves"] == 1
            continue
        t = next(kept)
        compare_tree(t, T, ub, b2c)
        for path in I.leaf_paths(t) if cons is not None else ():
            assert any(set(path) <= set(c) for c in cons), (k, path)
    return model, Ts


def on_ranks(R, base_port, body, device_of=lambda r: 0, timeout=120):
    """body(r) on R rank-threads of this process, rank r on device_of(r), between network_init and network_free (in finally; one rank
    needs no network).  Returns the bodies' results and the (rank, error) pairs."""
    from mmlspark_b200 import capi
    machines = ",".join("127.0.0.1:%d" % (base_port + r) for r in range(R))
    out, errs = [None] * R, []

    def task(r):
        try:
            capi.set_device(device_of(r))
            if R == 1:
                out[r] = body(r)
                return
            capi.network_init(machines, base_port + r, timeout, R)
            try:
                out[r] = body(r)
            finally:
                capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, str(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(R)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(300)
    assert not any(t.is_alive() for t in ts), "a rank-thread did not finish"
    return out, errs


def boost(X, y, params, iters, dsp, group=None, rank_rows=None, port=None, grads=False):
    """trains `iters` iterations on the objective's own gradients; rank_rows: data-parallel shards, each rank a thread on this device
    (every rank's model must be equal).  Returns the model text, or with `grads` (model, per iteration the gradients of all rows read back
    before it, whether the hessian is constant)."""
    from mmlspark_b200 import capi
    rank_rows = rank_rows or [len(X)]
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        full = capi.Dataset.from_mat(X, dsp)
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=full).set_field("label", np.asarray(y[sl], np.float32))
        if group is not None:
            ds.set_field("group", np.asarray(group, np.int32))
        b = capi.Booster(ds, params)
        try:
            seen = []
            for _ in range(iters):
                if grads:
                    seen.append(b.get_gradients())
                b.update_one_iter()
            return b.save_model_to_string(), seen, b.get_info()["constant_hessian"]
        finally:
            b.free(); ds.free(); full.free()

    if len(rank_rows) == 1:
        res = [body(0)]
    else:
        res, errs = on_ranks(len(rank_rows), port, body)
        assert not errs, errs
        assert all(trees(r[0]) == trees(res[0][0]) for r in res)
    if not grads:
        return res[0][0]
    seen = [(np.concatenate([r[1][it][0] for r in res]), np.concatenate([r[1][it][1] for r in res])) for it in range(iters)]
    if len(rank_rows) > 1:      # class-major per rank: regroup per class over all rows
        K = len(res[0][1][0][0]) // rank_rows[0]
        seen = [tuple(np.concatenate([r[1][it][j].reshape(K, -1) for r in res], axis=1).reshape(-1) for j in (0, 1)) for it in range(iters)]
    return res[0][0], seen, res[0][2]


def quantized(v):
    """K3's fixed-point grid: q = rint(v * 2^e), e = 34 - ilogb(max |v|) over every rank's rows; the histograms are exact sums of q, so
    NumPy's fp64 sums of q * 2^-e equal the engine's int64 ones"""
    m = np.float32(np.max(np.abs(v)))
    e = 34 - (int(np.frexp(m)[1]) - 1) if m > 0 and np.isfinite(m) else 0
    return np.rint(v.astype(np.float64) * 2.0 ** e) * 2.0 ** -e


def lcg_next(x):
    """LightGBM's Random: x <- 214013 x + 2531011 (mod 2^32); returns (x, float draw ((x >> 16) & 0x7fff) / 32768)"""
    x = (x * np.uint64(214013) + np.uint64(2531011)) & np.uint64(0xFFFFFFFF)
    return x, ((x >> np.uint64(16)) & np.uint64(0x7FFF)).astype(np.float64) / 32768.0


def bags(n, iters, fraction, seed, freq=1, label=None, pos=1.0, neg=1.0):
    """GBDT::Bagging on one rank: per 1024-row block an LCG seeded seed + block, row j of a block takes the next draw < its fraction:
    `fraction`, or with `label` (balanced bagging) `pos` where label > 0 and `neg` elsewhere.  The first draw is at iteration 0, the next
    ones at it % freq == 0; in between the bag and the states stay.  The states carry over to the next draw."""
    blocks = (n + 1023) // 1024
    x = np.arange(blocks, dtype=np.uint64) + np.uint64(seed)
    frac = np.full(blocks * 1024, fraction, np.float64)
    if label is not None:
        frac[:n] = np.where(np.asarray(label) > 0, pos, neg)
    out = []
    for it in range(iters):
        if it > 0 and it % freq != 0:
            out.append(out[-1])
            continue
        take = np.zeros(blocks * 1024, bool)
        for j in range(1024):
            live = j < n - np.arange(blocks) * 1024
            nx, draw = lcg_next(x)
            x = np.where(live, nx, x)
            at = np.arange(blocks) * 1024 + j
            take[at] = live & (draw < frac[at])
        out.append(take[:n])
    return out
