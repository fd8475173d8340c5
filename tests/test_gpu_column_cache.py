"""The partition kernel's column cache: when the full column-major copy of the training tiles does not fit, the booster keeps a pool of
column slots and fills it, between trees, with the storage columns the trees split on (B200GBM_COLUMN_CACHE_COLUMNS=k forces this mode
with at most k slots).  Which columns are cached only changes where k_partition reads a bin, so the models must be identical byte for
byte with the full copy, with no copy and with any slot budget, and the cache must build and evict exactly as its policy says."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0 categorical_feature=3"
PARAMS = ("objective=binary metric= num_leaves=63 learning_rate=0.1 min_data_in_leaf=20 feature_fraction=0.3 verbosity=-1 "
          "max_bin=255 num_threads=0")
N, ITERS, STRIDE = 70_001, 10, 70_144            # two tiles, the second partly filled; 256-row column stride
BUILDS_PER_TREE = 8                              # kColumnBuildsMax in kernels.cuh


def data(n=N, seed=91):
    """37 dense features (3: categorical, 5: 5 % NaN) and a mutually exclusive sparse pair 37/38 that shares one storage column"""
    rng = np.random.default_rng(seed)
    X = np.zeros((n, 39))
    X[:, :37] = rng.standard_normal((n, 37))
    X[:, 3] = rng.integers(0, 30, n)
    X[rng.random(n) < 0.05, 5] = np.nan
    owner = rng.integers(0, 4, n)
    X[owner == 0, 37] = rng.integers(1, 40, (owner == 0).sum()) * 0.1      # few bins each, so that both fit one 256-bin column
    X[owner == 1, 38] = rng.integers(1, 40, (owner == 1).sum()) * rng.choice([-0.1, 0.1], (owner == 1).sum())
    z = (X[:, 0] + np.sin(2 * X[:, 1]) + (X[:, 3] % 3) + 0.5 * X[:, 36] + 0.2 * X[:, 37] - 0.2 * X[:, 38]
         + 0.4 * X[:, 7:20].sum(axis=1) + 0.3 * rng.standard_normal(n))
    return X, (z > 1.0).astype(np.float32)


def split_columns(model_text, column_of):
    """storage columns of the splits of every tree, in training order"""
    trees = []
    for block in model_text.split("\nTree=")[1:]:
        line = next((l for l in block.split("\n") if l.startswith("split_feature=")), None)
        trees.append([int(column_of[int(f)]) for f in line.split("=")[1].split()] if line else [])
    return trees


def simulate(trees, slots):
    """the cache policy of Booster::UpdateColumnCache: (columns built, evictions)"""
    counts, slot_col, cached = {}, [-1] * slots, set()
    builds = evictions = 0
    for cols in trees:
        for c in cols:
            counts[c] = counts.get(c, 0) + 1
        made = 0
        for c in sorted((c for c in counts if c not in cached), key=lambda c: (-counts[c], c)):
            if made == BUILDS_PER_TREE:
                break
            if -1 in slot_col:
                s = slot_col.index(-1)
            else:
                s = min(range(slots), key=lambda s: counts[slot_col[s]])
                if counts[slot_col[s]] >= counts[c]:
                    break
                cached.discard(slot_col[s])
                evictions += 1
            slot_col[s] = c
            cached.add(c)
            builds += 1
            made += 1
    return builds, evictions


def _train(capi, X, y, monkeypatch, env, params=PARAMS):
    monkeypatch.delenv("B200GBM_COLUMN_COPY", raising=False)
    monkeypatch.delenv("B200GBM_COLUMN_CACHE_COLUMNS", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ds = capi.Dataset.from_mat(X, DS_PARAMS)
    ds.set_field("label", y)
    b = capi.Booster(ds, params)
    for _ in range(ITERS):
        assert not b.update_one_iter()
    out = dict(text=b.save_model_to_string(), copy=b.get_memory_info()["partition_column_copy_bytes"], cache=b.get_column_cache_info(),
               bundles=ds.bundles())
    b.free(); ds.free()
    return out


def test_column_cache_is_transparent(built, monkeypatch):
    """full copy, no copy, and the cache at 0, 1 and 3 slots: identical models, matching the oracle; the pool size is what the
    memory info reports, and the builds and evictions are the policy's"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    X, y = data()
    runs = {name: _train(capi, X, y, monkeypatch, env) for name, env in (
        ("full", {}), ("none", {"B200GBM_COLUMN_COPY": "0"}), ("k0", {"B200GBM_COLUMN_CACHE_COLUMNS": "0"}),
        ("k1", {"B200GBM_COLUMN_CACHE_COLUMNS": "1"}), ("k3", {"B200GBM_COLUMN_CACHE_COLUMNS": "3"}))}
    ncols, column_of = runs["full"]["bundles"]
    assert ncols == 38 and column_of[37] == column_of[38], column_of      # the sparse pair is one bundle column
    for name, r in runs.items():
        assert r["text"] == runs["full"]["text"], name
    assert runs["full"]["copy"] == 2 * 32 * STRIDE and runs["full"]["cache"]["slots"] == 0
    assert runs["none"]["copy"] == 0 and runs["k0"]["copy"] == 0 and runs["k0"]["cache"]["slots"] == 0
    trees = split_columns(runs["full"]["text"], column_of)
    assert any(column_of[37] in t for t in trees)                             # the bundle column is split on, and so cached
    for k in (1, 3):
        r = runs["k%d" % k]
        assert r["copy"] == k * STRIDE and r["cache"]["slots"] == k and r["cache"]["slots_used"] == k
        assert (r["cache"]["builds"], r["cache"]["evictions"]) == simulate(trees, k), (k, r["cache"])
    assert runs["k1"]["cache"]["evictions"] > 0 and runs["k1"]["cache"]["builds"] > 1      # evicted and rebuilt
    ods = O.OracleDataset(X, DS_PARAMS)
    ods.set_field("label", y)
    ob = O.OracleBooster(ods, PARAMS)
    ob.train(ITERS)
    compare_models(parse_model(runs["k1"]["text"]), parse_model(ob.model_string()))


def test_column_cache_builds_bounded_per_tree(built, monkeypatch):
    """a pool larger than the columns split on: every split-on column is cached once and never evicted, at most 8 builds per tree
    (the first tree, on every feature, splits on more than 8 columns)"""
    from mmlspark_b200 import capi
    X, y = data()
    r = _train(capi, X, y, monkeypatch, {"B200GBM_COLUMN_CACHE_COLUMNS": "64"}, PARAMS.replace("feature_fraction=0.3", "feature_fraction=1.0"))
    ncols, column_of = r["bundles"]
    trees = split_columns(r["text"], column_of)
    split_on = len({c for t in trees for c in t})
    assert r["cache"]["slots"] == ncols and r["copy"] == ncols * STRIDE       # capped at the number of storage columns
    assert r["cache"]["evictions"] == 0 and r["cache"]["builds"] == r["cache"]["slots_used"]
    assert (r["cache"]["builds"], 0) == simulate(trees, ncols)
    assert len(set(trees[0])) > BUILDS_PER_TREE and r["cache"]["builds"] == split_on


RANK_SCRIPT = r"""
import hashlib, json, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_gpu_column_cache as T
from mmlspark_b200 import capi
r, port = int(sys.argv[1]), int(sys.argv[2])
capi.set_device(r)
capi.network_init("127.0.0.1:%d,127.0.0.1:%d" % (port, port + 1), port + r, 120, 2)
X, y = T.data()
half = len(X) // 2
ds = capi.Dataset.from_mat(X[r * half:(r + 1) * half], T.DS_PARAMS)
ds.set_field("label", y[r * half:(r + 1) * half])
b = capi.Booster(ds, T.PARAMS + " tree_learner=data num_machines=2")
for _ in range(T.ITERS):
    b.update_one_iter()
text = b.save_model_to_string().split("\nparameters:")[0]
print(json.dumps(dict(hash=hashlib.sha256(text.encode()).hexdigest(), cache=b.get_column_cache_info())))
b.free(); ds.free()
capi.network_free()
"""


def _ngpu():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return len([l for l in out.splitlines() if l.startswith("GPU ")])
    except Exception:
        return 0


def _two_ranks(envs, port):
    import json
    script = RANK_SCRIPT.format(root=ROOT, tests=os.path.dirname(os.path.abspath(__file__)))
    procs = []
    for r, extra in enumerate(envs):
        env = {k: v for k, v in os.environ.items() if k not in ("B200GBM_COLUMN_COPY", "B200GBM_COLUMN_CACHE_COLUMNS")}
        env.update(extra)
        procs.append(subprocess.Popen([sys.executable, "-c", script, str(r), str(port)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.PIPE, text=True))
    outs = []
    for p in procs:
        so, se = p.communicate(timeout=300)
        assert p.returncode == 0, se[-2000:]
        outs.append(json.loads(so.strip().splitlines()[-1]))
    return outs


def test_two_ranks_with_different_budgets(built):
    """data-parallel, one process per GPU: rank 0 caches 1 column, rank 1 keeps the full copy; the model equals the one trained
    without any copy"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    a = _two_ranks([{"B200GBM_COLUMN_CACHE_COLUMNS": "1"}, {}], 23640)
    b = _two_ranks([{"B200GBM_COLUMN_COPY": "0"}, {"B200GBM_COLUMN_COPY": "0"}], 23660)
    assert a[0]["cache"]["slots"] == 1 and a[0]["cache"]["builds"] > 0 and a[1]["cache"]["slots"] == 0
    assert a[0]["hash"] == a[1]["hash"] == b[0]["hash"] == b[1]["hash"]
