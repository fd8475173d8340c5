"""Small end-to-end runs for compute-sanitizer (memcheck / racecheck / synccheck): every hand-synchronised kernel of the engine at shapes a
sanitizer finishes in minutes — K4 with TMA bulk copies (root) and cp.async gathers (leaves), the ticket-elected pick step of k_scan, the
software grid barriers of k_partition, the threshold selection + short bitonic sorts of k_scan_wide, the column-major copy (k_tiles_to_columns), k4_hist_wide, bagging, lambdarank, the device metrics, including the pair batches of auc_mu, and the voting-parallel chain (k_scan's local and global
modes, k_vote_pack) on two rank-threads of one device."""
import sys

import numpy as np

sys.path.insert(0, ".")
from mmlspark_b200 import capi  # noqa: E402

DS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 learning_rate=0.1 min_data_in_leaf=20 verbosity=-1 "
rng = np.random.default_rng(0)


def run(name, X, y, params, ds_params=DS, group=None, iters=2, metric=True):
    ds = capi.Dataset.from_mat(X, ds_params).set_field("label", y)
    if group is not None:
        ds.set_field("group", group)
    b = capi.Booster(ds, BASE + params)
    for _ in range(iters):
        b.update_one_iter()
    ev = b.get_eval(0) if metric else []
    print(name, "ok", len(b.save_model_to_string()), list(np.round(ev, 6)))
    b.free(); ds.free()


n, F = 40000, 70                       # 3 feature tiles, > 2^14 rows: K4 flushes mid-pass; 20 partition chunks
X = rng.standard_normal((n, F))
X[:, 3] = np.where(rng.random(n) < 0.2, np.nan, X[:, 3])
s = X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 2] * np.nan_to_num(X[:, 3]) + 0.3 * rng.standard_normal(n)
run("binary+auc", X, (s > 0).astype(np.float32), "objective=binary metric=auc,binary_logloss")
run("regression(const hessian)+bagging", X, s.astype(np.float32), "objective=regression bagging_fraction=0.5 bagging_freq=1 metric=l2")
run("multiclass", X[:15000], np.digitize(s[:15000], [-1, 0, 1]).astype(np.float32), "objective=multiclass num_class=4 metric=multi_logloss", iters=1)
sizes = rng.integers(5, 60, 400).astype(np.int32)
m = int(sizes.sum())
rel = np.clip(np.round(X[:m, 0] + 1.5), 0, 4).astype(np.float32)
run("lambdarank+ndcg", X[:m], rel, "objective=lambdarank metric=ndcg,map eval_at=1,3 min_data_in_leaf=5", group=sizes)
Xc = X[:30000].copy()
Xc[:, 5] = np.floor(3000.0 ** rng.random(30000)) - 1      # a wide categorical column (hundreds of bins)
Xc[:, 6] = rng.integers(0, 30, 30000)
yc = (s[:30000] + 0.5 * (Xc[:, 5] % 3) > 0.5).astype(np.float32)
run("wide categorical", Xc, yc, "objective=binary metric=binary_error", ds_params=DS + " categorical_feature=5,6")
# average_precision on the auc pipeline; auc_mu with 4 classes: 6 pairs hold 3n items, so several pair batches and segmented sorts run
run("binary+average_precision", X, (s > 0.5).astype(np.float32), "objective=binary metric=average_precision,auc")
yk = np.digitize(s[:15000], [-1, 0, 1]).astype(np.float32)
run("multiclass+auc_mu", X[:15000], yk, "objective=multiclass num_class=4 metric=auc_mu,multi_logloss", iters=1)
run("multiclassova+auc_mu dense matrix", X[:15000], yk,
    "objective=multiclassova num_class=4 metric=auc_mu auc_mu_weights=0,1,2,3,1,0,1,2,2,1,0,1,3,2,1,0", iters=1)


def run_voting():
    """tree_learner=voting on 2 rank-threads of this process (same-device collective): k_scan's local and global modes, the ticket-elected
    top-k step, the all-gather and k_vote_pack"""
    import threading
    Xv, yv = X[:20000], s[:20000].astype(np.float32)
    errs = []

    def task(r):
        try:
            capi.set_device(0)
            capi.network_init("127.0.0.1:31700,127.0.0.1:31701", 31700 + r, 120, 2)
            ds = capi.Dataset.from_mat(Xv[r * 10000:(r + 1) * 10000], DS).set_field("label", yv[r * 10000:(r + 1) * 10000])
            b = capi.Booster(ds, BASE + "objective=regression tree_learner=voting top_k=5 num_machines=2")
            for _ in range(2):
                b.update_one_iter()
            b.free(); ds.free()
            capi.network_free()
        except Exception as e:   # noqa
            errs.append(repr(e))
    ts = [threading.Thread(target=task, args=(r,)) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    print("voting(2 ranks, one device)", "ok" if not errs else errs)


run_voting()
print("sanitize smoke done")
