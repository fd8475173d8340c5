"""Plain NumPy/fp64 restatement of LightGBM 3.2's voting-parallel tree learner (VotingParallelTreeLearner, the PV-Tree algorithm) over R
row shards, built on split_scan_ref.py's scans: the rule tree_ref.grow_tree applies with `voting`.  It imports neither mmlspark_b200
nor oracle.

Per round, for each new leaf (smaller / larger by global counts):
1. every rank scans its local histogram of each of its flagged features with the local config (min_data_in_leaf // R,
   min_sum_hessian_in_leaf / R), the leaf's local sums and its true local row count; the scan sets that rank's is_splittable flags;
2. every rank sends its top_k candidates by (gain desc, real feature asc) as (feature, gain, left_count, right_count);
3. the vote, the same on every rank: mean = global count / R in fp32 (score_t); a record weighs gain * (left_count + right_count) / mean;
   each feature keeps its largest weight (strict >); the top_k features by (weight desc, feature asc) with a finite weight are voted;
4. the voted features alone are scanned on the global histogram with the training config, the leaf's global sums and its global count,
   whatever the local flags.  The best of those is the leaf's split, and the tree grows as in the data-parallel learner: the recorded
   counts are the split's hessian-rebuilt left count and the leaf's global count minus it.
One rank is the serial learner (true counts, no vote).  Local histograms are exact for every feature (upstream keeps a stale buffer for a
feature that is locally unsplittable in the parent; see DESIGN.md §5)."""
import numpy as np

import split_scan_ref as ref

NEG_INF = ref.NEG_INF


def local_params(p, R):
    q = ref.Params(**{k: getattr(p, k) for k in ref.Params.DEFAULTS})
    q.min_data_in_leaf = p.min_data_in_leaf // R
    q.min_sum_hessian_in_leaf = p.min_sum_hessian_in_leaf / R
    return q


def local_top_k(scans, top_k):
    """records (feature, gain, left_count, right_count) of the top_k candidates of one rank's scans; -inf candidates send nothing"""
    cands = sorted((s for s in scans.values() if s.gain > NEG_INF), key=lambda s: (-s.gain, s.feature))[:top_k]
    return [(s.feature, s.gain, s.left_count, s.num_data - s.left_count) for s in cands]


def vote(records, global_count, R, top_k):
    """GlobalVoting over every rank's records, in rank order: the voted features, best first"""
    mean = float(np.float32(global_count) / np.float32(R))
    best = {}
    for f, gain, lc, rc in records:
        if f < 0:
            continue
        w = gain * (lc + rc) / mean
        if w > best.get(f, NEG_INF):
            best[f] = w
    top = sorted(best.items(), key=lambda kv: (-kv[1], kv[0]))[:top_k]
    return [f for f, w in top if w > NEG_INF]
