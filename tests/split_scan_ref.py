"""Plain NumPy/fp64 restatement of LightGBM 3.2's split search, used to pin the engine's scan kernels (K5/K6: k_scan, k_scan_wide)
and the pick step (d_pick_block / d_choose_leaf) tree by tree.  It imports neither mmlspark_b200 nor oracle.

Restated from LightGBM 3.2 (FeatureHistogram, SerialTreeLearner):
- FindBestThresholdNumerical: the reverse pass, the NaN-as-missing forward pass (incl. the implicit bin 0 when offset == 1) and
  default_left; `continue` and `break` where FindBestThresholdSequentially uses them; counts rebuilt from hessians as
  RoundInt(h * num_data / (sum_h + 2 kEpsilon)).
- GetLeafGain / CalculateSplittedLeafOutput: L1 soft threshold, L2, max_delta_step; min_gain_shift.
- FindBestThresholdCategorical: one-hot, and many-vs-many over the bins with >= cat_smooth rebuilt rows, stably sorted by
  g / (h + cat_smooth) and walked from both ends; cat_l2 enters the gains and leaf outputs but not min_gain_shift.
- The feature choice per leaf (gain, then smaller real feature index) and the row partition of a split; tree_ref.py grows the trees
  from them (the leaf choice, child sums taken from the split, is_splittable inheritance).

Histograms are sums of values on a fixed-point grid, so every bin and prefix sum is exact in fp64 and kEpsilon is added once to an exact
sum, as the engine's int64 histograms do.  (Upstream accumulates kEpsilon + h_1 + h_2 + ... in fp64; that differs only in the rounding of
kEpsilon, far below the 1e-12 margin the tests require between competing gains.)  The many-vs-many walk sums bins in its own order in
fp64, as upstream and the engine do.

Every scan also reports what a comparison needs to know whether its result is *decided*: all candidates with their gains and fp64 sums,
min_gain_shift, and the distance of every rebuilt count from a .5 rounding boundary."""
import math

import numpy as np

K_EPS = 1e-15
K_ZERO = 1e-35              # Tree::Shrinkage / AddBias round |x| <= kZeroThreshold to 0
NEG_INF = -math.inf


class Params:
    DEFAULTS = dict(lambda_l1=0.0, lambda_l2=0.0, max_delta_step=0.0, min_gain_to_split=0.0, min_sum_hessian_in_leaf=1e-3,
                    min_data_in_leaf=20, cat_l2=10.0, cat_smooth=10.0, max_cat_threshold=32, max_cat_to_onehot=4, min_data_per_group=100)

    def __init__(self, **kw):
        unknown = set(kw) - set(self.DEFAULTS)
        assert not unknown, unknown
        for k, v in self.DEFAULTS.items():
            setattr(self, k, type(v)(kw.get(k, v)))

    def as_string(self):
        return " ".join("%s=%r" % (k, getattr(self, k)) for k in self.DEFAULTS)


def round_int(x):
    """Common::RoundInt: static_cast<int>(x + 0.5), i.e. truncation toward zero (negative hessians give negative counts)."""
    return int(x + 0.5)


def half_margin(x):
    """distance of x from the nearest k + 0.5 (where RoundInt changes)"""
    return abs((x - math.floor(x)) - 0.5)


def _sign(x):
    return (x > 0) - (x < 0)


def _threshold_l1(s, l1):
    return _sign(s) * max(0.0, abs(s) - l1)


def calc_output(g, h, p, l2):
    """CalculateSplittedLeafOutput (no monotone constraints, no path smoothing)"""
    ret = -_threshold_l1(g, p.lambda_l1) / (h + l2) if p.lambda_l1 > 0 else -g / (h + l2)
    if p.max_delta_step > 0 and abs(ret) > p.max_delta_step:
        ret = _sign(ret) * p.max_delta_step
    return ret


def leaf_gain(g, h, p, l2):
    """GetLeafGain"""
    if not p.max_delta_step > 0:
        sg = _threshold_l1(g, p.lambda_l1) if p.lambda_l1 > 0 else g
        return (sg * sg) / (h + l2)
    out = calc_output(g, h, p, l2)
    sg = _threshold_l1(g, p.lambda_l1) if p.lambda_l1 > 0 else g
    return -(2.0 * sg * out + (h + l2) * out * out)


class Scan:
    """Result of one (leaf, feature) search.  gain = best gain - min_gain_shift (-inf if none); left_h keeps its +kEpsilon."""

    def __init__(self, feature, shift):
        self.feature, self.shift = feature, shift
        self.gain, self.splittable = NEG_INF, False
        self.threshold, self.default_left, self.is_cat, self.cat_bins = 0, True, False, ()
        self.left_g = self.left_h = 0.0
        self.left_count, self.l2 = 0, 0.0
        self.candidates = []      # (gain, left_g, left_h, right_g, right_h, tag) of every candidate that passed the count/hessian tests
        self.margins = []         # half_margin of every rebuilt count the scan used
        self.win = None          # the winning entry of `candidates`

    def _offer(self, gain, lg, lh, rg, rh, tag):
        self.candidates.append((gain, lg, lh, rg, rh, tag))
        return self.candidates[-1]


def find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature=0):
    """hg/hh: per-bin sums indexed by bin (bin 0's entry is ignored when offset == 1, as upstream does not store it).
    missing_type: 0 none, 2 NaN (the NaN bin is num_bin - 1)."""
    sum_h = sum_h_in + 2 * K_EPS
    cnt_factor = num_data / sum_h
    l2 = p.lambda_l2
    shift = leaf_gain(sum_g, sum_h, p, l2) + p.min_gain_to_split
    r = Scan(feature, shift)
    r.l2 = l2
    xs = [float(hh[b]) * cnt_factor for b in range(num_bin)]
    cnt = [round_int(x) for x in xs]
    r.margins = [half_margin(x) for x in xs]
    two_way = num_bin > 2 and missing_type == 2
    na = 1 if two_way else 0
    best = None                  # (gain, threshold, lg, lh, lc, default_left, candidate)
    # reverse pass: bins num_bin-1-na .. 1, threshold b - 1
    rg, rh, rc = 0.0, 0.0, 0
    for b in range(num_bin - 1 - na, 0, -1):
        rg += float(hg[b]); rh += float(hh[b]); rc += cnt[b]
        srh = K_EPS + rh
        if rc < p.min_data_in_leaf or srh < p.min_sum_hessian_in_leaf:
            continue
        lc = num_data - rc
        slh = sum_h - srh
        if lc < p.min_data_in_leaf or slh < p.min_sum_hessian_in_leaf:
            break
        slg = sum_g - rg
        gain = leaf_gain(slg, slh, p, l2) + leaf_gain(rg, srh, p, l2)
        c = r._offer(gain, slg, slh, rg, srh, ("rev", b - 1))
        if gain <= shift:
            continue
        r.splittable = True
        if best is None or gain > best[0]:
            best = (gain, b - 1, slg, slh, lc, True, c)
    if two_way:
        # forward pass: thresholds 0 .. num_bin-2, the NaN bin goes right
        if offset == 1:          # implicit bin 0 = leaf total - every stored bin (incl. the NaN bin)
            base_g = sum_g - math.fsum(float(hg[b]) for b in range(1, num_bin))
            base_h = (sum_h - K_EPS) - math.fsum(float(hh[b]) for b in range(1, num_bin))
            base_c = num_data - sum(cnt[1:num_bin])
        else:
            base_g, base_h, base_c = 0.0, K_EPS, 0
        pg, ph, pc = 0.0, 0.0, 0
        fbest = None
        for b in range(0, num_bin - 1):
            if b >= offset:
                pg += float(hg[b]); ph += float(hh[b]); pc += cnt[b]
            slg, slh, lc = base_g + pg, base_h + ph, base_c + pc
            if lc < p.min_data_in_leaf or slh < p.min_sum_hessian_in_leaf:
                continue
            rc = num_data - lc
            srh = sum_h - slh
            if rc < p.min_data_in_leaf or srh < p.min_sum_hessian_in_leaf:
                break
            srg = sum_g - slg
            gain = leaf_gain(slg, slh, p, l2) + leaf_gain(srg, srh, p, l2)
            c = r._offer(gain, slg, slh, srg, srh, ("fwd", b))
            if gain <= shift:
                continue
            r.splittable = True
            if fbest is None or gain > fbest[0]:
                fbest = (gain, b, slg, slh, lc, False, c)
        if fbest is not None and (best is None or fbest[0] > best[0]):      # only a strictly larger gain replaces the reverse result
            best = fbest
    if r.splittable and best[0] > shift:
        r.gain = best[0] - shift
        _, r.threshold, r.left_g, r.left_h, r.left_count, r.default_left, r.win = best
    if not two_way and missing_type == 2:
        r.default_left = False
    return r


def find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature=0):
    """Bins 1 .. num_bin-1 are categories; bin 0 (NaN, negative and unseen categories) always goes right."""
    sum_h = sum_h_in + 2 * K_EPS
    cnt_factor = num_data / sum_h
    shift = leaf_gain(sum_g, sum_h, p, p.lambda_l2) + p.min_gain_to_split
    r = Scan(feature, shift)
    r.is_cat, r.default_left = True, False
    xs = [float(hh[b]) * cnt_factor for b in range(num_bin)]
    cnt = [round_int(x) for x in xs]
    r.margins = [half_margin(x) for x in xs[1:]]
    best = None                  # (gain, bins, lg, lh, lc)
    if num_bin <= p.max_cat_to_onehot:
        l2 = p.lambda_l2
        for b in range(1, num_bin):
            g, h, c = float(hg[b]), float(hh[b]), cnt[b]
            if c < p.min_data_in_leaf or h < p.min_sum_hessian_in_leaf:
                continue
            if num_data - c < p.min_data_in_leaf:
                continue
            oh = sum_h - h - K_EPS
            if oh < p.min_sum_hessian_in_leaf:
                continue
            gain = leaf_gain(sum_g - g, oh, p, l2) + leaf_gain(g, h + K_EPS, p, l2)
            cand = r._offer(gain, g, h + K_EPS, sum_g - g, oh, ("onehot", b))
            if gain <= shift:
                continue
            r.splittable = True
            if best is None or gain > best[0]:
                best = (gain, (b,), g, h + K_EPS, c, cand)
    else:
        l2 = p.lambda_l2 + p.cat_l2
        used = [b for b in range(1, num_bin) if cnt[b] >= p.cat_smooth]
        order = sorted(used, key=lambda b: (float(hg[b]) / (float(hh[b]) + p.cat_smooth), b))     # stable sort by ctr
        max_num_cat = min(p.max_cat_threshold, (len(used) + 1) // 2)
        for d, seq in ((1, order), (-1, order[::-1])):
            slg, slh, lc, grp = 0.0, K_EPS, 0, 0
            for i in range(min(len(used), max_num_cat)):
                t = seq[i]
                slg += float(hg[t]); slh += float(hh[t]); lc += cnt[t]; grp += cnt[t]
                if lc < p.min_data_in_leaf or slh < p.min_sum_hessian_in_leaf:
                    continue
                rc = num_data - lc
                if rc < p.min_data_in_leaf or rc < p.min_data_per_group:
                    break
                srh = sum_h - slh
                if srh < p.min_sum_hessian_in_leaf:
                    break
                if grp < p.min_data_per_group:
                    continue
                grp = 0
                gain = leaf_gain(slg, slh, p, l2) + leaf_gain(sum_g - slg, srh, p, l2)
                cand = r._offer(gain, slg, slh, sum_g - slg, srh, ("dir%+d" % d, i))
                if gain <= shift:
                    continue
                r.splittable = True
                if best is None or gain > best[0]:
                    best = (gain, tuple(seq[:i + 1]), slg, slh, lc, cand)
    r.l2 = l2
    if r.splittable:
        r.gain = best[0] - shift
        _, bins, r.left_g, r.left_h, r.left_count, r.win = best
        r.cat_bins = tuple(sorted(bins))
    return r


def better_split(a_gain, a_feat, b_gain, b_feat):
    """SplitInfo::operator> on (gain, real feature index); a feature of -1 ranks last"""
    fa = a_feat if a_feat >= 0 else 1 << 31
    fb = b_feat if b_feat >= 0 else 1 << 31
    return a_gain > b_gain or (a_gain == b_gain and fa < fb)


class Feature:
    def __init__(self, real_index, num_bin, missing_type=0, offset=0, is_cat=False):
        self.real_index, self.num_bin, self.missing_type, self.offset, self.is_cat = real_index, num_bin, missing_type, offset, is_cat


def best_of_leaf(scans):
    best = None
    for fi in sorted(scans):
        s = scans[fi]
        if s.gain == NEG_INF:
            continue
        if best is None or better_split(s.gain, fi, best.gain, best.feature):
            best = s
    return best


def goes_left(col, f, s):
    """row partition of a split on feature f (bins of its rows in col)"""
    if s.is_cat:
        return np.isin(col, np.asarray(s.cat_bins))
    left = col <= s.threshold
    if f.missing_type == 2:
        left = np.where(col == f.num_bin - 1, s.default_left, left)
    return left


def undecided(T, rel=1e-12, count_margin=1e-9):
    """Reasons the reference's result could depend on rounding that another correct fp64 implementation may do differently; [] when
    every choice is decided.  A choice is decided when the winner's gain beats every other candidate (and min_gain_shift) by more than
    `rel` relative, or ties it exactly by construction: the competitor has bit-identical fp64 sums, so every implementation of the same
    formula computes the same gain.  Every rebuilt count must be further than `count_margin` from a .5 boundary."""
    why = []

    def close(a, b):
        return a != b and abs(a - b) <= rel * max(abs(a), abs(b), 1e-300)      # exactly equal is an exact tie, not a near one

    def same_sums(c, d):
        # gains depend on |g| only (L1, L2 and max_delta_step are symmetric) and add the two sides commutatively, so mirrored sums
        # and swapped sides tie exactly
        a, b = (abs(c[1]), c[2], abs(c[3]), c[4]), (abs(d[1]), d[2], abs(d[3]), d[4])
        return a == b or a == b[2:] + b[:2]

    for k, rnd in enumerate(T["rounds"]):
        last = k == len(T["rounds"]) - 1         # the flags of the last round's leaves are never read
        for l, L, scans in rnd:
            for fi, s in scans.items():
                bad = [m for m in s.margins if m <= count_margin]
                if bad:
                    why.append("leaf %d feature %d: a rebuilt count is %.3g from a .5 boundary" % (l, fi, min(bad)))
                near = [c for c in s.candidates if close(c[0], s.shift)]
                # a gain at min_gain_shift matters when it could flip the feature's splittable flag or be the winner
                if near and (s.win in near or (s.win is None and not last)):
                    why.append("leaf %d feature %d %s: gain %.17g within %g of min_gain_shift" % (l, fi, near[0][5], near[0][0], rel))
            b = L["best"]
            if b is None:
                continue
            win = b.win
            for fi, s in scans.items():
                for c in s.candidates:
                    if c is win or c[0] <= s.shift or not (close(c[0], win[0]) or c[0] == win[0]):
                        continue
                    if not same_sums(c, win):
                        why.append("leaf %d: feature %d %s ties feature %d %s (%.17g vs %.17g) with different sums" %
                                   (l, fi, c[5], b.feature, win[5], c[0], win[0]))
    for cands in T["picks"]:                # the leaf to split: ties between leaves must come from identical sums as well
        if not cands:
            continue
        top = max(cands, key=lambda c: c[1].gain)[1]
        for li, b in cands:
            if b is not top and (close(b.gain, top.gain) or b.gain == top.gain) and not same_sums(b.win, top.win):
                why.append("leaves: leaf %d's best gain %.17g ties %.17g with different sums" % (li, b.gain, top.gain))
    return why
