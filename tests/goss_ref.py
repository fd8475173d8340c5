"""NumPy restatement of the GOSS sample as the engine draws it (kernels.cuh k_goss_draw): LightGBM 3.2's GOSS::BaggingHelper applied to
every rank-local block of 1024 rows.  Upstream's blocks depend on the thread count; the engine fixes them at 1024 rows, the size of its
bagging blocks, so that a sample does not depend on the machine.  It imports neither mmlspark_b200 nor oracle.

Per block of cnt rows, with its own LCG (tree_check.lcg_next) seeded bagging_seed + block:
- tg of a row is the float32 sum, in class order, of |float32(g * h)| over the classes;
- top_k = max(1, int(cnt * top_rate)), other_k = int(cnt * other_rate), threshold = the top_k-th largest tg,
  multiply = float32(cnt - top_k) / other_k in float32;
- in row order, a row with tg >= threshold is kept; every other row advances the LCG once and is kept when the draw is below
  rest_need / rest_all (a double: the sample rows still wanted over the rows left that are not top rows), and then its g and h are
  multiplied by `multiply` in float32 for every class.
The states carry from one draw to the next.  The first int(1 / learning_rate) iterations draw nothing and train on every row."""
import numpy as np

from tree_check import lcg_next

BLOCK = 1024


def seeds(n, seed):
    """the block states of n rank-local rows before the first draw"""
    return np.arange((n + BLOCK - 1) // BLOCK, dtype=np.uint64) + np.uint64(seed)


def warm_up(learning_rate):
    """the iterations that draw nothing: it < int(1.0f / learning_rate), a double quotient"""
    return int(1.0 / learning_rate)


def block_draw(g, h, x, top_rate, other_rate):
    """one block: g, h float32 [K][cnt]; x its LCG state.  Returns (flag per row: 0 out, 1 top, 2 sampled; multiply; new state)."""
    K, cnt = g.shape
    tg = np.zeros(cnt, np.float32)
    for k in range(K):
        tg = (tg + np.abs(g[k] * h[k])).astype(np.float32)
    top_k = max(1, int(cnt * top_rate))
    other_k = int(cnt * other_rate)
    with np.errstate(divide="ignore"):
        multiply = np.float32(cnt - top_k) / np.float32(other_k)
    threshold = np.sort(tg)[::-1][top_k - 1]
    flag = np.zeros(cnt, np.int8)
    left = big = 0
    x = np.uint64(x)
    for i in range(cnt):
        if tg[i] >= threshold:
            flag[i] = 1
            left += 1
            big += 1
            continue
        rest_need = other_k - (left - big)
        rest_all = (cnt - i) - (top_k - big)
        x, draw = lcg_next(x)
        if draw < rest_need / rest_all:
            flag[i] = 2
            left += 1
    return flag, multiply, x


def draw(g, h, states, top_rate, other_rate):
    """one GOSS draw over a rank's rows: g, h float32 [K][n] (class-major); states from seeds() or the previous draw.
    Returns (in-bag mask, amplified g, amplified h, new states)."""
    g = np.array(g, np.float32, copy=True)
    h = np.array(h, np.float32, copy=True)
    n = g.shape[1]
    states = np.array(states, np.uint64, copy=True)
    bag = np.zeros(n, bool)
    for b in range(len(states)):
        sl = slice(b * BLOCK, min(n, (b + 1) * BLOCK))
        flag, multiply, states[b] = block_draw(g[:, sl], h[:, sl], states[b], top_rate, other_rate)
        bag[sl] = flag > 0
        amp = np.nonzero(flag == 2)[0] + b * BLOCK
        g[:, amp] = (g[:, amp] * multiply).astype(np.float32)
        h[:, amp] = (h[:, amp] * multiply).astype(np.float32)
    return bag, g, h, states


def ranks_draw(g, h, states, rank_rows, top_rate, other_rate):
    """draw() on every rank's shard of the columns (rank_rows rows each, in rank order); states: one array per rank"""
    offs = np.concatenate([[0], np.cumsum(rank_rows)]).astype(int)
    out = [draw(g[:, offs[r]:offs[r + 1]], h[:, offs[r]:offs[r + 1]], states[r], top_rate, other_rate) for r in range(len(rank_rows))]
    return (np.concatenate([o[0] for o in out]), np.concatenate([o[1] for o in out], axis=1), np.concatenate([o[2] for o in out], axis=1),
            [o[3] for o in out])
