"""numpy restatements of the message-passing ops (tf_euler/kernels/gather_op.cc, scatter_op.cc, mp_ops.py) and of the dense
feature fetch, in float32 with the reference's order of operations, plus float64 restatements of their gradients.
(Test infrastructure.)"""
import numpy as np

MAX_INIT = np.float32(-1e9)   # scatter_op.cc:77-91 fills the output with -1e9
EP = np.float32(1e-7)         # scatter_mean's epsilon (mp_ops.py:65-69), added in float32


def rank_in_row(idx):
    """each edge's position among the edges of its output row, in index order"""
    idx = np.asarray(idx, np.int64)
    order = np.argsort(idx, kind="stable")
    s = idx[order]
    first = np.r_[True, s[1:] != s[:-1]] if len(s) else np.zeros(0, bool)
    start = np.maximum.accumulate(np.where(first, np.arange(len(s)), 0))
    rank = np.empty(len(idx), np.int64)
    rank[order] = np.arange(len(s)) - start
    return rank


def _serial(step, init, upd, idx, size):
    """out = init; for i in index order: out[idx[i]] = step(out[idx[i]], upd[i]).  The edges of one rank (see rank_in_row)
    touch distinct rows, so each rank is one vector step and every row still sees its edges in index order."""
    upd = np.asarray(upd, np.float32)
    idx = np.asarray(idx, np.int64)
    out = np.full((int(size), upd.shape[1]), init, np.float32)
    if len(idx) == 0:
        return out
    rank = rank_in_row(idx)
    order = np.lexsort((np.arange(len(idx)), rank))
    bounds = np.searchsorted(rank[order], np.arange(rank.max() + 2))
    for k in range(rank.max() + 1):
        sel = order[bounds[k]:bounds[k + 1]]
        out[idx[sel]] = step(out[idx[sel]], upd[sel])
    return out


def gather(params, idx):
    return np.asarray(params, np.float32)[np.asarray(idx, np.int64)]


def scatter_add(upd, idx, size):
    """MPScatterAdd: zero init, float32 adds in index order"""
    return _serial(lambda o, u: o + u, 0, upd, idx, size)


def scatter_max(upd, idx, size):
    """MPScatterMax: -1e9 init, out = upd where upd > out (strict: NaN never wins, the first of equal values stays)"""
    return _serial(lambda o, u: np.where(u > o, u, o), MAX_INIT, upd, idx, size)


def counts(idx, size):
    """scatter_add(ones[E, 1], idx, size): exact in float32 below 2^24 edges per row"""
    return np.bincount(np.asarray(idx, np.int64), minlength=int(size)).astype(np.float32)[:, None]


def scatter_mean(upd, idx, size):
    """mp_ops.scatter_mean: scatter_add(upd) / (scatter_add(ones) + 1e-7), each step rounded to float32"""
    return scatter_add(upd, idx, size) / (counts(idx, size) + EP)


def scatter_max_order_free(upd, idx, size):
    """scatter_max where the order of the edges is not kept: among equal zeros +0.0 wins over -0.0 wherever it stands (what
    an atomic max on the float's bits gives); every other result as scatter_max"""
    want = scatter_max(upd, idx, size)
    upd = np.asarray(upd, np.float32)
    plus0 = np.zeros(want.shape, bool)
    if len(idx):
        np.logical_or.at(plus0, np.asarray(idx, np.int64), (upd == 0) & ~np.signbit(upd))
    return np.where((want == 0) & plus0, np.float32(0), want)


def sum_abs64(upd, idx, size):
    """sum of |upd| per output entry in float64: the scale of a float32 sum's rounding in any order"""
    s = np.zeros((int(size), np.asarray(upd).shape[1]), np.float64)
    np.add.at(s, np.asarray(idx, np.int64), np.abs(np.asarray(upd, np.float64)))
    return s


def scatter_add64(upd, idx, size):
    s = np.zeros((int(size), np.asarray(upd).shape[1]), np.float64)
    np.add.at(s, np.asarray(idx, np.int64), np.asarray(upd, np.float64))
    return s


# ------------------------------------------------------------------ gradients (mp_ops.py:39-62), float64
def gather_grad64(grad, idx, n):
    """MPGather's gradient: scatter_add(grad, idx, n)"""
    return scatter_add64(grad, idx, n)


def scatter_add_grad64(grad, idx):
    """MPScatterAdd's gradient: gather(grad, idx)"""
    return np.asarray(grad, np.float64)[np.asarray(idx, np.int64)]


def scatter_mean_grad64(grad, idx, size):
    """the composition add / (count + 1e-7): gather(grad / (count + 1e-7), idx)"""
    return scatter_add_grad64(np.asarray(grad, np.float64) / (counts(idx, size).astype(np.float64) + 1e-7), idx)


def scatter_max_grad64(upd, idx, out, grad):
    """MPScatterMax's gradient: the upstream gradient split evenly among the updates equal to their row's maximum"""
    idx = np.asarray(idx, np.int64)
    ind = (np.asarray(upd, np.float32) == np.asarray(out, np.float32)[idx]).astype(np.float64)
    num = scatter_add64(ind, idx, len(out))
    return ind / num[idx] * np.asarray(grad, np.float64)[idx]


def scatter_softmax64(upd, idx, size):
    """mp_ops.scatter_softmax in float64 over scatter_max's (exact) result"""
    idx = np.asarray(idx, np.int64)
    m = scatter_max(upd, idx, size).astype(np.float64)
    e = np.exp(np.asarray(upd, np.float64) - m[idx])
    return e / scatter_add64(e, idx, size)[idx]


# ------------------------------------------------------------------ dense features
def rows_of(graph_ids, ids):
    """the stored row of each id, -1 for an id not in the graph"""
    graph_ids = np.asarray(graph_ids, np.uint64)
    order = np.argsort(graph_ids, kind="stable")
    q = np.asarray(ids, np.int64).reshape(-1).astype(np.uint64)
    pos = np.minimum(np.searchsorted(graph_ids[order], q), len(graph_ids) - 1)
    return np.where(graph_ids[order][pos] == q, order[pos], -1)


def dense_feature(feat, slot_dims, rows, fid, dim):
    """get_dense_feature of slot fid: the slot's stored values, clipped to dim or zero-padded to it; zeros for an absent row
    or an unknown slot"""
    feat = np.asarray(feat, np.float32)
    out = np.zeros((len(rows), dim), np.float32)
    if 0 <= fid < len(slot_dims):
        off, w = int(np.sum(slot_dims[:fid])), min(int(slot_dims[fid]), dim)
        have = rows >= 0
        out[have, :w] = feat[rows[have], off:off + w]
    return out


def whole_rows(feat, rows, dim):
    """what the fused SAGE aggregation reads per neighbor: columns [0, min(dim, feat_dim)) of the whole stored row, zeros
    beyond, zeros for an absent row"""
    return dense_feature(feat, [np.asarray(feat).shape[1]], rows, 0, dim)


def fanout_aggregate(feat, rows, dim, mean):
    """whole_rows of rows i64[R, count] reduced per R in ascending j, as scatter_add / scatter_mean over
    repeat(range(R), count) order them; one vector step per j"""
    R, count = rows.shape
    acc = np.zeros((R, dim), np.float32)
    for j in range(count):
        acc = acc + whole_rows(feat, rows[:, j], dim)
    return acc / (np.float32(count) + EP) if mean else acc
