"""numpy restatements of the unsupervised skip-gram step (UnsuperviseModel.__call__, mp_utils/base.py:50-91; PosNegLogits,
xent_loss, utils/metrics.py) and of its gradient, used by the CPU and GPU tests of ops.skipgram_xent_loss."""
import numpy as np


def context_ids(pos, negs):
    """the J = P + K context ids of each pair row: the positives, then the negatives"""
    return np.concatenate([np.asarray(pos, np.int64).reshape(len(pos), -1), np.asarray(negs, np.int64).reshape(len(pos), -1)], 1)


def dot_fixed_order_f32(a, b):
    """k_agnn_dot's order over one pair of f32 rows: lane l of G lanes (G = the power of two >= ceil(dim / 4), <= 32) adds with
    fma from +0 the columns of its 4-column chunks l, l + G, ..., left to right; then a butterfly, xor distances G/2 .. 1.
    fma is emulated in f64 (exact for the dyadic inputs the tests use)."""
    dim = len(a)
    nch = (dim + 3) // 4
    G = 1
    while G < 32 and G < nch:
        G *= 2
    acc = [np.float32(0)] * G
    for l in range(G):
        for ch in range(l, nch, G):
            for d in range(4 * ch, min(4 * ch + 4, dim)):
                acc[l] = np.float32(np.float64(a[d]) * np.float64(b[d]) + np.float64(acc[l]))
    o = G // 2
    while o > 0:
        acc = [np.float32(acc[l] + acc[l ^ o]) for l in range(G)]
        o //= 2
    return acc[0]


def logits_f32(target, context, src, ctx):
    """logits [B, J] in the fixed order"""
    B, J = ctx.shape
    out = np.zeros((B, J), np.float32)
    for b in range(B):
        for j in range(J):
            out[b, j] = dot_fixed_order_f32(target[src[b]], context[ctx[b, j]])
    return out


def rank_closed_form(logits, P):
    """#{j != P-1 : x_j >= x_{P-1}} per row"""
    x = np.asarray(logits)
    last = x[:, P - 1:P]
    ge = x >= last
    ge[:, P - 1] = False
    return ge.sum(1).astype(np.int64)


def rank_top_k_literal(pos_logits, neg_logits):
    """mrr_score's ranks[:, -1], literally: all = concat([neg, pos]); indices_of_ranks = top_k(all) (stable: a descending sort
    in which equal values keep index order); ranks = top_k(-indices_of_ranks), the inverse permutation; its last entry"""
    out = []
    for p, n in zip(np.asarray(pos_logits), np.asarray(neg_logits)):
        scores = list(n) + list(p)
        idx = sorted(range(len(scores)), key=lambda i: (-scores[i], i))
        neg_idx = [-i for i in idx]
        ranks = sorted(range(len(neg_idx)), key=lambda m: (-neg_idx[m], m))
        out.append(ranks[-1])
    return np.asarray(out, np.int64)


def xent64(x, z):
    """sigmoid_cross_entropy_with_logits in f64: max(x, 0) - x z + log1p(exp(-|x|))"""
    x = np.asarray(x, np.float64)
    return np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))


def loss64(logits, P):
    x = np.asarray(logits, np.float64)
    z = np.zeros_like(x)
    z[:, :P] = 1
    return xent64(x, z).mean() if x.size else np.nan


def metric(rank, name):
    """mrr (f32 mean of reciprocals), hitK (f32 mean), mr (tf.reduce_mean of int64: the integer mean, truncated)"""
    rank = np.asarray(rank, np.int64)
    if name == 'mrr':
        return np.float32(np.mean(np.float32(1) / (rank + 1).astype(np.float32), dtype=np.float64))
    if name.startswith('hit'):
        return np.float32(np.mean(rank < int(name[3:])))
    if name == 'mr':
        return int(rank.sum() // max(len(rank), 1))
    raise ValueError(name)


def forward64(target, context, src, ctx, P):
    """(logits f64 [B, J], loss) of the step in f64"""
    t = np.asarray(target, np.float64)[src]
    c = np.asarray(context, np.float64)[ctx]
    x = np.einsum('bd,bjd->bj', t, c)
    return x, loss64(x, P)


def grads64(target, context, src, ctx, P, g=1.0, logits=None):
    """dense f64 gradients of g * loss for the target and the context table (add them for a shared table).  logits: the
    logits to take sigmoid of (default: the f64 ones)"""
    t = np.asarray(target, np.float64)
    cx = np.asarray(context, np.float64)
    x = forward64(target, context, src, ctx, P)[0] if logits is None else np.asarray(logits, np.float64)
    B, J = x.shape
    z = np.zeros_like(x)
    z[:, :P] = 1
    coef = (1 / (1 + np.exp(-x)) - z) * g / max(B * J, 1)
    gt = np.zeros_like(t)
    gc = np.zeros_like(cx)
    np.add.at(gt, src, np.einsum('bj,bjd->bd', coef, cx[ctx]))
    np.add.at(gc, ctx.reshape(-1), (coef[:, :, None] * t[src][:, None, :]).reshape(B * J, -1))
    return gt, gc


def gen_pair_count(path_len, left, right):
    """gen_pair's pairs per walk of path_len nodes (gen_pair_op.cc): each node with the nodes up to `left` before and `right`
    after it"""
    return sum(min(i, left) + min(path_len - 1 - i, right) for i in range(path_len))


# ------------------------------------------------------------------------------------ device helpers of the GPU tests
def device_table(n_rows, dim, rng, offset=0, dyadic=True):
    """a f32 table on the device whose data pointer is `offset` floats past a 16-byte boundary; dyadic: values k / 8,
    |k| <= 8"""
    import torch
    v = rng.randint(-8, 9, size=n_rows * dim + offset) / 8.0 if dyadic else rng.randn(n_rows * dim + offset) * 0.3
    t = torch.tensor(v, dtype=torch.float32).cuda()
    return t[offset:].view(n_rows, dim)


def pair_ids(rng, B, P, K, n_rows):
    """random (src [B], pos [B, P], negs [B, K]), the last row named by a few src and pos entries"""
    src = rng.randint(0, n_rows, size=B)
    pos = rng.randint(0, n_rows, size=(B, P))
    negs = rng.randint(0, n_rows, size=(B, K))
    src[:3] = n_rows - 1            # the default row max_id + 1 of a table of max_id + 2 rows
    pos[3:6, 0] = n_rows - 1
    return src, pos, negs


def device_forward(src, pos, negs, target, context):
    """one eu_skipgram_loss: (logits, rank, loss)"""
    import torch
    from euler_b200 import ops
    d = lambda a: torch.as_tensor(a, dtype=torch.int64).cuda().contiguous()   # noqa: E731
    return ops._raw_skipgram(d(src).reshape(-1), d(pos), d(negs).reshape(len(src), -1), target, context)


def device_grads(src, pos, negs, target, context, shared=False, sparse=False, g=None):
    """(loss, the target table's gradient, the context table's or None when shared) of skipgram_xent_loss on copies of the
    tables, the loss's upstream gradient g (default 1)"""
    import torch
    import euler_b200
    T = target.clone().requires_grad_(True)
    Cx = T if shared else context.clone().requires_grad_(True)
    loss, _ = euler_b200.skipgram_xent_loss(src, pos, negs, T, Cx, sparse_grad=sparse)
    loss.backward(None if g is None else torch.tensor(g, dtype=torch.float32, device="cuda"))
    return loss, T.grad, (None if shared else Cx.grad)
