"""The unsupervised models of Euler's skip-gram family over id embeddings: DeepWalk and node2vec (examples/deepwalk, over
BaseNode2Vec.to_sample) and LINE of first and second order (examples/line), on UnsuperviseModel
(tf_euler/python/mp_utils/base.py:50-91).

Each model draws its ids on the device (sample_neighbor / random_walk + gen_pair, and sample_node for the negatives), and its
__call__ returns (embedding, loss, metric_name, metric) as upstream.  With fused=True (the default) the step after the ids --
the three embedding lookups, PosNegLogits, xent_loss and the metric -- is one device op, ops.skipgram_xent_loss; with
fused=False it is the literal torch composition of those pieces (composed_skipgram_loss), which is also the reference the
fused op is measured and tested against.

The encoders here are id tables, ShallowEncoder(max_id=max_id) with ids only: layers.Embedding(max_id + 1, dim), a table of
max_id + 2 rows, so the default node max_id + 1 that random_walk and sample_neighbor pad with is a row of its own.
Upstream's neg_condition (sample_node with an index query) is not supported.

table_dtype=torch.bfloat16 stores the id tables (and, through the optimizer, their slots) in bfloat16: half the HBM.  Such
tables take no autograd gradient (torch would round it to nearest bf16, losing most small updates); train_step(batch,
optimizer) runs the fused forward and sparse backward and hands the f32 rows and values to the optimizer's apply_sparse,
which writes the tables back by stochastic rounding.  It needs fused=True and one of optimizers.py's fused optimizers.

DGI (examples/dgi/dgi.py) is the one model here over a GraphSAGE encoder: encoders.ShuffleSageEncoder with ShallowEncoder's
feature inputs, a bilinear decoder against the batch's readout, and the same rank metrics (composed_metric).  The
unsupervised GraphSage / GCN models are solution.UnsuperviseSolution over two encoders.
"""
import torch
import torch.nn.functional as F

from . import _lib
from .ops import (SKIPGRAM_METRICS, gen_pair, random_walk, sample_neighbor, sample_node, skipgram_xent_loss,
                  skipgram_xent_loss_sparse_grads)


def _truncated_normal_(t, stddev):
    """tf.truncated_normal_initializer: normal draws, those beyond two standard deviations drawn again"""
    torch.nn.init.trunc_normal_(t, mean=0.0, std=stddev, a=-2 * stddev, b=2 * stddev)
    return t


class Embedding(torch.nn.Module):
    """layers.Embedding(max_id, dim) (utils/layers.py:119-149): a table f32[max_id + 1, dim] initialised truncated-normal with
    stddev 0.1; forward(ids) = tf.nn.embedding_lookup, shape ids.shape + (dim,)."""

    def __init__(self, max_id, dim, device=None, dtype=torch.float32):
        super().__init__()
        table = _truncated_normal_(torch.empty(max_id + 1, dim, device=device), 0.1)
        if dtype == torch.float32:
            self.embeddings = torch.nn.Parameter(table)
        else:   # initialised in f32, rounded once to nearest; trained without autograd (UnsuperviseModel.train_step)
            self.embeddings = torch.nn.Parameter(table.to(dtype), requires_grad=False)

    def forward(self, ids):
        return F.embedding(ids, self.embeddings)


def check_table_dtype(table_dtype, fused):
    """ValueError unless table_dtype is float32, or bfloat16 with fused=True (bf16 tables train without autograd)"""
    if table_dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("table_dtype must be torch.float32 or torch.bfloat16, got %r" % (table_dtype,))
    if table_dtype == torch.bfloat16 and not fused:
        raise ValueError("table_dtype=torch.bfloat16 needs fused=True: the composed step trains through autograd")


def _stable_ranks(pos_logits, neg_logits):
    """metrics.py's rank of the last entry of concat([neg, pos], 2): top_k (stable: ties to the lower index) and its inverse"""
    scores = torch.cat([neg_logits, pos_logits], 2)
    order = torch.sort(scores, dim=2, descending=True, stable=True).indices   # top_k's indices_of_ranks
    return torch.argsort(order, dim=2)[:, :, -1]                                # ranks[:, :, -1]: the inverse permutation


def composed_metric(pos_logits, neg_logits, name):
    """mrr_score / hitk_score / mr_score (utils/metrics.py) on logits [B, 1, P] and [B, 1, K], composed from torch ops"""
    rank = _stable_ranks(pos_logits, neg_logits)
    if name == 'mrr':
        return torch.reciprocal((rank + 1).to(torch.float32)).mean()
    if name in ('hit1', 'hit3', 'hit10'):
        return (rank < int(name[3:])).to(torch.float32).mean()
    if name == 'mr':
        return torch.div(rank.sum(), max(rank.numel(), 1), rounding_mode='trunc')
    raise ValueError("metric must be one of %s, got %r" % (SKIPGRAM_METRICS, name))


def xent_loss(logits, neg_logits):
    """solution/losses.py's xent_loss: the mean sigmoid cross entropy of logits against ones and neg_logits against zeros,
    over every entry of both"""
    true_xent = F.binary_cross_entropy_with_logits(logits, torch.ones_like(logits), reduction='none')
    negative_xent = F.binary_cross_entropy_with_logits(neg_logits, torch.zeros_like(neg_logits), reduction='none')
    return torch.cat([true_xent.reshape(-1, 1), negative_xent.reshape(-1, 1)], 0).mean()


def composed_skipgram_loss(emb, pos_emb, neg_emb, metric='mrr'):
    """PosNegLogits + xent_loss + the metric, literally (solution/logits.py, solution/losses.py): emb [B, 1, dim], pos_emb
    [B, P, dim], neg_emb [B, K, dim] -> (loss, metric)."""
    logit = torch.matmul(emb, pos_emb.transpose(1, 2))
    neg_logit = torch.matmul(emb, neg_emb.transpose(1, 2))
    return xent_loss(logit, neg_logit), composed_metric(logit.detach(), neg_logit.detach(), metric)


class UnsuperviseModel(torch.nn.Module):
    """UnsuperviseModel(node_type, edge_type, max_id, num_negs=20, metric_name='mrr') with id-table encoders of dim columns.
    to_sample: src = inputs, one positive from sample_neighbor(inputs, edge_type, 1, max_id + 1), num_negs negatives per row
    from sample_node.  share_context: the context encoder is the target encoder (LINE's first order).  table_dtype: float32, or
    bfloat16 (fused only), trained by train_step."""

    def __init__(self, node_type, edge_type, max_id, dim, num_negs=20, metric_name='mrr', fused=True, sparse_grad=False,
                 share_context=False, device=None, table_dtype=torch.float32):
        super().__init__()
        if metric_name not in SKIPGRAM_METRICS:
            raise ValueError("metric_name must be one of %s, got %r" % (SKIPGRAM_METRICS, metric_name))
        check_table_dtype(table_dtype, fused)
        self.node_type, self.edge_type, self.max_id = node_type, edge_type, max_id
        self.num_negs, self.metric_name = num_negs, metric_name
        self.fused, self.sparse_grad, self.table_dtype = fused, sparse_grad, table_dtype
        self.target_encoder = Embedding(max_id + 1, dim, device=device, dtype=table_dtype)
        self.context_encoder = (self.target_encoder if share_context
                                else Embedding(max_id + 1, dim, device=device, dtype=table_dtype))

    def embed(self, ids):
        return self.target_encoder(ids)

    def embed_context(self, ids):
        return self.context_encoder(ids)

    def sample_shapes(self, batch_size):
        """the shapes of (src, pos, negs) that to_sample draws for a batch of batch_size nodes"""
        return (batch_size, 1), (batch_size, 1), (batch_size, self.num_negs)

    def to_sample(self, inputs):
        B = inputs.numel()
        src = inputs.reshape(-1, 1)
        pos = sample_neighbor(inputs, self.edge_type, 1, self.max_id + 1)[0]
        negs = sample_node(B * self.num_negs, self.node_type).reshape(B, self.num_negs)
        return src, pos, negs

    def loss_and_metric(self, src, pos, negs):
        """the step after the ids: (loss, metric), fused or composed"""
        if self.fused:
            return skipgram_xent_loss(src, pos, negs, self.target_encoder.embeddings, self.context_encoder.embeddings,
                                      metric=self.metric_name, sparse_grad=self.sparse_grad)
        return composed_skipgram_loss(self.embed(src), self.embed_context(pos), self.embed_context(negs), self.metric_name)

    def forward(self, inputs):
        src, pos, negs = self.to_sample(inputs)
        loss, metric = self.loss_and_metric(src, pos, negs)
        return self.embed(inputs), loss, self.metric_name, metric

    def train_step(self, batch, optimizer):
        """One training step on the node ids `batch` without autograd: to_sample, the fused forward and sparse backward
        (ops.skipgram_xent_loss_sparse_grads), then optimizer.apply_sparse with the tables' f32 rows and values.  The way to
        train bf16 tables; f32 tables take the same step.  optimizer is one of optimizers.py's, fused, over these tables.
        Returns (loss, metric)."""
        if not self.fused:
            raise ValueError("train_step runs the fused step: build the model with fused=True")
        if not hasattr(optimizer, 'apply_sparse'):
            raise ValueError("train_step needs one of euler_b200.optimizers' optimizers, got %s" % type(optimizer).__name__)
        src, pos, negs = self.to_sample(batch)
        target, context = self.target_encoder.embeddings, self.context_encoder.embeddings
        loss, metric, grads = skipgram_xent_loss_sparse_grads(src, pos, negs, target, context, metric=self.metric_name)
        tables = [target] if context is target else [target, context]
        optimizer.apply_sparse(tables, [r for r, _ in grads], [v for _, v in grads])
        return loss, metric


def pairs_per_walk(walk_len, left_win_size, right_win_size):
    """gen_pair's pairs per walk of walk_len steps (walk_len + 1 nodes): BaseNode2Vec.batch_size_ratio"""
    return int(_lib.load().eu_gen_pair_count(walk_len + 1, left_win_size, right_win_size))


class BaseNode2Vec(UnsuperviseModel):
    """BaseNode2Vec (examples/deepwalk/deepwalk.py): to_sample walks walk_len steps from each input (random_walk with p, q and
    default_node max_id + 1), cuts the walks into skip-gram pairs (gen_pair), and draws num_negs negatives per pair: src and
    pos [B * pairs, 1], negs [B * pairs, num_negs]."""

    def __init__(self, node_type, edge_type, max_id, dim, walk_len=3, walk_p=1, walk_q=1, left_win_size=1, right_win_size=1,
                 num_negs=5, metric_name='mrr', **kwargs):
        super().__init__(node_type, edge_type, max_id, dim, num_negs=num_negs, metric_name=metric_name, **kwargs)
        self.walk_len, self.walk_p, self.walk_q = walk_len, walk_p, walk_q
        self.left_win_size, self.right_win_size = left_win_size, right_win_size
        self.batch_size_ratio = pairs_per_walk(walk_len, left_win_size, right_win_size)

    def sample_shapes(self, batch_size):
        n = batch_size * self.batch_size_ratio
        return (n, 1), (n, 1), (n, self.num_negs)

    def to_sample(self, inputs):
        B = inputs.numel()
        path = random_walk(inputs, [self.edge_type] * self.walk_len, p=self.walk_p, q=self.walk_q, default_node=self.max_id + 1)
        pair = gen_pair(path, self.left_win_size, self.right_win_size)
        n = B * pair.shape[1]
        src = pair[:, :, 0].reshape(n, 1)
        pos = pair[:, :, 1].reshape(n, 1)
        negs = sample_node(n * self.num_negs, self.node_type).reshape(n, self.num_negs)
        return src, pos, negs


class DeepWalk(BaseNode2Vec):
    """DeepWalk (examples/deepwalk/deepwalk.py) with id encoders: uniform walks unless walk_p / walk_q are given."""


class Node2Vec(DeepWalk):
    """node2vec: DeepWalk's model with biased walks (walk_p, walk_q)."""


class Line(UnsuperviseModel):
    """Line (examples/line/line.py), order 1 or 'first' (the context encoder IS the target encoder: one shared table) or
    2 or 'second' (a context table of its own)."""

    def __init__(self, node_type, edge_type, max_id, dim, num_negs=5, order=1, metric_name='mrr', **kwargs):
        order = {1: 'first', 2: 'second'}.get(order, order)
        if order not in ('first', 'second'):
            raise ValueError('Line order must be one of 1, 2, "first", or "second" got {}:'.format(order))
        super().__init__(node_type, edge_type, max_id, dim, num_negs=num_negs, metric_name=metric_name,
                         share_context=order == 'first', **kwargs)
        self.order = order


class DGI(torch.nn.Module):
    """DGI (examples/dgi/dgi.py:24-90), upstream's arguments: the target encoder is ShuffleSageEncoder(metapath, fanouts, dim,
    aggregator, concat, ..), which embeds the batch over its sample tree and over the tree with shuffled rows (the negatives).
    decoder scores kernel(embedding) and kernel(embedding_negs) (a bias-free Dense(dim)) against the readout, the sigmoid of
    the batch's mean embedding, with sigmoid cross entropy (ones for the true rows, zeros for the shuffled ones) and
    composed_metric for the rank metric.  __call__(inputs, generator=None) returns upstream's
    (embedding, loss, metric_name, metric), the embedding from a second pass of the encoder with fresh samples, as upstream;
    generator fixes the shuffles.  num_negs is kept and unused, as upstream.  fused / sparse_grad / table_dtype are
    SageEncoder's (bfloat16 tables train with optimizers.minimize)."""

    def __init__(self, node_type, edge_type, max_id, metapath, fanouts, dim, aggregator='mean', concat=False, feature_idx=-1,
                 feature_dim=0, use_feature=None, use_id=False, sparse_feature_idx=-1, sparse_feature_max_id=-1, embedding_dim=16,
                 use_hash_embedding=False, use_residual=False, num_negs=5, metric='mrr', fused=True, sparse_grad=False, device=None,
                 table_dtype=torch.float32):
        super().__init__()
        from .encoders import Dense, ShuffleSageEncoder   # encoders builds on Embedding above
        if metric not in SKIPGRAM_METRICS:
            raise ValueError("metric must be one of %s, got %r" % (SKIPGRAM_METRICS, metric))
        self.node_type, self.edge_type, self.max_id = node_type, edge_type, max_id
        self.num_negs, self.dim, self.metric_name = num_negs, dim, metric
        self.kernel = Dense(dim, dim, device=device)
        self._target_encoder = ShuffleSageEncoder(
            metapath, fanouts, dim, aggregator, concat, feature_idx=feature_idx, feature_dim=feature_dim, max_id=max_id,
            use_id=use_id, sparse_feature_idx=sparse_feature_idx, sparse_feature_max_id=sparse_feature_max_id,
            embedding_dim=embedding_dim, use_hash_embedding=use_hash_embedding, use_residual=use_residual, fused=fused,
            sparse_grad=sparse_grad, device=device, table_dtype=table_dtype)

    def target_encoder(self, inputs, generator=None):
        return self._target_encoder(inputs, generator)

    def readout_func(self, inputs):
        return torch.sigmoid(inputs.mean(0, keepdim=True)).expand(inputs.shape[0], -1, -1)

    def decoder(self, embedding, embedding_pos, embedding_negs):
        logits = torch.matmul(self.kernel(embedding), embedding_pos.transpose(1, 2))
        neg_logits = torch.matmul(self.kernel(embedding_negs), embedding_pos.transpose(1, 2))
        metric = composed_metric(logits.detach(), neg_logits.detach(), self.metric_name)
        return xent_loss(logits, neg_logits), metric

    def forward(self, inputs, generator=None):
        src = inputs.unsqueeze(-1)
        embedding, embedding_negs = self.target_encoder(src, generator)
        loss, metric = self.decoder(embedding, self.readout_func(embedding), embedding_negs)
        embedding = self.target_encoder(inputs, generator)[0]
        return embedding, loss, self.metric_name, metric
