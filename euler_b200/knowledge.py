"""Euler's knowledge-graph embedding models over id tables: TransE, TransH, TransR and TransD (examples/TransX, on TransX) and
DistMult (examples/distmult).

Each model draws its ids on the device -- the triples are the input edges (sample_edge in training), the relation id is the
edge's dense feature 'id' cast to int64, and the corrupted entities come from sample_node -- and forward(edges) returns
ModelOutput(embedding=[src_emb, rel_emb, dst_emb], loss, metric_name, metric) as upstream's call does.  With fused=True (the
default) the step after the ids -- lookups, row maps, scores, margin loss and metric -- is one device op, ops.kg_margin_loss;
with fused=False it is the literal torch composition of upstream's code (composed_kg_loss: tile, normalise, project, norm,
hinge and stable sort), which is also the reference the fused op is tested and measured against.

Tables are layers.Embedding(max_id + 1, dim): max_id + 2 rows, truncated-normal with stddev 0.1 (unsupervised.Embedding).

table_dtype=torch.bfloat16 stores every table of a model (and, through the optimizer, their slots) in bfloat16: half the
HBM.  Such tables take no autograd gradient (torch would round it to nearest bf16, losing most small updates);
train_step(edges, optimizer) runs the fused forward and sparse backward (ops.kg_margin_loss_sparse_grads) and hands the f32
rows and values to the optimizer's apply_sparse, which writes the tables back by stochastic rounding.  It needs fused=True
and one of optimizers.py's fused optimizers; forward still gives the loss, metric and embeddings, without a gradient.

One documented departure: upstream's norm_emb reshapes the relation rows to [-1, ent_dim] before normalising, which for TransR
with rel_dim != ent_dim normalises chunks that span triples (and fails when B rel_dim % ent_dim != 0).  Here each relation row
is normalised over its own rel_dim, and TransR's embeddings are [B, rel_dim], in both paths.  The two agree when the dims are
equal.
"""
import collections

import torch

from .ops import KG_MODELS, SKIPGRAM_METRICS, get_edge_dense_feature, kg_margin_loss, kg_margin_loss_sparse_grads, sample_node
from .unsupervised import Embedding, check_table_dtype, composed_metric

ModelOutput = collections.namedtuple('ModelOutput', ['embedding', 'loss', 'metric_name', 'metric'])

TRANSX_METRICS = ('mrr', 'mr', 'hit10')


def l2_normalize(x, eps=1e-12):
    """tf.nn.l2_normalize over the last axis: x * rsqrt(max(sum x^2, eps)); clamp, like TF's maximum, passes the gradient to
    sum x^2 when it is >= eps and none below"""
    return x * torch.rsqrt(torch.clamp(x.pow(2).sum(-1, keepdim=True), min=eps))


def _transx_score(s, r, d, l1):
    """calculate_scores: -||s + r - d|| over the last axis, L1 or L2"""
    return -torch.linalg.vector_norm(s + r - d, ord=1 if l1 else 2, dim=-1)


def _distmult_score(s, r, d):
    """DistMult's calculate_scores: sum s (diag(r) d), the einsum written as the product it is"""
    return (s * (r * d)).sum(-1)


def composed_kg_loss(model, tables, src, dst, neg, rel, l1=True, corrupt='both', margin=1.0, metric='mrr'):
    """The literal torch composition of TransX.call / DistMult.call after the ids, on any device:
        tables as ops.kg_margin_loss takes them; src, dst, rel [B] ids; neg [B, K] ids.
    Returns (loss, metric, (src_emb, rel_emb, dst_emb)) with the embeddings [B, dim] (TransR: [B, rel_dim])."""
    pos_scores, neg_scores, emb = composed_kg_scores(model, tables, src, dst, neg, rel, l1=l1, corrupt=corrupt)
    B = pos_scores.shape[0]
    neg_mean = neg_scores.reshape(B, -1).mean(-1, keepdim=True).reshape(-1, 1, 1)
    loss = torch.clamp(margin + neg_mean - pos_scores, min=0).mean()
    return loss, composed_metric(pos_scores.detach(), neg_scores.detach(), metric), emb


def composed_kg_scores(model, tables, src, dst, neg, rel, l1=True, corrupt='both'):
    """composed_kg_loss's scores: pos [B, 1, 1], neg [B, 1, C K] (front then tail), and the embeddings"""
    name = str(model).lower()
    if name not in KG_MODELS:
        raise ValueError("model must be one of %s, got %r" % (sorted(KG_MODELS), model))
    B, K = neg.shape
    src, dst, rel = src.reshape(B, 1), dst.reshape(B, 1), rel.reshape(B, 1)
    ent, relt = tables[0], tables[1]
    ent_dim, rel_dim = ent.shape[1], relt.shape[1]
    src_emb, dst_emb, neg_emb, rel_emb = ent[src], ent[dst], ent[neg], relt[rel]   # [B, 1 | K, dim]
    if name in ('transe', 'distmult'):
        src_emb, dst_emb, neg_emb = l2_normalize(src_emb), l2_normalize(dst_emb), l2_normalize(neg_emb)
    elif name == 'transh':
        hyper = tables[2][rel]
        hyper_expand = hyper.repeat(1, K, 1)

        def projection(e, h):
            h = l2_normalize(h)
            return e - (e * h).sum(-1, keepdim=True) * h
        src_emb, dst_emb, neg_emb = projection(src_emb, hyper), projection(dst_emb, hyper), projection(neg_emb, hyper_expand)
    elif name == 'transr':
        matrix = tables[2][rel].reshape(-1, ent_dim, rel_dim)
        matrix_expand = matrix.reshape(-1, 1, ent_dim * rel_dim).repeat(1, K, 1)

        def projection(e, m):
            n = e.shape[1]
            out = torch.matmul(e.reshape(-1, 1, ent_dim), m.reshape(-1, ent_dim, rel_dim)).reshape(-1, rel_dim)
            return l2_normalize(out).reshape(B, n, rel_dim)
        src_emb, dst_emb, neg_emb = projection(src_emb, matrix), projection(dst_emb, matrix), projection(neg_emb, matrix_expand)
    else:   # transd
        et, rt = tables[2], tables[3][rel]
        rt_expand = rt.repeat(1, K, 1)

        def projection(e, t, r_t):
            return l2_normalize(e + (e * t).sum(-1, keepdim=True) * r_t)
        src_emb = projection(src_emb, et[src], rt)
        dst_emb = projection(dst_emb, et[dst], rt)
        neg_emb = projection(neg_emb, et[neg], rt_expand)
    rel_emb = l2_normalize(rel_emb)   # over its own rel_dim (see the module docstring)

    score = _distmult_score if name == 'distmult' else (lambda a, r, c: _transx_score(a, r, c, l1))
    src_expand, rel_expand, dst_expand = src_emb.repeat(1, K, 1), rel_emb.repeat(1, K, 1), dst_emb.repeat(1, K, 1)
    pos_scores = score(src_emb, rel_emb, dst_emb).reshape(-1, 1, 1)
    if corrupt == 'front':
        neg_scores = score(neg_emb, rel_expand, dst_expand).reshape(-1, 1, K)
    elif corrupt == 'tail':
        neg_scores = score(src_expand, rel_expand, neg_emb).reshape(-1, 1, K)
    elif corrupt == 'both':
        front = score(neg_emb, rel_expand, dst_expand)
        tail = score(src_expand, rel_expand, neg_emb)
        neg_scores = torch.cat([front, tail], -1).reshape(-1, 1, 2 * K)
    else:
        raise ValueError("corrupt must be 'front', 'tail' or 'both', got %r" % (corrupt,))
    return pos_scores, neg_scores, (src_emb.reshape(B, -1), rel_emb.reshape(B, -1), dst_emb.reshape(B, -1))


class _KgModel(torch.nn.Module):
    """What TransX and DistMult share: the tables, generate_triplets, forward and train_step.  table_dtype: float32, or
    bfloat16 (fused only) for every table, trained by train_step."""
    model = None
    metrics = SKIPGRAM_METRICS

    def __init__(self, node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=5, margin=1., l1=True,
                 metric_name='mrr', corrupt='both', fused=True, sparse_grad=False, device=None, table_dtype=torch.float32):
        super().__init__()
        if metric_name not in self.metrics:
            raise ValueError('Metric name :{} not in list {}'.format(metric_name, list(self.metrics)))
        if corrupt not in ('front', 'tail', 'both'):
            raise ValueError("corrupt must be 'front', 'tail' or 'both', got %r" % (corrupt,))
        check_table_dtype(table_dtype, fused)
        self.node_type, self.edge_type = node_type, edge_type
        self.node_max_id, self.edge_max_id = node_max_id, edge_max_id
        self.ent_dim, self.rel_dim = ent_dim, rel_dim
        self.num_negs, self.margin, self.l1 = num_negs, margin, l1
        self.metric_name, self.corrupt = metric_name, corrupt
        self.fused, self.sparse_grad, self.table_dtype = fused, sparse_grad, table_dtype
        self.entity_encoder = Embedding(node_max_id + 1, ent_dim, device=device, dtype=table_dtype)
        self.relation_encoder = Embedding(edge_max_id + 1, rel_dim, device=device, dtype=table_dtype)

    def tables(self):
        """the tables in the order ops.kg_margin_loss takes them"""
        return [self.entity_encoder.embeddings, self.relation_encoder.embeddings]

    def generate_triplets(self, inputs):
        """edges [B, 3] -> src, dst [B], neg [B, num_negs], rel [B] (the 'id' edge feature cast to int64)"""
        inputs = torch.as_tensor(inputs, dtype=torch.int64)
        B = inputs.shape[0]
        src, dst = inputs[:, 0], inputs[:, 1]
        rel = get_edge_dense_feature(inputs, ['id'], [1])[0].to(torch.int64).reshape(B)
        neg = sample_node(B * self.num_negs, self.node_type).reshape(B, self.num_negs)
        return src, dst, neg, rel

    def loss_and_metric(self, src, dst, neg, rel):
        """the step after the ids: (loss, metric, [src_emb, rel_emb, dst_emb]), fused or composed"""
        if self.fused:
            loss, metric, s, r, d = kg_margin_loss(src, dst, neg, rel, self.tables(), self.model, l1=self.l1, corrupt=self.corrupt,
                                                   margin=self.margin, metric=self.metric_name, sparse_grad=self.sparse_grad,
                                                   with_embeddings=True)
            return loss, metric, [s, r, d]
        loss, metric, (s, r, d) = composed_kg_loss(self.model, self.tables(), src, dst, neg, rel, l1=self.l1, corrupt=self.corrupt,
                                                   margin=self.margin, metric=self.metric_name)
        return loss, metric, [s, r, d]

    def forward(self, inputs):
        src, dst, neg, rel = self.generate_triplets(inputs)
        loss, metric, emb = self.loss_and_metric(src, dst, neg, rel)
        return ModelOutput(embedding=emb, loss=loss, metric_name=self.metric_name, metric=metric)

    def train_step(self, inputs, optimizer):
        """One training step on the edges `inputs` without autograd: generate_triplets, the fused forward and sparse backward
        (ops.kg_margin_loss_sparse_grads), then optimizer.apply_sparse with every table's f32 rows and values.  The way to
        train bf16 tables; f32 tables take the same step.  optimizer is one of optimizers.py's, fused, over these tables.  An
        id outside its table raises before the optimizer runs: no table or slot changes.  Returns forward's ModelOutput.
        DistMult(l2_regular=True) is refused: its L2 term is a dense gradient of the whole tables, which a sparse step
        cannot carry (train it through forward and autograd)."""
        if not self.fused:
            raise ValueError("train_step runs the fused step: build the model with fused=True")
        if getattr(self, 'l2_regular', False):
            raise ValueError("train_step is a sparse step: l2_regular's whole-table term needs forward and autograd")
        if not hasattr(optimizer, 'apply_sparse'):
            raise ValueError("train_step needs one of euler_b200.optimizers' optimizers, got %s" % type(optimizer).__name__)
        src, dst, neg, rel = self.generate_triplets(inputs)
        tables = self.tables()
        loss, metric, grads, emb = kg_margin_loss_sparse_grads(
            src, dst, neg, rel, tables, self.model, l1=self.l1, corrupt=self.corrupt, margin=self.margin,
            metric=self.metric_name, with_embeddings=True)
        optimizer.apply_sparse(tables, [r for r, _ in grads], [v for _, v in grads])
        return ModelOutput(embedding=emb, loss=loss, metric_name=self.metric_name, metric=metric)


class TransX(_KgModel):
    """TransX (examples/TransX/transX.py): TransE's scores on the entity and relation tables; metric_name mrr, mr or hit10."""
    model = 'transe'
    metrics = TRANSX_METRICS


class TransE(TransX):
    """TransE (transE.py): y = n(e), r = n(r), score -||s + r - d||."""

    def __init__(self, node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=5, margin=1., l1=True,
                 metric_name='mrr', corrupt='both', **kwargs):
        if ent_dim != rel_dim:
            raise ValueError('Entity dim and Relation dim should be equal in TransE')
        super().__init__(node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=num_negs, margin=margin,
                         l1=l1, metric_name=metric_name, corrupt=corrupt, **kwargs)


class TransH(TransX):
    """TransH (transH.py): y = e - (e . h) h with h = n(hyper[rel]), not normalised."""
    model = 'transh'

    def __init__(self, node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=5, margin=1., l1=True,
                 metric_name='mrr', corrupt='both', device=None, **kwargs):
        if ent_dim != rel_dim:
            raise ValueError('Entity dim and Relation dim should be equal in TransH')
        super().__init__(node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=num_negs, margin=margin,
                         l1=l1, metric_name=metric_name, corrupt=corrupt, device=device, **kwargs)
        self.hyper_vector = Embedding(edge_max_id + 1, ent_dim, device=device, dtype=self.table_dtype)

    def tables(self):
        return super().tables() + [self.hyper_vector.embeddings]


class TransR(TransX):
    """TransR (transR.py): y = n(e M_rel), M_rel = transfer_matrix[rel] as [ent_dim, rel_dim]; the fused op supports
    ent_dim * rel_dim up to 16384 (128 x 128), dims up to 512."""
    model = 'transr'

    def __init__(self, node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=5, margin=1., l1=True,
                 metric_name='mrr', corrupt='both', device=None, **kwargs):
        super().__init__(node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=num_negs, margin=margin,
                         l1=l1, metric_name=metric_name, corrupt=corrupt, device=device, **kwargs)
        self.transfer_matrix = Embedding(edge_max_id + 1, ent_dim * rel_dim, device=device, dtype=self.table_dtype)

    def tables(self):
        return super().tables() + [self.transfer_matrix.embeddings]


class TransD(TransX):
    """TransD (transD.py): y = n(e + (e . e_t) r_t), e_t = entity_transfer[id], r_t = relation_transfer[rel]."""
    model = 'transd'

    def __init__(self, node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=5, margin=1., l1=True,
                 metric_name='mrr', corrupt='both', device=None, **kwargs):
        if ent_dim != rel_dim:
            raise ValueError('Entity dim and Relation dim should be equal in TransD')
        super().__init__(node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=num_negs, margin=margin,
                         l1=l1, metric_name=metric_name, corrupt=corrupt, device=device, **kwargs)
        self.entity_transfer = Embedding(node_max_id + 1, ent_dim, device=device, dtype=self.table_dtype)
        self.relation_transfer = Embedding(edge_max_id + 1, rel_dim, device=device, dtype=self.table_dtype)

    def tables(self):
        return super().tables() + [self.entity_transfer.embeddings, self.relation_transfer.embeddings]


class DistMult(_KgModel):
    """DistMult (examples/distmult/distmult.py): y = n(e), r = n(r), score sum s (r d).  metric_name is one of metrics.get's
    ranking metrics (mrr, hit1, hit3, hit10, mr); its acc / auc / f1 take labels, not score pairs, and raise ValueError.
    l2_regular adds regular_param * (sum E^2 + sum R^2) over both whole tables, a torch term in both paths (not with
    sparse_grad, bfloat16 tables or train_step: it is a dense whole-table autograd gradient).  The fused op needs ent_dim ==
    rel_dim, which upstream's einsum needs too."""
    model = 'distmult'

    def __init__(self, node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=5, margin=1, metric_name='mrr',
                 corrupt='both', l2_regular=False, regular_param=0.0001, **kwargs):
        if ent_dim != rel_dim:
            raise ValueError('Entity dim and Relation dim should be equal in DistMult')
        if l2_regular and kwargs.get('table_dtype', torch.float32) == torch.bfloat16:
            raise ValueError('l2_regular is a dense autograd gradient of the whole tables: it cannot train bfloat16 tables')
        super().__init__(node_type, edge_type, node_max_id, edge_max_id, ent_dim, rel_dim, num_negs=num_negs, margin=margin,
                         metric_name=metric_name, corrupt=corrupt, **kwargs)
        if l2_regular and self.sparse_grad:
            raise ValueError('l2_regular sums over the whole tables: it cannot be combined with sparse_grad')
        self.l2_regular, self.regular_param = l2_regular, regular_param

    def loss_and_metric(self, src, dst, neg, rel):
        loss, metric, emb = super().loss_and_metric(src, dst, neg, rel)
        if self.l2_regular:
            loss = loss + self.regular_param * self.entity_encoder.embeddings.pow(2).sum()
            loss = loss + self.regular_param * self.relation_encoder.embeddings.pow(2).sum()
        return loss, metric, emb
