"""tf_euler.solution (tf_euler/python/solution/{base_supervise,base_unsupervise,samplers,logits,losses,utils}.py) over torch
modules: the way upstream trains any node encoder, supervised from a label slot or unsupervised from positive and negative
samples, with upstream's constructor arguments and defaults.

An encoder is any callable that maps int64 node ids [N] to rows [N, D], e.g. encoders.SageEncoder, encoders.GCNEncoder or
encoders.ShallowEncoder.  Both solutions are torch modules, so the encoders and logits they are given (when those are modules)
are their submodules and solution.parameters() lists every trainable tensor.  __call__(inputs) returns upstream's
(embedding, loss, metric_name, metric).

The step after the encoders is plain torch: PosNegLogits + xent_loss + the rank metric are unsupervised.py's composition
(the rows already exist as encoder outputs, so a fused id-table op has nothing to save there).  By default metrics are
each batch's own value, where upstream's f1 / acc are streaming tf.metrics: 'f1' and 'acc' for SuperviseSolution, 'mrr',
'hit1', 'hit3', 'hit10' and 'mr' for UnsuperviseSolution (per batch upstream too).  SuperviseSolution(..., streaming=True)
takes upstream's streaming metrics instead -- 'f1', 'acc' or 'auc' (tf.metrics.auc at 5000 thresholds, applied to
sigmoid(logit) with its own sigmoid, as upstream) -- as the device module solution.metric (euler_b200/metrics.py), whose
value covers every batch since construction or solution.metric.reset().  Without streaming, 'auc' is refused.
SuperviseSampleSolution / UnsuperviseSampleSolution, which parse text sample files on the host, are not provided either.
"""
import torch
import torch.nn.functional as F

from . import metrics, ops
from .convolution import l2_normalize
from .ops import SKIPGRAM_METRICS
from .supervised import f1_score
from .unsupervised import composed_metric, xent_loss  # noqa: F401  (xent_loss is solution/losses.py's)


# ------------------------------------------------------------------------------------ utils, logits, losses
class GetLabelFromFea(object):
    """utils.GetLabelFromFea: the label of each node is its dense feature label_idx, label_dim columns wide"""

    def __init__(self, label_idx, label_dim):
        self.label_idx = label_idx
        self.label_dim = label_dim

    def __call__(self, inputs):
        label, = ops.get_dense_feature(inputs, [self.label_idx], [self.label_dim])
        return label


class DenseLogits(torch.nn.Module):
    """logits.DenseLogits: a bias-free tf.layers.Dense(logits_dim) with a glorot-uniform kernel, built as
    supervised.SuperviseModel.out_fc is; dim is the width of its inputs, which torch needs up front"""

    def __init__(self, logits_dim, *, dim, device=None):
        super().__init__()
        self.out_fc = torch.nn.Linear(dim, logits_dim, bias=False, device=device)
        torch.nn.init.xavier_uniform_(self.out_fc.weight)

    def forward(self, inputs, **kwargs):
        return self.out_fc(inputs)


class PosNegLogits(object):
    """logits.PosNegLogits: (emb pos_emb^T, emb neg_emb^T) over the last two axes"""

    def __call__(self, emb, pos_emb, neg_emb):
        return torch.matmul(emb, pos_emb.transpose(-1, -2)), torch.matmul(emb, neg_emb.transpose(-1, -2))


class CosineLogits(object):
    """logits.CosineLogits: 5 <l2_normalize(x), l2_normalize(y)> over the last axis, kept as an axis of 1"""

    def __call__(self, target_emb, context_emb):
        return (l2_normalize(target_emb) * l2_normalize(context_emb)).sum(-1, keepdim=True) * 5.0


def sigmoid_loss(labels, logits):
    """losses.sigmoid_loss: the mean sigmoid cross entropy of logits against labels"""
    return F.binary_cross_entropy_with_logits(logits, labels.reshape(logits.shape))


# ------------------------------------------------------------------------------------ metrics
def acc_score(labels, predict):
    """metrics.acc_score for one batch: the share of elements where floor(predict + 0.5) equals the label"""
    return (torch.floor(predict + 0.5) == labels.reshape(predict.shape).to(predict.dtype)).to(torch.float32).mean()


SUPERVISED_METRICS = {'f1': f1_score, 'acc': acc_score}


def _metric(name, known):
    """the metric function of `name` among `known`; auc, upstream's streaming tf.metrics.auc, is refused with its reason"""
    if name == 'auc':
        raise NotImplementedError("metric 'auc' is tf.metrics.auc, a streaming histogram over the session's batches, and is "
                                  "not provided; use one of %s" % (sorted(known),))
    if name not in known:
        raise ValueError("metric_name must be one of %s, got %r" % (sorted(known), name))
    return known[name]


# ------------------------------------------------------------------------------------ samplers
class SampleNegWithTypes(object):
    """samplers.SampleNegWithTypes: num_negs nodes per input from sample_node of each listed type, [B, num_negs]; a list of
    them, one per type, when several types are listed (which UnsuperviseSolution refuses, as upstream)"""

    def __init__(self, neg_type, num_negs=5):
        if not isinstance(neg_type, list):
            neg_type = [neg_type]
        self.num_negs = num_negs
        self.neg_type = neg_type

    def __call__(self, inputs):
        batch_size = inputs.shape[0]
        group = [ops.sample_node(batch_size * self.num_negs, t).reshape(batch_size, self.num_negs) for t in self.neg_type]
        return group[0] if len(self.neg_type) == 1 else group


class SamplePosWithTypes(object):
    """samplers.SamplePosWithTypes: num_pos neighbours of each input over edge_type, default node max_id + 1, [B, num_pos]"""

    def __init__(self, edge_type, num_pos=1, max_id=-1):
        self.edge_type = edge_type
        self.num_pos = num_pos
        self.max_id = max_id

    def __call__(self, inputs):
        return ops.sample_neighbor(inputs, self.edge_type, self.num_pos, self.max_id + 1)[0]


# ------------------------------------------------------------------------------------ solutions
class SuperviseSolution(torch.nn.Module):
    """base_supervise.SuperviseSolution: label = get_label_fn(inputs), embedding = encoder_fn(inputs),
    logit = logit_fn(embedding); loss_fn(label, logit) and the metric of (label, sigmoid(logit)).  streaming=True takes the
    streaming metric solution.metric ('f1', 'acc' or 'auc'; see the top of the file)."""

    def __init__(self, get_label_fn, encoder_fn, logit_fn, metric_name='f1', loss_fn=sigmoid_loss, *, streaming=False):
        super().__init__()
        self.get_label_fn = get_label_fn
        self.metric_name = metric_name
        self.streaming = bool(streaming)
        if self.streaming:
            self.metric = metrics.get(metric_name)
            self.metric_class = None
        else:
            self.metric_class = _metric(metric_name, SUPERVISED_METRICS)
        self.encoder = encoder_fn
        self.logit_fn = logit_fn
        self.loss_fn = loss_fn

    def embed(self, n_id):
        return self.encoder(n_id)

    def forward(self, inputs):
        label = self.get_label_fn(inputs)
        embedding = self.embed(inputs)
        logit = self.logit_fn(embedding)
        metric = (self.metric if self.streaming else self.metric_class)(label, torch.sigmoid(logit.detach()))
        loss = self.loss_fn(label, logit)
        return embedding, loss, self.metric_name, metric


class UnsuperviseSolution(torch.nn.Module):
    """base_unsupervise.UnsuperviseSolution: src = inputs[:, None], pos = pos_sample_fn(inputs) [B, P], negs =
    neg_sample_fn(inputs) [B, K]; the target encoder embeds src and the context encoder pos and negs, each reshaped to
    [B, -1, D]; logit_fn gives (logits, neg_logits), loss_fn their loss and the rank metric reads them.  The returned
    embedding is a second target pass over inputs, as upstream (a sampling encoder draws again)."""

    def __init__(self, target_encoder_fn, context_encoder_fn, pos_sample_fn, neg_sample_fn, metric_name='mrr',
                 logit_fn=PosNegLogits(), loss_fn=xent_loss):
        super().__init__()
        self.metric_name = metric_name
        rank = _metric(metric_name, {m: m for m in SKIPGRAM_METRICS})
        self.metric_class = lambda logits, neg_logits: composed_metric(logits, neg_logits, rank)
        self.target_encoder = target_encoder_fn
        self.context_encoder = context_encoder_fn
        self.pos_sample_fn = pos_sample_fn
        self.neg_sample_fn = neg_sample_fn
        self.logit_fn = logit_fn
        self.loss_fn = loss_fn

    @staticmethod
    def _embed(encoder, n_id):
        emb = encoder(n_id.reshape(-1))
        return emb.reshape(n_id.shape[0], -1, emb.shape[-1])

    def target_embed(self, n_id):
        return self._embed(self.target_encoder, n_id)

    def context_embed(self, n_id):
        return self._embed(self.context_encoder, n_id)

    def to_sample(self, inputs):
        src = inputs.unsqueeze(-1)
        pos = self.pos_sample_fn(inputs)
        negs = self.neg_sample_fn(inputs)
        if not (torch.is_tensor(negs) and negs.dim() == 2 and torch.is_tensor(pos) and pos.dim() == 2):
            raise ValueError("UnsuperviseSolution: pos_sample_fn and neg_sample_fn must each return one [B, n] tensor "
                             "(SampleNegWithTypes over several types returns a list)")
        return src, pos, negs

    def forward(self, inputs):
        src, pos, negs = self.to_sample(inputs)
        embedding = self.target_embed(src)
        embedding_pos = self.context_embed(pos)
        embedding_negs = self.context_embed(negs)
        logits, neg_logits = self.logit_fn(embedding, embedding_pos, embedding_negs)
        loss = self.loss_fn(logits, neg_logits)
        metric = self.metric_class(logits.detach(), neg_logits.detach())
        embedding = self.target_embed(inputs)
        return embedding, loss, self.metric_name, metric
