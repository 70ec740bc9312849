"""SuperviseModel (tf_euler/python/mp_utils/base.py:24-47): the supervised training step over any node encoder, and f1_score
(tf_euler/python/utils/metrics.py:35-48)."""
import torch
import torch.nn.functional as F

from . import metrics, ops


def f1_score(labels, predict):
    """metrics.f1_score for one batch: predictions = floor(predict + 0.5), true / false positives and false negatives counted
    over every element, precision = tp / (1e-7 + tp + fp), recall = tp / (1e-7 + tp + fn),
    f1 = 2 precision recall / (precision + recall + 1e-7).  Upstream's metric is streaming (tf.metrics accumulates the counts
    over the session's batches); this one is the batch's own value, and metrics.StreamingF1 is the streaming one."""
    predictions = torch.floor(predict + 0.5) != 0
    labels = labels != 0
    epsilon = 1e-7
    tp = (labels & predictions).sum().to(torch.float32)
    fn = (labels & ~predictions).sum().to(torch.float32)
    fp = (~labels & predictions).sum().to(torch.float32)
    precision = tp / (epsilon + tp + fp)
    recall = tp / (epsilon + tp + fn)
    return 2.0 * precision * recall / (precision + recall + epsilon)


class SuperviseModel(torch.nn.Module):
    """SuperviseModel(label_idx, label_dim, metric_name='f1'): __call__(inputs) reads the label slot
    (get_dense_feature(inputs, [label_idx], [label_dim])), embeds the nodes (embed, the subclass's encoder), maps the
    embedding through a bias-free out_fc (tf.layers.Dense: glorot-uniform kernel) and returns
    (embedding, mean sigmoid cross entropy, metric_name, metric of (label, sigmoid(logit))).  dim is the width of embed's
    rows, which torch needs to build out_fc.

    With streaming=False (the default) only 'f1' is provided, as each batch's own value (f1_score).  With streaming=True the
    metric is upstream's streaming one, the module model.metric (metrics.get(metric_name): 'f1', 'acc' or 'auc'): each call
    adds the batch to its device state and returns the value over every batch since construction or model.metric.reset().
    As upstream, 'auc' applies sigmoid to sigmoid(logit) again.  The metric's state is not part of the state_dict."""

    def __init__(self, label_idx, label_dim, metric_name='f1', *, dim, device=None, streaming=False):
        super().__init__()
        self.streaming = bool(streaming)
        if self.streaming:
            self.metric = metrics.get(metric_name, device)
        elif metric_name != 'f1':
            raise ValueError("metric_name must be 'f1', got %r" % (metric_name,))
        self.label_idx, self.label_dim, self.metric_name = label_idx, label_dim, metric_name
        self.out_fc = torch.nn.Linear(dim, label_dim, bias=False, device=device)
        torch.nn.init.xavier_uniform_(self.out_fc.weight)

    def embed(self, n_id):
        raise NotImplementedError

    def forward(self, inputs):
        label, = ops.get_dense_feature(inputs, [self.label_idx], [self.label_dim])
        embedding = self.embed(inputs)
        logit = self.out_fc(embedding)
        metric = (self.metric if self.streaming else f1_score)(label, torch.sigmoid(logit.detach()))
        loss = F.binary_cross_entropy_with_logits(logit, label.reshape(logit.shape))
        return embedding, loss, self.metric_name, metric


class GeniePath(SuperviseModel):
    """examples/geniepath/geniepath.py:26-48: SuperviseModel over GenieEncoder(metapath, dim, 'attention', .., head_num).
    fused, sparse_grad, device and table_dtype are passed to the encoder (see GCNEncoder); streaming to SuperviseModel."""

    def __init__(self, dim, metapath, label_idx, label_dim, max_id=-1, feature_idx=-1, feature_dim=0, use_id=False,
                 sparse_feature_idx=-1, sparse_feature_max_id=-1, embedding_dim=16, use_hash_embedding=False,
                 use_residual=False, head_num=4, metric_name='f1', fused=True, sparse_grad=False, device=None, *,
                 streaming=False, table_dtype=torch.float32):
        from .encoders import GenieEncoder
        super().__init__(label_idx, label_dim, metric_name, dim=dim, device=device, streaming=streaming)
        self._encoder = GenieEncoder(
            metapath, dim, 'attention', feature_idx=feature_idx, feature_dim=feature_dim, max_id=max_id, use_id=use_id,
            sparse_feature_idx=sparse_feature_idx, sparse_feature_max_id=sparse_feature_max_id, embedding_dim=embedding_dim,
            use_hash_embedding=use_hash_embedding, use_residual=use_residual, head_num=head_num, fused=fused,
            sparse_grad=sparse_grad, device=device, table_dtype=table_dtype)

    def embed(self, n_id):
        return self._encoder(n_id)


class LGCN(SuperviseModel):
    """examples/lgcn/lgcn.py:26-37: SuperviseModel over LGCEncoder(metapath, feature_idx, feature_dim, k, dim, nb_num,
    out_dim) -- dim is the encoder's hidden_dim and metapath its edge_type list.  The embedding is out_dim wide, so out_fc
    reads out_dim columns.  fused and device are passed to the encoder; streaming to SuperviseModel."""

    def __init__(self, dim, metapath, label_idx, label_dim, feature_idx=-1, feature_dim=0, k=3, nb_num=10, out_dim=64,
                 metric_name='f1', fused=True, device=None, *, streaming=False):
        from .encoders import LGCEncoder
        super().__init__(label_idx, label_dim, metric_name, dim=out_dim, device=device, streaming=streaming)
        self._encoder = LGCEncoder(metapath, feature_idx, feature_dim, k, dim, nb_num, out_dim, fused=fused, device=device)

    def embed(self, n_id):
        return self._encoder(n_id)
