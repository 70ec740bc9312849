"""The graph auto-encoders of tf_euler: BaseGraphAutoEncoder (tf_euler/python/mp_utils/base_gae.py) and the GAE / VGAE models
of examples/gae/gae.py, over any node encoder.

An encoder is any callable that maps int64 node ids [N] to rows [N, dim] (encoders.SageEncoder, encoders.GCNEncoder,
encoders.ShallowEncoder, ..); a module encoder is a submodule, so model.parameters() lists its tensors.  to_sample draws on
the device in upstream's order -- sample_neighbor(inputs, edge_type, num_negs, max_id + 1), then sample_node(B * num_negs,
node_type) -- and __call__ embeds src, pos, negs and then inputs, in that order, so an encoder that samples draws as
upstream's does.  __call__(inputs) returns upstream's (embedding, loss, 'acc', acc) with the embedding [B, 1, dim].

fused=True (the default) computes the step after the encoders -- the logits, the sigmoid cross entropy, acc and, for VGAE,
the reparameterisation and the KL term -- in one device op, ops.gae_loss; fused=False is the literal torch composition of
base_gae.py / gae.py (composed_gae_loss), which consumes the same draws and the same noise.

streaming=True makes acc upstream's streaming tf.metrics.accuracy: the device module model.metric
(metrics.StreamingAccuracy), whose value covers every batch since construction or model.metric.reset().  The fused path adds
ops.gae_loss's correct count of the 2BK predictions to it (no second pass); fused=False adds the composed predictions.

Departures from upstream: the encoder is injected (examples/gae builds GNN(BaseGNNNet), which this package does not have);
by default acc is the batch's own value, where upstream's is the streaming tf.metrics.accuracy (streaming=True gives that);
VGAE returns the mu rows as its embedding, where upstream returns the tuple (mu, log_var, emb) in that slot.
"""
import math

import torch

from . import metrics, ops
from .encoders import ShallowEncoder
from .solution import acc_score
from .unsupervised import xent_loss


def composed_gae_loss(emb, emb_pos, emb_negs, metric=acc_score):
    """base_gae.py's step after the encoders, literally: emb [B, 1, dim], emb_pos and emb_negs [B, K, dim] -> (loss, acc),
    acc = metric(label, predict) (acc_score, or a streaming metrics.StreamingAccuracy)"""
    logits = torch.matmul(emb, emb_pos.transpose(1, 2))
    neg_logits = torch.matmul(emb, emb_negs.transpose(1, 2))
    loss = xent_loss(logits, neg_logits)
    predict, neg_predict = torch.sigmoid(logits.detach()), torch.sigmoid(neg_logits.detach())
    label = torch.cat([torch.ones_like(predict), torch.zeros_like(neg_predict)], 2)
    return loss, metric(label, torch.cat([predict, neg_predict], 2))


def kl(mu, log_var):
    """VariationalGraphAutoEncoder.kl: -0.5 (log_var - exp(log_var) - mu^2 + 1), flattened"""
    return (-0.5 * (log_var - torch.exp(log_var) - torch.pow(mu, 2) + 1)).reshape(-1)


def _fused_acc(correct, logits_count):
    return correct.to(torch.float32) / logits_count


class BaseGraphAutoEncoder(torch.nn.Module):
    """BaseGraphAutoEncoder(node_type, edge_type, max_id, num_negs=20): num_negs positives per input from sample_neighbor over
    edge_type (default node max_id + 1) and num_negs negatives per input from sample_node of node_type.  A subclass provides
    embed(n_id) -> [B, n, dim] rows.  streaming=True makes acc the streaming model.metric (see the top of the file)."""

    def __init__(self, node_type, edge_type, max_id, num_negs=20, fused=True, *, streaming=False):
        super().__init__()
        if int(num_negs) < 1:
            raise ValueError("num_negs must be at least 1, got %r" % (num_negs,))
        self.node_type = node_type
        self.edge_type = edge_type
        self.max_id = max_id
        self.num_negs = int(num_negs)
        self.fused = fused
        self.streaming = bool(streaming)
        if self.streaming:
            self.metric = metrics.StreamingAccuracy()

    def to_sample(self, inputs):
        batch_size = inputs.numel()
        src = inputs.reshape(-1, 1)
        pos = ops.sample_neighbor(inputs, self.edge_type, self.num_negs, self.max_id + 1)[0]
        negs = ops.sample_node(batch_size * self.num_negs, self.node_type).reshape(batch_size, self.num_negs)
        return src, pos, negs

    def embed(self, n_id):
        raise NotImplementedError

    def fused_acc(self, correct, logits_count):
        """acc from the fused op's correct count of logits_count predictions"""
        return self.metric.add_counts(correct, logits_count) if self.streaming else _fused_acc(correct, logits_count)

    def composed_metric(self):
        """the acc of the composed step: acc_score, or the streaming metric"""
        return self.metric if self.streaming else acc_score

    def loss_and_acc(self, emb, emb_pos, emb_negs):
        """the step after the encoders: (loss, acc), fused or composed"""
        if self.fused:
            loss, correct = ops.gae_loss(emb, emb_pos, emb_negs)
            return loss, self.fused_acc(correct, 2 * emb_pos.shape[0] * emb_pos.shape[1])
        return composed_gae_loss(emb, emb_pos, emb_negs, self.composed_metric())

    def embedding(self, rows):
        """the returned embedding of embed(inputs)'s result"""
        return rows

    def forward(self, inputs):
        src, pos, negs = self.to_sample(inputs)
        embedding = self.embed(src)
        embedding_pos = self.embed(pos)
        embedding_negs = self.embed(negs)
        loss, acc = self.loss_and_acc(embedding, embedding_pos, embedding_negs)
        embedding = self.embedding(self.embed(inputs))
        return embedding, loss, 'acc', acc


def _rows(encoder, n_id):
    """encoder(n_id) reshaped as upstream's embed does: [batch, -1, dim]"""
    emb = encoder(n_id.reshape(-1))
    return emb.reshape(n_id.shape[0], -1, emb.shape[-1])


class GraphAutoEncoder(BaseGraphAutoEncoder):
    """GraphAutoEncoder (examples/gae/gae.py) over the node encoder `encoder`: embed(n_id) = encoder(n_id) as [B, n, dim]."""

    def __init__(self, encoder, node_type, edge_type, max_id, num_negs=5, fused=True, *, streaming=False):
        super().__init__(node_type, edge_type, max_id, num_negs, fused=fused, streaming=streaming)
        if not callable(encoder):
            raise ValueError("encoder must map node ids to rows, got %r" % (encoder,))
        self.encoder = encoder

    def embed(self, n_id):
        return _rows(self.encoder, n_id)


def _encoder_dim(encoder):
    """the width of an encoder's rows: dims[-1] (SageEncoder, GCNEncoder), else output_dim or dim"""
    dims = getattr(encoder, 'dims', None)
    if dims:
        return int(dims[-1])
    for name in ('output_dim', 'dim'):
        d = getattr(encoder, name, None)
        if isinstance(d, int):
            return d
    raise ValueError("the encoder's row width is unknown: pass dim")


class VariationalGraphAutoEncoder(BaseGraphAutoEncoder):
    """VariationalGraphAutoEncoder (examples/gae/gae.py) over the node encoder `encoder`, which gives mu.  log_var_encoder is
    ShallowEncoder(dim=dim, feature_idx=-1, max_id=max_id, combiner='add'), as upstream; dim is the encoder's row width
    (dims[-1], output_dim or dim) unless given.  embed(n_id) returns (mu, log_var, noise), each [B, n, dim]: with train=True
    noise is torch.randn from `generator` (the rows are emb = mu + radius * noise * sqrt(exp(log_var))), with train=False it
    is None and emb = mu.  The loss adds mean(kl) over src, pos and negs; the returned embedding is the mu rows."""

    def __init__(self, radius, encoder, node_type, edge_type, max_id, num_negs=5, train=True, generator=None, fused=True,
                 dim=None, device=None, *, streaming=False):
        super().__init__(node_type, edge_type, max_id, num_negs, fused=fused, streaming=streaming)
        if not callable(encoder):
            raise ValueError("encoder must map node ids to rows, got %r" % (encoder,))
        self.radius = float(radius)
        if not math.isfinite(self.radius):
            raise ValueError("radius must be finite, got %r" % (radius,))
        self.encoder = encoder
        self.dim = int(dim) if dim is not None else _encoder_dim(encoder)
        self.log_var_encoder = ShallowEncoder(dim=self.dim, feature_idx=-1, max_id=max_id, combiner='add', fused=fused,
                                              device=device)
        self.train_mode = train
        self.generator = generator

    def kl(self, mu, log_var):
        return kl(mu, log_var)

    def embed(self, n_id):
        mu = _rows(self.encoder, n_id)
        log_var = _rows(self.log_var_encoder, n_id)
        noise = None
        if self.train_mode:
            noise = torch.randn(log_var.shape, generator=self.generator, dtype=torch.float32, device=log_var.device)
        return mu, log_var, noise

    def reparameterize(self, mu, log_var, noise):
        """emb = mu + radius * noise * sqrt(exp(log_var)), or mu without noise"""
        return mu if noise is None else mu + self.radius * noise * torch.sqrt(torch.exp(log_var))

    def loss_and_acc(self, emb, emb_pos, emb_negs):
        (mu, lv, nz), (mu_p, lv_p, nz_p), (mu_n, lv_n, nz_n) = emb, emb_pos, emb_negs
        if self.fused:
            loss, correct = ops.gae_loss(mu, mu_p, mu_n, log_var=(lv, lv_p, lv_n),
                                         noise=None if nz is None else (nz, nz_p, nz_n), radius=self.radius)
            return loss, self.fused_acc(correct, 2 * mu_p.shape[0] * mu_p.shape[1])
        loss, acc = composed_gae_loss(self.reparameterize(mu, lv, nz), self.reparameterize(mu_p, lv_p, nz_p),
                                      self.reparameterize(mu_n, lv_n, nz_n), self.composed_metric())
        kls = torch.cat([self.kl(mu, lv), self.kl(mu_p, lv_p), self.kl(mu_n, lv_n)], 0)
        return loss + torch.mean(kls), acc

    def embedding(self, rows):
        return rows[0]
