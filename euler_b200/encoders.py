"""SparseEmbedding (tf_euler/python/utils/layers.py:152-169), the embedding the sparse-feature encoders apply to uint64
feature slots (ShallowEncoder, encoders.py:151-160; SageEncoderNew, encoders.py:590-612).

Callers size the table as the encoders do: SparseEmbedding(max_id + 1, dim) for values in [0, max_id] and
default = max_id + 1 for nodes without values, so the table has max_id + 2 rows and the default row is the last one.

Upstream quirk: ShallowEncoder's use_hash_embedding=True names layers.HashSparseEmbedding (encoders.py:117-119), which the
reference tree does not define, so that option fails there; it is not provided here either.
"""
import torch

from .ops import sparse_feature_embedding


def _truncated_normal_(t, stddev):
    """tf.truncated_normal_initializer: normal draws, those beyond two standard deviations drawn again"""
    torch.nn.init.trunc_normal_(t, mean=0.0, std=stddev, a=-2 * stddev, b=2 * stddev)
    return t


class SparseEmbedding(torch.nn.Module):
    """layers.SparseEmbedding(max_id, dim, initializer=None, combiner='sum'): a table f32[max_id + 1, dim] initialised
    truncated-normal with stddev 0.0002 (layers.py:157-165).

    __call__(sparse) takes the (indices, values, dense_shape) triple ops.get_sparse_feature returns and restates
    tf.nn.embedding_lookup_sparse(table, sp_ids, None, combiner) in torch: the reference path, composed of a gather and a
    segment sum.  lookup(nodes, feature_name, default_value) goes from node ids to the same rows in one fused device op
    (ops.sparse_feature_embedding)."""

    def __init__(self, max_id, dim, combiner='sum', device=None):
        super().__init__()
        if combiner not in ('sum', 'mean', 'sqrtn'):
            raise ValueError("combiner must be 'sum', 'mean' or 'sqrtn'")
        self.combiner = combiner
        self.embeddings = torch.nn.Parameter(_truncated_normal_(torch.empty(max_id + 1, dim, device=device), 0.0002))

    def forward(self, sparse):
        indices, values, dense_shape = sparse
        rows = indices[:, 0].long()
        n = int(dense_shape[0])
        emb = self.embeddings[values.long()]
        out = torch.zeros((n, emb.shape[1]), dtype=emb.dtype, device=emb.device).index_add(0, rows, emb)
        if self.combiner == 'sum':
            return out
        cnt = torch.zeros(n, dtype=emb.dtype, device=emb.device).index_add(0, rows, torch.ones_like(rows, dtype=emb.dtype))
        den = cnt if self.combiner == 'mean' else cnt.sqrt()
        return out / den.clamp(min=1)[:, None]

    def lookup(self, nodes, feature_name, default_value):
        return sparse_feature_embedding(nodes, feature_name, self.embeddings, default_value, self.combiner)
