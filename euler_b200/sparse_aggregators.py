"""The full-neighbourhood aggregators of GCNEncoder / GenieEncoder (tf_euler/python/utils/sparse_aggregators.py) in torch,
with upstream's constructor arguments after in_dim (the width of the inputs, which torch needs up front): GCNAggregator,
MeanAggregator, SingleAttentionAggregator, AttentionAggregator and get(name).

Each takes (self_embedding [n, Din], neigh_embedding [m, Din], adj) where adj is one hop of ops.get_multi_hop_neighbor,
(indptr i64[n+1], cols i64[nnz], weights): row i's entries are (i, cols[k]) for k in [indptr[i], indptr[i+1]).  As
upstream (_sparse_ones_like), the weights are ignored and every entry counts once, multi-edges included.

fused=True (the default) runs the hot part on the device:
    'gcn', 'mean'   the neighbour mean S / max(deg, 1e-7) is one ops.adjacency_mean; 'gcn' adds self_embedding after the
                    division, as upstream writes it
    'attention'     every head's dense kernel stacked into one [Din, H*C] GEMM, the per-head self / neighbour scores, then
                    one ops.gat_attention_aggregate over the edges (row, cols) for all heads: leaky_relu slope 0.2 and a
                    softmax per row less its maximum, as tf.nn.leaky_relu and tf.sparse_softmax; a row without entries gives
                    zeros.  That op synchronises once per call (to check that its targets are sorted; they are), and it
                    gives each row's entries to one lane group: on hops with rows of ~10^3 entries and more it was measured
                    slower than the composition (DESIGN §3.16), though it never writes the [nnz, H*C] messages
renorm=True always takes the composition: GCNEncoder never passes it.  fused=False is the literal composition in plain
torch (index_select / index_add and a per-row softmax), which runs on CPU tensors and in float64.
"""
import torch
import torch.nn.functional as F

from . import ops
from .encoders import Dense


def _entry_rows(indptr, nnz):
    """each entry's row, i64[nnz] (no host synchronisation)"""
    n = indptr.numel() - 1
    return torch.repeat_interleave(torch.arange(n, device=indptr.device), indptr[1:] - indptr[:-1], output_size=nnz)


def _degree(indptr, dtype):
    return (indptr[1:] - indptr[:-1]).to(dtype)[:, None]


def _adj_sum(neigh, indptr, cols):
    """sparse_tensor_dense_matmul(ones-like adj, neigh): the sum of each row's neighbour rows"""
    rows = _entry_rows(indptr, cols.numel())
    out = torch.zeros((indptr.numel() - 1, neigh.shape[1]), dtype=neigh.dtype, device=neigh.device)
    return out.index_add(0, rows, neigh.index_select(0, cols))


def _adj_mean(neigh, adj, fused):
    indptr, cols = adj[0], adj[1]
    if fused:
        return ops.adjacency_mean(neigh, (indptr, cols))
    return _adj_sum(neigh, indptr, cols) / torch.clamp(_degree(indptr, neigh.dtype), min=1e-7)


def _segment_softmax(logits, rows, n):
    """tf.sparse_softmax over the entries of each row: exp(v - row max) / row sum; logits [nnz, H]"""
    H = logits.shape[1]
    idx = rows[:, None].expand(-1, H)
    mx = torch.full((n, H), float('-inf'), dtype=logits.dtype, device=logits.device).scatter_reduce(0, idx, logits, 'amax')
    e = torch.exp(logits - mx.index_select(0, rows))
    s = torch.zeros((n, H), dtype=logits.dtype, device=logits.device).index_add(0, rows, e)
    return e / s.index_select(0, rows)


class GCNAggregator(torch.nn.Module):
    """sparse_aggregators.py:37-54: dense(self + S / max(deg, 1e-7)), or with renorm dense((self + S) / (1 + deg))"""

    def __init__(self, in_dim, dim, activation=torch.relu, renorm=False, fused=True, device=None, **kwargs):
        super().__init__()
        self.renorm = renorm
        self.fused = fused
        self.dense = Dense(in_dim, dim, activation=activation, device=device)
        self.output_dim = dim

    def forward(self, inputs):
        self_embedding, neigh_embedding, adj = inputs
        if self.renorm:
            indptr, cols = adj[0], adj[1]
            agg = (self_embedding + _adj_sum(neigh_embedding, indptr, cols)) / (1. + _degree(indptr, neigh_embedding.dtype))
        else:
            agg = self_embedding + _adj_mean(neigh_embedding, adj, self.fused)
        return self.dense(agg)


class MeanAggregator(torch.nn.Module):
    """sparse_aggregators.py:57-84: self_layer(self) + neigh_layer(S / max(deg, 1e-7)), or their concatenation (dim halved,
    rounding down, as upstream)"""

    def __init__(self, in_dim, dim, activation=torch.relu, concat=False, fused=True, device=None, **kwargs):
        super().__init__()
        if concat:
            dim //= 2
        self.concat = concat
        self.fused = fused
        self.self_layer = Dense(in_dim, dim, activation=activation, device=device)
        self.neigh_layer = Dense(in_dim, dim, activation=activation, device=device)
        self.output_dim = 2 * dim if concat else dim

    def forward(self, inputs):
        self_embedding, neigh_embedding, adj = inputs
        from_self = self.self_layer(self_embedding)
        from_neighs = self.neigh_layer(_adj_mean(neigh_embedding, adj, self.fused))
        return torch.cat([from_self, from_neighs], 1) if self.concat else from_self + from_neighs


def _attention_composed(self_embedding, neigh_embedding, adj, kernel, w_self, w_neigh, renorm):
    """sparse_aggregators.py:87-124 for H heads at once: kernel [Din, H*C], w_self / w_neigh [H, C] (each head's
    self_layer / neigh_layer kernel); returns the heads' outputs before the activation, [n, H*C]"""
    indptr, cols = adj[0], adj[1]
    n, H = self_embedding.shape[0], w_self.shape[0]
    rows = _entry_rows(indptr, cols.numel())
    if renorm:   # [eye | adj]: every row first attends to itself, column i of from_all
        from_all = torch.cat([self_embedding, neigh_embedding], 0) @ kernel
        from_self = from_all[:n]
        ar = torch.arange(n, device=rows.device)
        rows, cols = torch.cat([ar, rows]), torch.cat([ar, cols + n])
    else:
        from_all = neigh_embedding @ kernel
        from_self = self_embedding @ kernel
    C = kernel.shape[1] // H
    self_weight = (from_self.reshape(n, H, C) * w_self).sum(-1)
    all_weight = (from_all.reshape(-1, H, C) * w_neigh).sum(-1)
    coef = F.leaky_relu(self_weight.index_select(0, rows) + all_weight.index_select(0, cols), 0.2)
    coef = _segment_softmax(coef, rows, n)
    msg = (coef[:, :, None] * from_all.index_select(0, cols).reshape(-1, H, C)).reshape(-1, H * C)
    output = torch.zeros((n, H * C), dtype=msg.dtype, device=msg.device).index_add(0, rows, msg)
    return output if renorm else from_self + output


class SingleAttentionAggregator(torch.nn.Module):
    """sparse_aggregators.py:87-124: one attention head of width dim"""

    def __init__(self, in_dim, dim, activation=torch.relu, renorm=False, fused=True, device=None, **kwargs):
        super().__init__()
        self.dense = Dense(in_dim, dim, device=device)
        self.self_layer = Dense(dim, 1, device=device)
        self.neigh_layer = Dense(dim, 1, device=device)
        self.activation = activation
        self.renorm = renorm
        self.fused = fused
        self.output_dim = dim

    def forward(self, inputs):
        return _attention([self], inputs, self.activation, self.renorm, self.fused)


def _attention(heads, inputs, activation, renorm, fused):
    self_embedding, neigh_embedding, adj = inputs
    kernel = torch.cat([h.dense.kernel for h in heads], 1)
    w_self = torch.stack([h.self_layer.kernel[:, 0] for h in heads])
    w_neigh = torch.stack([h.neigh_layer.kernel[:, 0] for h in heads])
    if fused and not renorm:
        out = _attention_fused(self_embedding, neigh_embedding, adj, kernel, w_self, w_neigh)
    else:
        out = _attention_composed(self_embedding, neigh_embedding, adj, kernel, w_self, w_neigh, renorm)
    return activation(out) if activation else out


def _attention_fused(self_embedding, neigh_embedding, adj, kernel, w_self, w_neigh):
    indptr, cols = adj[0], adj[1]
    n, m, H = self_embedding.shape[0], neigh_embedding.shape[0], w_self.shape[0]
    C = kernel.shape[1] // H
    from_all = neigh_embedding @ kernel
    from_self = self_embedding @ kernel
    s_dst = (from_self.reshape(n, H, C) * w_self).sum(-1)
    s_src = (from_all.reshape(m, H, C) * w_neigh).sum(-1)
    edge_index = torch.stack([_entry_rows(indptr, cols.numel()), cols])
    return from_self + ops.gat_attention_aggregate(from_all, s_dst, s_src, edge_index, (n, m))


class AttentionAggregator(torch.nn.Module):
    """sparse_aggregators.py:127-137: head_num SingleAttentionAggregators of width dim // head_num, concatenated"""

    def __init__(self, in_dim, dim, head_num=4, activation=torch.relu, renorm=False, fused=True, device=None, **kwargs):
        super().__init__()
        dim //= head_num
        self.attentions = torch.nn.ModuleList(
            [SingleAttentionAggregator(in_dim, dim, activation, renorm, fused, device=device) for _ in range(head_num)])
        self.activation = activation
        self.renorm = renorm
        self.fused = fused
        self.output_dim = head_num * dim

    def forward(self, inputs):
        return _attention(list(self.attentions), inputs, self.activation, self.renorm, self.fused)


aggregators = {
    'gcn': GCNAggregator,
    'mean': MeanAggregator,
    'attention': AttentionAggregator
}


def get(aggregator):
    return aggregators.get(aggregator)
