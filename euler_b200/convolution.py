"""Message-passing blocks of tf_euler's convolutions over the euler_b200 mp ops (gather / scatter_*): the access patterns of
GCNConv and RelationConv (SURVEY.md section 8a, row a-13).  The dense layers (tf.layers.Dense, the per-relation matmul) stay
with the framework (torch here): they are GEMMs, not part of the sampling / aggregation path.

  gcn_aggregate      tf_euler/python/convolution/gcn_conv.py:32-48   deg^-1/2 norms via scatter_add(ones) on both sides of
                                                                      edge_index, gather of x_j and of both norms, scatter_add
  relation_aggregate tf_euler/python/convolution/relation_conv.py:53-70  x_j gathered, transformed by its relation's matrix
                                                                      (unique -> gather -> matmul), scatter_mean to the targets
  relation_aggregate_fused  the same, fused: rows summed per (target, relation) pair, one matvec per pair
                                                                      (ops.relation_mean_aggregate)
  sage_aggregate     tf_euler/python/convolution/sage_conv.py:33-38   gather(x, edge_index[1]) -> scatter_mean
  gat_aggregate      tf_euler/python/convolution/gat_conv.py:53-78    per-node attention scores, then the fused softmax-weighted
                                                                      sum over each target's edges (ops.gat_attention_aggregate)
  agnn_aggregate     tf_euler/python/convolution/agnn_conv.py:32-54   l2_normalize in torch, then the fused cosine logits,
                                                                      softmax and weighted sum (ops.agnn_attention_aggregate)
  group_dense        tf_euler/python/convolution/dna_conv.py:27-69    GroupDense: a block-diagonal matmul plus bias
  dna_aggregate      tf_euler/python/convolution/dna_conv.py:115-170  lin_q / lin_k / lin_v per node, gcn_norm, then the fused
                                                                      head-by-head attention and scatter_mean
                                                                      (ops.dna_attention_aggregate)
"""
import torch

from . import ops
from ._lib import EulerError


def gcn_norm(edge_index, size):
    """GCNConv.norm (gcn_conv.py:32-40): (deg_0 ** -0.5, deg_1 ** -0.5), deg_i = scatter_add(ones, edge_index[i], size[i])"""
    e = edge_index.shape[1]
    ones = torch.ones((e, 1), dtype=torch.float32, device=edge_index.device)
    return tuple(ops.scatter_add(ones, edge_index[i].to(torch.int32), int(size[i])) ** -0.5 for i in (0, 1))


def gcn_aggregate(x, edge_index, size):
    """GCNConv.__call__ up to (not including) the Dense layer (gcn_conv.py:42-55): x = (x_target, x_source) or one tensor for
    both sides; returns scatter_add(norm_i * norm_j * x_j, edge_index[0], size[0])."""
    x0, x1 = (x, x) if torch.is_tensor(x) else (x[0], x[1] if x[1] is not None else x[0])
    del x0
    idx0, idx1 = edge_index[0].to(torch.int32), edge_index[1].to(torch.int32)
    n0, n1 = gcn_norm(edge_index, size)
    x_j = ops.gather(x1, idx1)
    out = ops.gather(n0, idx0) * ops.gather(n1, idx1) * x_j
    return ops.scatter_add(out, idx0, int(size[0]))


def relation_aggregate(x, edge_index, size, edge_attr, matrix):
    """RelationConv.__call__ up to apply_node (relation_conv.py:53-70): matrix f32[num_relations, dim, fea_dim];
    out[i] = mean over edges e with target i of matrix[edge_attr[e]] @ x_source[edge_index[1][e]]."""
    x1 = x if torch.is_tensor(x) else (x[1] if x[1] is not None else x[0])
    idx0, idx1 = edge_index[0].to(torch.int32), edge_index[1].to(torch.int32)
    x_j = ops.gather(x1, idx1)
    rel, inv = torch.unique(edge_attr, return_inverse=True)          # tf.unique + the two gathers of apply_edge
    m = matrix[rel][inv]                                             # [E, dim, fea_dim]
    out = torch.matmul(m, x_j.unsqueeze(-1)).squeeze(-1)
    return ops.scatter_mean(out, idx0, int(size[0]))


def relation_aggregate_fused(x, edge_index, size, edge_attr, matrix):
    """relation_aggregate's signature and result, to rounding, as one fused device op (ops.relation_mean_aggregate): the edges
    are summed per (target, relation) pair and each pair is transformed once, so no [E, dim, fea_dim] matrix and no [E, dim]
    message is ever made."""
    x1 = x if torch.is_tensor(x) else (x[1] if x[1] is not None else x[0])
    return ops.relation_mean_aggregate(x1, matrix, edge_attr, edge_index, size)


def sage_aggregate(x, edge_index, size):
    """SAGEConv's neighbor mean (sage_conv.py:33-38): scatter_mean(gather(x_source, edge_index[1]), edge_index[0], size[0])"""
    x1 = x if torch.is_tensor(x) else (x[1] if x[1] is not None else x[0])
    return ops.scatter_mean(ops.gather(x1, edge_index[1].to(torch.int32)), edge_index[0].to(torch.int32), int(size[0]))


def gat_aggregate(x, edge_index, size, att_i, att_j, improved=False, aggr='add'):
    """GATConv.__call__ after its `fc` (gat_conv.py:53-78), for H heads of width C laid out as the concatenation of H
    single-head convs (gat.py's calculate_conv): x = (x_target, x_source), both already projected to [n, H*C]; att_i, att_j
    [H, C] are the weights of the two Attention layers (Dense(1) per head).  The scores att_i(x_i) and att_j(x_j) are
    computed once per node here, in torch, so autograd reaches att_* and x through them; the softmax-weighted sum over
    each target's edges is the fused device op.  improved adds x_target.  Head averaging (concat=False) stays with the
    caller.  Only aggr='add' (GATConv's default) is built."""
    if aggr != 'add':
        raise EulerError("gat_aggregate: aggr=%r is not built here; GATConv's aggregation is 'add'" % (aggr,))
    if torch.is_tensor(x) or x[0] is None:
        raise EulerError("gat_aggregate: x must be (x_target, x_source): att_i scores the targets")
    x0, x1 = x[0], x[1] if x[1] is not None else x[0]
    if att_i.dim() != 2 or att_j.shape != att_i.shape:
        raise EulerError("gat_aggregate: att_i and att_j must both be [H, C]; got %s, %s" % (tuple(att_i.shape), tuple(att_j.shape)))
    H, C = att_i.shape
    if x0.dim() != 2 or x1.dim() != 2 or x0.shape[1] != H * C or x1.shape[1] != H * C:
        raise EulerError("gat_aggregate: x_target and x_source must be [n, H*C] = [n, %d]; got %s, %s"
                         % (H * C, tuple(x0.shape), tuple(x1.shape)))
    s_dst = (x0.reshape(x0.shape[0], H, C) * att_i).sum(-1)
    s_src = (x1.reshape(x1.shape[0], H, C) * att_j).sum(-1)
    out = ops.gat_attention_aggregate(x1, s_dst, s_src, edge_index, size)
    return x0 + out if improved else out


def l2_normalize(x):
    """tf.nn.l2_normalize(x, axis=-1) as TF writes it: x * rsqrt(max(sum(x * x, -1), 1e-12))"""
    return x * torch.rsqrt(torch.clamp_min((x * x).sum(-1, keepdim=True), 1e-12))


def agnn_aggregate(x, edge_index, size, beta):
    """AGNNConv.__call__ (agnn_conv.py:32-54): x = (x_target, x_source), x_source None meaning x_target; beta the conv's
    trainable scalar (a one-element tensor, upstream tf.Variable([1.])).  l2_normalize runs here, in torch, so autograd
    reaches x through it; the cosine logits, the softmax over each target's edges and the weighted sum of the (raw) source
    rows are the fused device op.  apply_node is the identity."""
    if torch.is_tensor(x) or x[0] is None:
        raise EulerError("agnn_aggregate: x must be (x_target, x_source): the logits read the normalized targets")
    x0, x1 = x[0], x[1] if x[1] is not None else x[0]
    if not torch.is_tensor(beta) or beta.numel() != 1:
        raise EulerError("agnn_aggregate: beta must be a one-element tensor")
    if x0.dim() != 2 or x1.dim() != 2 or x0.shape[1] != x1.shape[1]:
        raise EulerError("agnn_aggregate: x_target and x_source must be [n, D] of one width; got %s, %s"
                         % (tuple(x0.shape), tuple(x1.shape)))
    n1 = l2_normalize(x1)
    n0 = n1 if x0 is x1 else l2_normalize(x0)
    return ops.agnn_attention_aggregate(x1, n0, n1, beta, edge_index, size)


def group_dense(x, kernel, bias=None):
    """GroupDense.call (dna_conv.py:50-69) without activation: kernel [G, in/G, out/G] is a block-diagonal matmul, group g
    mapping input columns [g*in/G, (g+1)*in/G) to output columns [g*out/G, (g+1)*out/G); bias [out] is added when given.
    G = 1 is a plain dense layer with kernel[0] (upstream's G = 1 branch reshapes the list [kernel, bias] and fails with a
    bias; DESIGN section 4)."""
    if not torch.is_tensor(x) or not torch.is_tensor(kernel) or x.dtype != torch.float32 or kernel.dtype != torch.float32:
        raise EulerError("group_dense: x and kernel must be float32 tensors")
    if kernel.dim() != 3 or x.dim() < 1:
        raise EulerError("group_dense: kernel must be [groups, in/groups, out/groups]; got %s" % (tuple(kernel.shape),))
    G, fi, fo = kernel.shape
    if G < 1 or x.shape[-1] != G * fi:
        raise EulerError("group_dense: x's width %d is not groups * in/groups = %d * %d" % (x.shape[-1], G, fi))
    if bias is not None and (not torch.is_tensor(bias) or bias.dtype != torch.float32 or bias.shape != (G * fo,)):
        raise EulerError("group_dense: bias must be a float32 [%d] tensor" % (G * fo))
    lead = x.shape[:-1]
    if G == 1:
        out = x.reshape(-1, fi) @ kernel[0]
    else:
        out = torch.matmul(x.reshape(-1, G, fi).transpose(0, 1), kernel).transpose(0, 1).reshape(-1, G * fo)
    if bias is not None:
        out = out + bias
    return out.reshape(*lead, G * fo)


def dna_aggregate(x, edge_index, size, lin_q, lin_k, lin_v, heads):
    """DNAConv.__call__ after in_fc (dna_conv.py:149-170): x = (x_target, x_source), both already through in_fc, x_source
    None meaning x_target; lin_q, lin_k and lin_v are (kernel, bias) pairs of GroupDense layers (bias may be None).  The
    linear maps act on each row, so they run here once per node (q on the targets, k and v on the sources) instead of once
    per edge; then gcn_norm and the fused attention, norm product and scatter_mean (ops.dna_attention_aggregate).
    apply_node is the identity."""
    if torch.is_tensor(x) or not isinstance(x, (tuple, list)) or len(x) != 2 or x[0] is None:
        raise EulerError("dna_aggregate: x must be (x_target, x_source): the queries read the targets")
    x0, x1 = x[0], x[1] if x[1] is not None else x[0]
    pairs = (("lin_q", lin_q), ("lin_k", lin_k), ("lin_v", lin_v))
    for nm, p in pairs:
        if not isinstance(p, (tuple, list)) or len(p) != 2:
            raise EulerError("dna_aggregate: %s must be a (kernel, bias) pair" % nm)
    if any(not torch.is_tensor(t) or t.dim() != 2 for t in (x0, x1)) or x0.shape[1] != x1.shape[1]:
        raise EulerError("dna_aggregate: x_target and x_source must be 2-D tensors of one width")
    dim = lin_q[0].shape[0] * lin_q[0].shape[2] if torch.is_tensor(lin_q[0]) and lin_q[0].dim() == 3 else None
    if dim is None or int(heads) < 1 or dim % int(heads):
        raise EulerError("dna_aggregate: dim = %s must be a positive multiple of heads = %s" % (dim, heads))
    q = group_dense(x0, *lin_q)
    k = group_dense(x1, *lin_k)
    v = group_dense(x1, *lin_v)
    n0, n1 = gcn_norm(edge_index, size)
    return ops.dna_attention_aggregate(q, k, v, n0, n1, edge_index, size, heads)
