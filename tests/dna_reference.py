"""DNAConv (tf_euler/python/convolution/dna_conv.py) restated in torch, for the CPU semantics test and the GPU tests.

literal_*: the upstream code line by line (reshapes, transposes and the [0] of restricted_softmax included), in whatever
dtype and device the inputs have.  closed_form_messages: the per-edge closed form the fused op implements
(include/euler_b200.h, eu_dna_aggregate)."""
import math

import torch


def literal_group_dense(inputs, kernel, bias, groups, dim):
    """GroupDense.call (dna_conv.py:50-69), activation None; for groups = 1 the kernel alone is reshaped (self.weights
    without a bias)"""
    if groups > 1:
        shape = list(inputs.shape)
        out_shape = shape[:-1] + [dim]
        x = inputs.reshape(-1, groups, shape[-1] // groups).permute(1, 0, 2)
        out = torch.matmul(x, kernel).permute(1, 0, 2).reshape(out_shape)
    else:
        out = torch.matmul(inputs, kernel.reshape(-1, dim))
    if bias is not None:
        out = out + bias
    return out


def literal_restricted_softmax(inputs):
    """restricted_softmax (dna_conv.py:72-80), dim = -1, margin = 0"""
    input_max = inputs.max(dim=-1, keepdim=True).values[0]
    input_max = input_max.clamp(0, torch.finfo(torch.float32).max)
    out = torch.exp(inputs - input_max)
    return out / (out.sum(-1, keepdim=True) + torch.exp(0 - input_max))


def literal_attention(query, key, value):
    """DNAConv.attention (dna_conv.py:115-124)"""
    score = torch.matmul(query, key.permute(0, 1, 3, 2))
    score = score / torch.sqrt(torch.tensor(float(key.shape[-1]), dtype=score.dtype, device=score.device))
    return torch.matmul(literal_restricted_softmax(score), value)


def literal_multi_head(query, key, value, lin_q, lin_k, lin_v, heads, groups, dim):
    """DNAConv.multi_head (dna_conv.py:126-147); lin_* = (kernel, bias)"""
    query = literal_group_dense(query, *lin_q, groups, dim)
    key = literal_group_dense(key, *lin_k, groups, dim)
    value = literal_group_dense(value, *lin_v, groups, dim)
    c = dim // heads
    query = query.reshape(-1, query.shape[1], heads, c).permute(1, 0, 2, 3)
    key = key.reshape(-1, key.shape[1], heads, c).permute(1, 0, 2, 3)
    value = value.reshape(-1, value.shape[1], heads, c).permute(1, 0, 2, 3)
    out = literal_attention(query, key, value).permute(1, 0, 2, 3)
    return out.reshape(-1, query.shape[1], dim)


def literal_apply_edge(x_i, x_j, norm_i, norm_j, lin_q, lin_k, lin_v, heads, groups, dim):
    """DNAConv.apply_edge (dna_conv.py:165-170): multi_head's out_shape reads the transposed query's axis 1 (E), so its
    result is [1, E, dim] and the squeeze of axis 0 leaves [E, dim]"""
    out = literal_multi_head(x_i.unsqueeze(1), x_j.unsqueeze(1), x_j.unsqueeze(1), lin_q, lin_k, lin_v, heads, groups, dim)
    return norm_i * norm_j * out.squeeze(0)


def gcn_norm(ei, size, dtype):
    """DNAConv.norm (dna_conv.py:105-113): deg^-1/2 of both sides, [n, 1]"""
    return tuple((torch.zeros(int(size[i]), dtype=dtype).index_add(0, ei[i], torch.ones(ei.shape[1], dtype=dtype)) ** -0.5)
                 .reshape(-1, 1) for i in (0, 1))


def scatter_mean(msg, idx, n):
    s = torch.zeros((n, msg.shape[1]), dtype=msg.dtype, device=msg.device).index_add(0, idx, msg)
    cnt = torch.zeros(n, dtype=msg.dtype, device=msg.device).index_add(0, idx, torch.ones(idx.shape[0], dtype=msg.dtype,
                                                                                          device=msg.device))
    return s / (cnt[:, None] + 1e-7)


def literal_dna_layer(x_tgt, x_src, ei, size, in_fc, lin_q, lin_k, lin_v, heads, groups):
    """DNAConv.__call__ (dna_conv.py:149-163) on the CPU: in_fc [dim, in] (Dense without bias), gather, apply_edge,
    scatter_mean"""
    dim = in_fc.shape[0]
    x0, x1 = x_tgt @ in_fc.T, x_src @ in_fc.T
    n0, n1 = gcn_norm(ei, size, x0.dtype)
    msg = literal_apply_edge(x0[ei[0]], x1[ei[1]], n0[ei[0]], n1[ei[1]], lin_q, lin_k, lin_v, heads, groups, dim)
    return scatter_mean(msg, ei[0], int(size[0]))


def closed_form_messages(q_e, k_e, v_e, w_e, heads):
    """the per-edge closed form: q_e, k_e, v_e [E, H*C] (the rows of each edge), w_e [E] the norm product; returns the
    messages [E, H*C] and a [E, H, H]"""
    E, dim = q_e.shape
    c = dim // heads
    q, k, v = (t.reshape(E, heads, c) for t in (q_e, k_e, v_e))
    s = torch.einsum("ehc,egc->ehg", q, k) / math.sqrt(c)
    m = torch.clamp_min(s.max(-1, keepdim=True).values, 0)
    ex = torch.exp(s - m)
    a = ex / (ex.sum(-1, keepdim=True) + torch.exp(-m))
    return w_e[:, None] * torch.einsum("ehg,egc->ehc", a, v).reshape(E, dim), a
