"""DNAConv's semantics on the CPU (torch, float64), no GPU: the literal restatement of dna_conv.py (reshapes and transposes
included) equals the per-edge closed form the fused op implements; convolution.group_dense equals GroupDense.call; and the
linear maps hoisted to once per node equal the per-edge application."""
import numpy as np
import pytest
import torch

import dna_reference as ref


def rand(rs, *shape):
    return torch.from_numpy(rs.randn(*shape))


def lin(rs, groups, dim, bias=True):
    return rand(rs, groups, dim // groups, dim // groups) * 0.4, (rand(rs, dim) * 0.1 if bias else None)


@pytest.mark.parametrize("heads", [1, 2, 4])
@pytest.mark.parametrize("groups", [1, 8])
def test_literal_restatement_equals_the_closed_form(heads, groups):
    rs = np.random.RandomState(heads * 10 + groups)
    dim, E = 32, 50
    x_i, x_j = rand(rs, E, dim), rand(rs, E, dim)
    n_i, n_j = rand(rs, E, 1).abs(), rand(rs, E, 1).abs()
    x_i[3] *= 20.0                                         # large logits: exp(-m) underflows against the scores
    lq, lk, lv = (lin(rs, groups, dim, bias=groups > 1) for _ in range(3))
    lit = ref.literal_apply_edge(x_i, x_j, n_i, n_j, lq, lk, lv, heads, groups, dim)
    q, k, v = (ref.literal_group_dense(x, *p, groups, dim) for x, p in ((x_i, lq), (x_j, lk), (x_j, lv)))
    closed, a = ref.closed_form_messages(q, k, v, (n_i * n_j).reshape(-1), heads)
    assert lit.shape == (E, dim)
    assert torch.allclose(lit, closed, rtol=1e-12, atol=1e-12)
    assert (a.sum(-1) <= 1).all() and (a >= 0).all()      # the extra logit 0 keeps every row's sum at most 1


@pytest.mark.parametrize("groups", [1, 2, 8])
@pytest.mark.parametrize("bias", [False, True])
def test_group_dense_equals_the_literal_group_dense(groups, bias):
    from euler_b200 import convolution as conv
    rs = np.random.RandomState(groups + 3 * bias)
    dim = 64
    x = torch.from_numpy(rs.randn(37, dim).astype(np.float32))
    kernel, b = lin(rs, groups, dim, bias)
    kernel, b = kernel.float(), (b.float() if bias else None)
    got = conv.group_dense(x, kernel, b)
    want = ref.literal_group_dense(x.double(), kernel.double(), b.double() if bias else None, groups, dim)
    assert got.shape == (37, dim)
    assert torch.allclose(got.double(), want, rtol=1e-5, atol=1e-5)
    # a leading axis of size one (apply_edge's expand_dims) keeps its shape
    assert conv.group_dense(x[:, None, :], kernel, b).shape == (37, 1, dim)


def test_group_dense_argument_errors():
    from euler_b200 import EulerError
    from euler_b200 import convolution as conv
    x, k = torch.zeros(4, 12), torch.zeros(4, 3, 3)
    for args in ((x[:, :10], k), (x.double(), k), (x, k[0]), (x, k, torch.zeros(5))):
        with pytest.raises(EulerError):
            conv.group_dense(*args)


@pytest.mark.parametrize("heads", [1, 2, 4])
def test_linear_maps_hoisted_per_node_equal_the_per_edge_maps(heads):
    """q, k, v computed once per node and then gathered equal lin_* applied to the gathered rows of every edge"""
    rs = np.random.RandomState(40 + heads)
    dim, groups, n_dst, n_src, E = 32, 8, 20, 30, 200
    xt, xs = rand(rs, n_dst, dim), rand(rs, n_src, dim)
    dst, src = torch.from_numpy(rs.randint(0, n_dst, E)), torch.from_numpy(rs.randint(0, n_src, E))
    lq, lk, lv = (lin(rs, groups, dim) for _ in range(3))
    n0, n1 = ref.gcn_norm(torch.stack([dst, src]), (n_dst, n_src), torch.float64)
    per_edge = ref.literal_apply_edge(xt[dst], xs[src], n0[dst], n1[src], lq, lk, lv, heads, groups, dim)
    q, k, v = (ref.literal_group_dense(x, *p, groups, dim) for x, p in ((xt, lq), (xs, lk), (xs, lv)))
    per_node, _ = ref.closed_form_messages(q[dst], k[src], v[src], (n0[dst] * n1[src]).reshape(-1), heads)
    assert torch.allclose(per_edge, per_node, rtol=1e-12, atol=1e-12)
    out_e, out_n = ref.scatter_mean(per_edge, dst, n_dst), ref.scatter_mean(per_node, dst, n_dst)
    assert torch.allclose(out_e, out_n, rtol=1e-12, atol=1e-12)
