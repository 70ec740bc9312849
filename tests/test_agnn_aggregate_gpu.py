"""AGNNConv's fused cosine-attention aggregation (eu_agnn_aggregate / eu_agnn_aggregate_backward, euler_b200/csrc/gat.cu)
on the GPU.

Forward: on dyadic inputs (entries k/8, beta a power of two) every partial sum of the cosine is exact, so the op equals the
composition gather -> mul -> sum -> scatter_softmax -> mul -> scatter_add bit for bit; on random normalized inputs it
equals that composition fed the op's own cos bit for bit, and a float64 restatement to 1e-5.  Unsorted targets give the
bits of the stably sorted list.  Backward: within 1e-4 of a float64 restatement and of autograd through the composition,
identical from run to run.  End to end: two AGNN layers over GCNDataFlow blocks against a float64 restatement of
agnn_conv.py and BaseGNNNet's loop."""
import numpy as np
import pytest
import torch

import graphs
from test_gat_aggregate_gpu import bits_equal, close, edge_list

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _graph():
    import euler_b200
    g = graphs.random_graph(seed=5, n=200, T=1, avg_deg=3)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    yield
    torch.cuda.synchronize()


def composition(x_src, nd, ns, beta, dst, src, n_dst):
    """agnn_conv.py:32-54 composed from the ops: gather -> mul -> beta * -> sum -> scatter_softmax -> mul -> scatter_add"""
    from euler_b200 import ops
    u = (beta * (ops.gather(nd, dst) * ops.gather(ns, src))).sum(-1, keepdim=True)
    alpha = ops.scatter_softmax(u, dst, n_dst)
    return ops.scatter_add(ops.gather(x_src, src) * alpha, dst, n_dst), alpha.view(-1)


def composition_from_cos(x_src, cos, beta, dst, src, n_dst):
    """the same composition from a given per-edge cosine: u = beta * cos"""
    from euler_b200 import ops
    alpha = ops.scatter_softmax((beta * cos).view(-1, 1), dst, n_dst)
    return ops.scatter_add(ops.gather(x_src, src) * alpha, dst, n_dst), alpha.view(-1)


def fused(x_src, nd, ns, beta, dst, src, n_dst, with_alpha=True):
    from euler_b200 import ops
    return ops._raw_agnn(x_src, nd, ns, beta.reshape(1), dst.contiguous(), src.contiguous(), n_dst, with_alpha)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def dyadic(rs, *shape):
    """entries k/8, |k| <= 4: every product and every partial sum of a cosine up to dim 1433 is exact in f32"""
    return cuda(rs.randint(-4, 5, size=shape) / 8.0)


def normalized(rs, n, dim):
    x = rs.randn(n, dim)
    return cuda(x / np.linalg.norm(x, axis=1, keepdims=True))


def unaligned(t):
    """the same values in a contiguous view 4 bytes past a 16-byte boundary"""
    buf = torch.empty(t.numel() + 1, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


DIMS = [1, 3, 4, 32, 64, 128, 602, 1433]


@pytest.mark.parametrize("dim", DIMS)
def test_forward_is_bit_exact_on_dyadic_inputs(dim):
    rs = np.random.RandomState(dim)
    beta = torch.tensor([(0.5, 2.0, -1.0, 0.25)[dim % 4]], device="cuda")
    cases = ((7, 5, 0, 0), (7, 5, 1, 0), (50, 40, 3, 0), (2000, 3000, 20000, 0), (300, 5000, 2000, 100_000))
    for n_dst, n_src, E, hub in cases:
        dst, src = edge_list(rs, n_dst, n_src, E, hub)
        x, nd, ns = dyadic(rs, n_src, dim), dyadic(rs, n_dst, dim), dyadic(rs, n_src, dim)
        what = "dim=%d E=%d hub=%d" % (dim, dst.numel(), hub)
        out, alpha, cos = fused(x, nd, ns, beta, dst, src, n_dst)
        want_out, want_alpha = composition(x, nd, ns, beta, dst, src, n_dst)
        bits_equal(out, want_out, "out " + what)
        bits_equal(alpha, want_alpha, "alpha " + what)
        assert torch.equal(cos, (nd[dst.long()] * ns[src.long()]).sum(-1)), "cos " + what   # a zero's sign may differ
        no_alpha, _, _ = fused(x, nd, ns, beta, dst, src, n_dst, with_alpha=False)   # logits in the op's scratch
        bits_equal(no_alpha, want_out, "out without alpha " + what)
        counts = torch.bincount(dst.long(), minlength=n_dst)
        assert (out[counts == 0] == 0).all(), what       # targets without edges: zero rows
        assert torch.isfinite(out).all()
        if E == 20000:                                   # unaligned rows: the scalar loads, the same bits
            u_out, u_alpha, u_cos = fused(unaligned(x), unaligned(nd), unaligned(ns), beta, dst, src, n_dst)
            bits_equal(u_out, want_out, "out, unaligned rows " + what)
            bits_equal(u_alpha, want_alpha, "alpha, unaligned rows " + what)
            bits_equal(u_cos, cos, "cos, unaligned rows " + what)


def f64_forward(x, nd, ns, beta, dst, src, n_dst):
    """float64 restatement: (out, alpha, cos)"""
    x, nd, ns = (t.detach().cpu().double().numpy() for t in (x, nd, ns))
    dst, src = dst.cpu().numpy().astype(np.int64), src.cpu().numpy().astype(np.int64)
    cos = (nd[dst] * ns[src]).sum(-1)
    u = float(beta) * cos
    m = np.full(n_dst, -1e9)
    np.maximum.at(m, dst, u)
    ex = np.exp(u - m[dst])
    den = np.zeros(n_dst)
    np.add.at(den, dst, ex)
    alpha = ex / den[dst]
    out = np.zeros((n_dst, x.shape[1]))
    np.add.at(out, dst, alpha[:, None] * x[src])
    return out, alpha, cos


@pytest.mark.parametrize("dim", [3, 32, 128, 1433])
def test_random_normalized_inputs(dim):
    rs = np.random.RandomState(100 + dim)
    n_dst, n_src = 1500, 4000
    dst, src = edge_list(rs, n_dst, n_src, 30000, hub=5000)
    x, nd, ns = cuda(rs.randn(n_src, dim)), normalized(rs, n_dst, dim), normalized(rs, n_src, dim)
    beta = torch.tensor([1.7], device="cuda")
    out, alpha, cos = fused(x, nd, ns, beta, dst, src, n_dst)
    w_out, w_alpha, w_cos = f64_forward(x, nd, ns, 1.7, dst, src, n_dst)
    terms = np.abs(nd.double().cpu().numpy()[dst.cpu().numpy()] * ns.double().cpu().numpy()[src.cpu().numpy()]).sum(-1)
    err = np.abs(cos.double().cpu().numpy() - w_cos)
    bound = 2 * dim * 2.0 ** -24 * terms + 2.0 ** -24 * np.abs(w_cos)
    assert (err <= bound).all(), "cos: worst error %g ulps-of-terms" % float((err / (2.0 ** -24 * terms + 1e-300)).max())
    c_out, c_alpha = composition_from_cos(x, cos, beta, dst, src, n_dst)
    bits_equal(out, c_out, "out vs the composition fed the op's cos")
    bits_equal(alpha, c_alpha, "alpha vs the composition fed the op's cos")
    close(cos, w_cos, "cos vs float64", rtol=1e-5)
    close(alpha, w_alpha, "alpha vs float64", rtol=1e-5)
    close(out, w_out, "out vs float64", rtol=1e-5)
    again = fused(x, nd, ns, beta, dst, src, n_dst)
    for nm, a, b in zip(("out", "alpha", "cos"), (out, alpha, cos), again):
        assert torch.equal(a, b), nm + " differs between two runs"


@pytest.mark.parametrize("beta", [0.0, -0.5])
def test_zero_and_negative_beta(beta):
    rs = np.random.RandomState(31)
    n_dst, n_src, dim = 300, 500, 32
    dst, src = edge_list(rs, n_dst, n_src, 5000)
    x, nd, ns = dyadic(rs, n_src, dim), dyadic(rs, n_dst, dim), dyadic(rs, n_src, dim)
    b = torch.tensor([beta], device="cuda")
    out, alpha, _ = fused(x, nd, ns, b, dst, src, n_dst)
    want_out, want_alpha = composition(x, nd, ns, b, dst, src, n_dst)
    bits_equal(out, want_out, "out")
    bits_equal(alpha, want_alpha, "alpha")
    if beta == 0.0:                                      # every logit 0: alpha = 1 / in-degree
        deg = torch.bincount(dst.long(), minlength=n_dst).float()
        assert torch.equal(alpha, 1.0 / deg[dst.long()])


def test_logits_below_minus_1e9_give_nan_alphas_as_the_composition():
    """un-normalized rows: beta * cos below -1e9 for every edge of some targets; scatter_max starts at -1e9, so exp(u - m)
    is 0 for each of their edges and alpha = 0 / 0"""
    rs = np.random.RandomState(9)
    n_dst, n_src, dim = 40, 30, 4
    dst, src = edge_list(rs, n_dst, n_src, 300, empty_frac=0.1)
    x, nd = dyadic(rs, n_src, dim), dyadic(rs, n_dst, dim)
    ns = cuda(rs.randint(1, 5, size=(n_src, dim)) / 8.0 * 2.0 ** 17)
    low = torch.unique(dst)[:5].long()
    nd[low] = -(2.0 ** 17)                               # cos <= -2^34 / 8 * 4 < -1e9
    beta = torch.tensor([1.0], device="cuda")
    out, alpha, _ = fused(x, nd, ns, beta, dst, src, n_dst)
    want_out, want_alpha = composition(x, nd, ns, beta, dst, src, n_dst)
    assert torch.isnan(alpha).any() and torch.isnan(out[low]).all()
    bits_equal(out, want_out, "out")
    bits_equal(alpha, want_alpha, "alpha")


@pytest.mark.parametrize("dim", [3, 32, 128])
def test_unsorted_targets_equal_the_stably_sorted_list(dim):
    rs = np.random.RandomState(17 + dim)
    n_dst, n_src = 500, 700
    dst, src = edge_list(rs, n_dst, n_src, 8000, hub=3000)
    perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
    udst, usrc = dst[perm].contiguous(), src[perm].contiguous()
    order = torch.from_numpy(np.argsort(udst.cpu().numpy(), kind="stable")).cuda()
    x, nd, ns = cuda(rs.randn(n_src, dim)), normalized(rs, n_dst, dim), normalized(rs, n_src, dim)
    beta = torch.tensor([2.3], device="cuda")
    out, alpha, cos = fused(x, nd, ns, beta, udst, usrc, n_dst)
    s_out, s_alpha, s_cos = fused(x, nd, ns, beta, udst[order], usrc[order], n_dst)
    bits_equal(out, s_out, "out vs the stably sorted list")
    bits_equal(alpha[order], s_alpha, "alpha vs the stably sorted list")
    bits_equal(cos[order], s_cos, "cos vs the stably sorted list")


def f64_backward(x, nd, ns, beta, dst, src, n_dst, g):
    """float64 restatement of the gradients with respect to x_src, nrm_dst, nrm_src, beta; and the magnitude of the
    terms of grad_beta (its cancellation floor)"""
    x, nd, ns, g = (t.detach().cpu().double().numpy() for t in (x, nd, ns, g))
    beta = float(beta)
    dst, src = dst.cpu().numpy().astype(np.int64), src.cpu().numpy().astype(np.int64)
    cos = (nd[dst] * ns[src]).sum(-1)
    u = beta * cos
    m = np.full(n_dst, -1e9)
    np.maximum.at(m, dst, u)
    ex = np.exp(u - m[dst])
    den = np.zeros(n_dst)
    np.add.at(den, dst, ex)
    alpha = ex / den[dst]
    da = (g[dst] * x[src]).sum(-1)
    S = np.zeros(n_dst)
    np.add.at(S, dst, alpha * da)
    du = alpha * (da - S[dst])
    g_x, g_nd, g_ns = np.zeros_like(x), np.zeros_like(nd), np.zeros_like(ns)
    np.add.at(g_x, src, alpha[:, None] * g[dst])
    np.add.at(g_nd, dst, (beta * du)[:, None] * ns[src])
    np.add.at(g_ns, src, (beta * du)[:, None] * nd[dst])
    return (g_x, g_nd, g_ns, np.array([(du * cos).sum()])), float(np.abs(du * cos).sum())


def grads_of(fn, leaves, g):
    leaves = [t.clone().requires_grad_(True) for t in leaves]
    out = fn(*leaves)
    out.backward(g)
    return out, [t.grad for t in leaves]


NAMES = ("grad_x_src", "grad_nrm_dst", "grad_nrm_src", "grad_beta")


def check_beta(got, want, terms, what):
    """grad_beta sums du * cos, whose per-target sums nearly cancel: held to 1e-4 of the terms' magnitude"""
    got, want = float(got.reshape(-1)[0]), float(want.reshape(-1)[0])
    assert abs(got - want) <= 1e-4 * max(terms, 1e-30), "%s: %g vs %g (terms %g)" % (what, got, want, terms)


@pytest.mark.parametrize("dim", [3, 32, 128])
@pytest.mark.parametrize("unsorted", [False, True])
def test_backward_against_float64_and_autograd(dim, unsorted):
    from euler_b200 import ops
    rs = np.random.RandomState(dim * 7 + (100 if unsorted else 0))
    n_dst, n_src = 400, 20_000                           # more sources than edges: some have none
    dst, src = edge_list(rs, n_dst, n_src, 6000, hub=5000)
    if unsorted:
        perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
        dst, src = dst[perm].contiguous(), src[perm].contiguous()
    x, nd, ns = cuda(rs.randn(n_src, dim)), normalized(rs, n_dst, dim), normalized(rs, n_src, dim)
    beta = torch.tensor([1.3], device="cuda")
    g = cuda(rs.randn(n_dst, dim))
    ei = torch.stack([dst, src])

    def op(a, b, c, d):
        return ops.agnn_attention_aggregate(a, b, c, d, ei, (n_dst, n_src))

    _, grads = grads_of(op, (x, nd, ns, beta), g)
    want, terms = f64_backward(x, nd, ns, 1.3, dst, src, n_dst, g)
    _, c_grads = grads_of(lambda a, b, c, d: composition(a, b, c, d, dst, src, n_dst)[0], (x, nd, ns, beta), g)
    for nm, a, w, c in zip(NAMES[:3], grads, want, c_grads):
        close(a, w, nm + " vs float64")
        close(a, c, nm + " vs autograd through the composition")
    check_beta(grads[3], want[3], terms, "grad_beta vs float64")
    check_beta(grads[3], c_grads[3].cpu().double().numpy(), terms, "grad_beta vs autograd through the composition")
    assert grads[3].shape == beta.shape
    _, again = grads_of(op, (x, nd, ns, beta), g)
    for nm, a, b in zip(NAMES, grads, again):
        assert torch.equal(a, b), nm + " differs between two runs"
    dst_used = torch.bincount(dst.long(), minlength=n_dst) > 0
    src_used = torch.bincount(src.long(), minlength=n_src) > 0
    assert (~dst_used).any() and (~src_used).any()
    assert (grads[1][~dst_used] == 0).all()
    assert (grads[0][~src_used] == 0).all() and (grads[2][~src_used] == 0).all()


def test_backward_without_edges_is_zero():
    from euler_b200 import ops
    leaves = [torch.randn(5, 8, device="cuda"), torch.randn(3, 8, device="cuda"), torch.randn(5, 8, device="cuda"),
              torch.tensor(1.0, device="cuda")]
    out, grads = grads_of(lambda a, b, c, d: ops.agnn_attention_aggregate(a, b, c, d, torch.zeros((2, 0), dtype=torch.int64,
                                                                                                  device="cuda"), (3, 5)),
                          leaves, torch.ones(3, 8, device="cuda"))
    assert out.shape == (3, 8) and (out == 0).all()
    for t, gr in zip(leaves, grads):
        assert gr.shape == t.shape and (gr == 0).all()


def l2n(x):
    """tf.nn.l2_normalize(x, -1) in float64 torch"""
    return x * torch.rsqrt(torch.clamp_min((x * x).sum(-1, keepdim=True), 1e-12))


def restated_agnn_layer(x_tgt, x_src, ei, size, beta):
    """agnn_conv.py:32-54 literally, in float64 torch on the CPU: gather the normalized rows of every edge, reduce_sum of
    beta * (norm_i * norm_j), scatter_softmax (max from -1e9), x_j * alpha, scatter_add"""
    n = size[0]
    ni, nj = l2n(x_tgt)[ei[0]], l2n(x_src)[ei[1]]
    a = (beta * (ni * nj)).sum(-1)
    m = torch.full((n,), -1e9, dtype=a.dtype).scatter_reduce(0, ei[0], a.detach(), "amax", include_self=True)
    ex = torch.exp(a - m[ei[0]])
    den = torch.zeros(n, dtype=a.dtype).index_add(0, ei[0], ex)
    alpha = ex / den[ei[0]]
    return torch.zeros((n, x_src.shape[1]), dtype=a.dtype).index_add(0, ei[0], x_src[ei[1]] * alpha[:, None])


@pytest.mark.parametrize("self_loops", [False, True])
def test_two_layer_agnn_over_gcn_dataflow_blocks(self_loops):
    """GCNDataFlow -> get_dense_feature -> agnn_aggregate -> relu, twice (BaseGNNNet's loop, one beta per layer) -> loss ->
    backward, against the float64 restatement; with self loops (BaseGNNNet's default) the targets arrive unsorted"""
    import euler_b200
    from euler_b200 import convolution as conv
    from euler_b200.dataflow import GCNDataFlow
    D = 24
    g = graphs.random_graph(seed=8, n=3000, T=1, avg_deg=4, feat_dim=D, hub=500)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    rs = np.random.RandomState(21)
    roots = torch.from_numpy(g["ids"][rs.randint(0, 3000, size=100)].astype(np.int64)).cuda()
    flow = GCNDataFlow([[0], [0]], add_self_loops=self_loops)(roots)
    x0 = euler_b200.get_dense_feature(flow[0].n_id, [0], [D])[0].clone().requires_grad_(True)
    betas = [torch.tensor([1.0], device="cuda", requires_grad=True), torch.tensor([0.6], device="cuda", requires_grad=True)]
    x = x0
    for blk, beta in zip(flow, betas):
        x = torch.relu(conv.agnn_aggregate((x[blk.res_n_id], x), blk.edge_index, blk.size, beta))
    wl = cuda(rs.randn(*x.shape))
    (x * wl).sum().backward()

    xr0 = x0.detach().cpu().double().requires_grad_(True)
    rbetas = [b.detach().cpu().double().requires_grad_(True) for b in betas]
    xr = xr0
    for blk, beta in zip(flow, rbetas):
        xr = torch.relu(restated_agnn_layer(xr[blk.res_n_id.cpu()], xr, blk.edge_index.cpu(), blk.size, beta))
    (xr * wl.cpu().double()).sum().backward()
    close(x, xr, "output")
    close(x0.grad, xr0.grad, "grad x")
    for i, (b, r) in enumerate(zip(betas, rbetas)):
        close(b.grad, r.grad, "grad beta%d" % (i + 1))


def test_x_source_none_means_x_target():
    from euler_b200 import convolution as conv
    rs = np.random.RandomState(4)
    x = cuda(rs.randn(60, 16))
    dst, src = edge_list(rs, 60, 60, 400)
    ei, beta = torch.stack([dst, src]), torch.tensor([1.0], device="cuda")
    assert torch.equal(conv.agnn_aggregate((x, None), ei, (60, 60), beta), conv.agnn_aggregate((x, x), ei, (60, 60), beta))


def test_bad_arguments_raise():
    import euler_b200
    from euler_b200 import _lib, ops
    from euler_b200 import convolution as conv
    x, nd, ns = torch.randn(5, 8, device="cuda"), torch.randn(3, 8, device="cuda"), torch.randn(5, 8, device="cuda")
    beta = torch.tensor([1.0], device="cuda")
    ei = torch.tensor([[0, 1], [2, 3]], device="cuda")
    bad = [
        (x, nd, torch.randn(5, 7, device="cuda"), beta, ei),          # widths disagree
        (x, torch.randn(4, 8, device="cuda"), ns, beta, ei),          # nrm_dst rows != n_dst
        (x, nd, ns, torch.ones(2, device="cuda"), ei),                # beta not a scalar
        (x.double(), nd, ns, beta, ei),                               # not f32
        (x, nd, ns, beta.double(), ei),                               # beta not f32
        (x, nd, ns, 1.0, ei),                                         # beta not a tensor
        (x, nd, ns, beta, ei[0]),                                     # edge_index not [2, E]
        (x[:, 0], nd, ns, beta, ei),                                  # 1-D rows
    ]
    for args in bad:
        with pytest.raises(euler_b200.EulerError):
            ops.agnn_attention_aggregate(*args, (3, 5))
    with pytest.raises(euler_b200.EulerError):
        conv.agnn_aggregate(x, ei, (3, 5), beta)                      # not (x_target, x_source)
    with pytest.raises(euler_b200.EulerError):
        conv.agnn_aggregate((x[:3, :6], x), ei, (3, 5), beta)          # widths disagree
    with pytest.raises(euler_b200.EulerError):
        conv.agnn_aggregate((x[:3], x), ei, (3, 5), torch.ones(1, 2, device="cuda"))   # beta not a scalar
    lib, ctx = _lib.load(), euler_b200.context()
    dst, src = ei[0].to(torch.int32), ei[1].to(torch.int32)
    out = torch.empty(3, 8, device="cuda")
    args = (x.data_ptr(), nd.data_ptr(), ns.data_ptr(), beta.data_ptr(), dst.data_ptr(), src.data_ptr())
    assert lib.eu_agnn_aggregate(ctx._h, *args, 2, 3, 5, 0, out.data_ptr(), None, None) == 1            # dim < 1
    assert lib.eu_agnn_aggregate(ctx._h, *args, -1, 3, 5, 8, out.data_ptr(), None, None) == 1           # negative E
    assert lib.eu_agnn_aggregate(ctx._h, *args, 2, 0, 5, 8, out.data_ptr(), None, None) == 1            # edges, no targets
    assert lib.eu_agnn_aggregate(ctx._h, *args[:3], None, *args[4:], 2, 3, 5, 8, out.data_ptr(), None, None) == 1  # null beta
    assert lib.eu_agnn_aggregate(ctx._h, *args, 2, 3, 5, 8, None, None, None) == 1                      # null out
    al, cs = torch.empty(2, device="cuda"), torch.empty(2, device="cuda")
    gx, gnd, gns, gb = (torch.empty_like(t) for t in (x, nd, ns, beta))
    bwd = [out.data_ptr(), *args[:4], al.data_ptr(), cs.data_ptr(), dst.data_ptr(), src.data_ptr(), 2, 3, 5, 8,
           gx.data_ptr(), gnd.data_ptr(), gns.data_ptr(), gb.data_ptr()]
    for i in (5, 6, 16):                                                                                 # null alpha, cos, grad_beta
        assert lib.eu_agnn_aggregate_backward(ctx._h, *bwd[:i], None, *bwd[i + 1:]) == 1
    assert lib.eu_agnn_aggregate(ctx._h, *args, 2, 3, 5, 8, out.data_ptr(), al.data_ptr(), cs.data_ptr()) == 0
    assert lib.eu_agnn_aggregate_backward(ctx._h, *bwd) == 0
