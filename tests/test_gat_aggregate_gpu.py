"""GATConv's fused attention aggregation (eu_gat_aggregate / eu_gat_aggregate_backward, euler_b200/csrc/gat.cu) on the GPU.

Forward: bit-exact against the composition of the existing mp ops for non-decreasing targets, bit-identical to the stably
sorted edge list for unsorted ones.  Backward: within 1e-4 of a float64 CPU restatement and of autograd through the
composition, identical from run to run.  End to end: GCNDataFlow blocks through two GAT layers against a float64 restatement
of gat_conv.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import graphs

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _graph():
    import euler_b200
    g = graphs.random_graph(seed=5, n=200, T=1, avg_deg=3)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    yield
    torch.cuda.synchronize()


def composition(h_src, s_dst, s_src, dst, src, n_dst):
    """the same aggregation composed from the existing ops (gat_conv.py:53-78 over mp_ops.py)"""
    from euler_b200 import ops
    E, H = dst.numel(), s_dst.shape[1]
    C = h_src.shape[1] // H
    u = F.leaky_relu(ops.gather(s_dst, dst) + ops.gather(s_src, src), 0.2)
    alpha = ops.scatter_softmax(u, dst, n_dst)
    out = ops.scatter_add((ops.gather(h_src, src).view(E, H, C) * alpha.view(E, H, 1)).view(E, H * C), dst, n_dst)
    return out, alpha


def fused(h_src, s_dst, s_src, dst, src, n_dst):
    from euler_b200 import ops
    return ops._raw_gat(h_src.contiguous(), s_dst.contiguous(), s_src.contiguous(), dst.contiguous(), src.contiguous(), n_dst, True)


def bits_equal(a, b, what):
    """bit for bit, NaNs (at the same places) compared as equal"""
    a, b = a.detach().cpu(), b.detach().cpu()
    assert a.shape == b.shape, what
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), what + ": NaN positions differ"
    bad = (a[~na].view(torch.int32) != b[~nb].view(torch.int32)).sum().item()
    assert bad == 0, "%s: %d of %d values differ" % (what, bad, a.numel())


def edge_list(rs, n_dst, n_src, E, hub=0, empty_frac=0.3):
    """sorted targets with empty rows, single-edge rows, multi-edges and optionally one hub target of `hub` edges"""
    live = rs.choice(n_dst, size=max(1, int(n_dst * (1 - empty_frac))), replace=False)
    dst = rs.choice(live, size=E) if E else np.zeros(0, np.int64)
    src = rs.randint(0, n_src, size=E)
    if E >= 4:
        dst[1], src[1] = dst[0], src[0]                      # a multi-edge
    if hub:
        dst = np.concatenate([dst, np.full(hub, live[0])])
        src = np.concatenate([src, rs.randint(0, n_src, size=hub)])
    order = np.argsort(dst, kind="stable")
    dst, src = dst[order], src[order]
    return torch.from_numpy(dst.astype(np.int32)).cuda(), torch.from_numpy(src.astype(np.int32)).cuda()


def inputs(rs, n_dst, n_src, H, C, scale=2.0):
    h = torch.from_numpy(rs.randn(n_src, H * C).astype(np.float32)).cuda()
    sd = torch.from_numpy((rs.randn(n_dst, H) * scale).astype(np.float32)).cuda()
    ss = torch.from_numpy((rs.randn(n_src, H) * scale).astype(np.float32)).cuda()
    return h, sd, ss


HC_CASES = [(1, 32), (8, 8), (4, 3), (2, 64), (3, 5)]     # float4 (H*C % 4 == 0) and scalar widths


@pytest.mark.parametrize("H,C", HC_CASES)
def test_forward_is_bit_exact_against_the_composition(H, C):
    rs = np.random.RandomState(H * 100 + C)
    for n_dst, n_src, E, hub in ((7, 5, 0, 0), (7, 5, 1, 0), (50, 40, 3, 0), (2000, 3000, 20000, 0), (300, 5000, 2000, 100_000)):
        dst, src = edge_list(rs, n_dst, n_src, E, hub)
        h, sd, ss = inputs(rs, n_dst, n_src, H, C)
        out, alpha = fused(h, sd, ss, dst, src, n_dst)
        want_out, want_alpha = composition(h, sd, ss, dst, src, n_dst)
        what = "H=%d C=%d E=%d hub=%d" % (H, C, dst.numel(), hub)
        bits_equal(out, want_out, "out " + what)
        bits_equal(alpha, want_alpha, "alpha " + what)
        from euler_b200 import ops
        no_alpha, _ = ops._raw_gat(h, sd, ss, dst, src, n_dst, False)   # alpha in the op's scratch: every no_grad call
        bits_equal(no_alpha, want_out, "out without alpha " + what)
        counts = torch.bincount(dst.long(), minlength=n_dst)
        assert (out[counts == 0] == 0).all(), what       # targets without edges: zero rows
        assert torch.isfinite(out).all()


def test_forward_unaligned_rows_take_the_scalar_path():
    """h_src and out at a 4-byte offset: the float4 loads are not allowed, the results are the same bits"""
    rs = np.random.RandomState(3)
    n_dst, n_src, H, C = 100, 80, 2, 8
    dst, src = edge_list(rs, n_dst, n_src, 900)
    h, sd, ss = inputs(rs, n_dst, n_src, H, C)
    buf = torch.empty(n_src * H * C + 1, device="cuda")
    hu = buf[1:].view(n_src, H * C)
    hu.copy_(h)
    from euler_b200 import ops
    out, alpha = ops._raw_gat(hu, sd, ss, dst, src, n_dst, True)
    want_out, want_alpha = composition(h, sd, ss, dst, src, n_dst)
    bits_equal(out, want_out, "out")
    bits_equal(alpha, want_alpha, "alpha")


def test_logits_below_minus_1e9_give_nan_alphas_as_the_composition():
    rs = np.random.RandomState(9)
    n_dst, n_src, H, C = 40, 30, 2, 4
    dst, src = edge_list(rs, n_dst, n_src, 300, empty_frac=0.1)
    h, sd, ss = inputs(rs, n_dst, n_src, H, C)
    low = torch.unique(dst)[:5].long()
    sd[low, 0] = -1e10                                   # leaky_relu(-1e10 + s) < -1e9: every logit of head 0 of these targets
    out, alpha = fused(h, sd, ss, dst, src, n_dst)
    want_out, want_alpha = composition(h, sd, ss, dst, src, n_dst)
    assert torch.isnan(alpha[:, 0]).any() and torch.isnan(out[low, :C]).all()
    bits_equal(out, want_out, "out")
    bits_equal(alpha, want_alpha, "alpha")


@pytest.mark.parametrize("H,C", [(1, 32), (4, 3)])
def test_unsorted_targets_equal_the_stably_sorted_list(H, C):
    rs = np.random.RandomState(17 + H)
    n_dst, n_src = 500, 700
    dst, src = edge_list(rs, n_dst, n_src, 8000, hub=3000)
    perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
    udst, usrc = dst[perm].contiguous(), src[perm].contiguous()
    order = torch.from_numpy(np.argsort(udst.cpu().numpy(), kind="stable")).cuda()
    h, sd, ss = inputs(rs, n_dst, n_src, H, C)
    out, alpha = fused(h, sd, ss, udst, usrc, n_dst)
    s_out, s_alpha = fused(h, sd, ss, udst[order], usrc[order], n_dst)
    bits_equal(out, s_out, "out vs the stably sorted list")
    bits_equal(alpha[order], s_alpha, "alpha vs the stably sorted list")
    c_out, c_alpha = composition(h, sd, ss, udst, usrc, n_dst)   # its scatters take the atomic path: reordered sums
    assert torch.allclose(out, c_out, rtol=1e-5, atol=1e-6)
    assert torch.allclose(alpha, c_alpha, rtol=1e-5, atol=1e-7)


def reference_backward(h, sd, ss, dst, src, n_dst, g):
    """float64 CPU restatement of the gradients of out = sum_e alpha * h_src[src_e] with respect to h_src, s_dst, s_src"""
    h, sd, ss, g = (x.detach().cpu().double().numpy() for x in (h, sd, ss, g))
    dst, src = dst.cpu().numpy().astype(np.int64), src.cpu().numpy().astype(np.int64)
    n_src, H = ss.shape
    C = h.shape[1] // H
    z = sd[dst] + ss[src]
    u = np.where(z > 0, z, 0.2 * z)
    m = np.full((n_dst, H), -1e9)
    np.maximum.at(m, dst, u)
    ex = np.exp(u - m[dst])
    den = np.zeros((n_dst, H))
    np.add.at(den, dst, ex)
    alpha = ex / den[dst]
    hv, gv = h.reshape(n_src, H, C), g.reshape(n_dst, H, C)
    da = (gv[dst] * hv[src]).sum(-1)
    S = np.zeros((n_dst, H))
    np.add.at(S, dst, alpha * da)
    du = alpha * (da - S[dst]) * np.where(z > 0, 1.0, 0.2)
    g_sd, g_ss, g_h = np.zeros((n_dst, H)), np.zeros((n_src, H)), np.zeros((n_src, H, C))
    np.add.at(g_sd, dst, du)
    np.add.at(g_ss, src, du)
    np.add.at(g_h, src, alpha[:, :, None] * gv[dst])
    return g_h.reshape(n_src, H * C), g_sd, g_ss


def close(got, want, what, rtol=1e-4):
    """within rtol relative, with an absolute floor of rtol times the largest magnitude (cancellation in d_alpha - S)"""
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else got
    want = want.detach().cpu().double().numpy() if torch.is_tensor(want) else want
    floor = rtol * max(float(np.abs(want).max()) if want.size else 0.0, 1e-30)
    assert np.allclose(got, want, rtol=rtol, atol=floor), "%s: max abs diff %g (largest %g)" % (
        what, float(np.abs(got - want).max()) if want.size else 0.0, floor / rtol)


def fused_grads(h, sd, ss, dst, src, n_dst, g):
    from euler_b200 import ops
    leaves = [x.clone().requires_grad_(True) for x in (h, sd, ss)]
    out = ops.gat_attention_aggregate(*leaves, torch.stack([dst, src]), (n_dst, h.shape[0]))
    out.backward(g)
    return out, [x.grad for x in leaves]


@pytest.mark.parametrize("H,C", HC_CASES)
@pytest.mark.parametrize("unsorted", [False, True])
def test_backward_against_float64_and_autograd(H, C, unsorted):
    rs = np.random.RandomState(H * 7 + C + (100 if unsorted else 0))
    n_dst, n_src = 400, 20_000                           # more sources than edges: some have none
    dst, src = edge_list(rs, n_dst, n_src, 6000, hub=5000)
    if unsorted:
        perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
        dst, src = dst[perm].contiguous(), src[perm].contiguous()
    h, sd, ss = inputs(rs, n_dst, n_src, H, C, scale=1.0)
    g = torch.from_numpy(rs.randn(n_dst, H * C).astype(np.float32)).cuda()
    out, grads = fused_grads(h, sd, ss, dst, src, n_dst, g)
    want = reference_backward(h, sd, ss, dst, src, n_dst, g)
    leaves = [x.clone().requires_grad_(True) for x in (h, sd, ss)]
    c_out, _ = composition(*leaves, dst, src, n_dst)
    c_out.backward(g)
    for nm, a, w, c in zip(("grad_h_src", "grad_s_dst", "grad_s_src"), grads, want, leaves):
        close(a, w, nm + " vs float64")
        close(a, c.grad, nm + " vs autograd through the composition")
    _, again = fused_grads(h, sd, ss, dst, src, n_dst, g)
    for nm, a, b in zip(("grad_h_src", "grad_s_dst", "grad_s_src"), grads, again):
        assert torch.equal(a, b), nm + " differs between two runs"
    dst_used = torch.bincount(dst.long(), minlength=n_dst) > 0
    src_used = torch.bincount(src.long(), minlength=n_src) > 0
    assert (~dst_used).any() and (~src_used).any()
    assert (grads[1][~dst_used] == 0).all()
    assert (grads[0][~src_used] == 0).all() and (grads[2][~src_used] == 0).all()


def test_backward_without_edges_is_zero():
    from euler_b200 import ops
    h = torch.randn(5, 8, device="cuda", requires_grad=True)
    sd = torch.randn(3, 2, device="cuda", requires_grad=True)
    ss = torch.randn(5, 2, device="cuda", requires_grad=True)
    out = ops.gat_attention_aggregate(h, sd, ss, torch.zeros((2, 0), dtype=torch.int64, device="cuda"), (3, 5))
    assert out.shape == (3, 8) and (out == 0).all()
    out.sum().backward()
    for x in (h, sd, ss):
        assert x.grad.shape == x.shape and (x.grad == 0).all()


def restated_gat_layer(x_tgt, x_src, ei, size, w, att_i, att_j):
    """gat_conv.py:53-78 literally, in float64 torch on the CPU: fc on both sides, Attention (Dense(1)) on the gathered
    rows of every edge, per head; heads concatenated (gat.py's calculate_conv)"""
    H, C = att_i.shape
    hi, hj = x_tgt @ w.T, x_src @ w.T
    n = size[0]
    outs = []
    for k in range(H):
        sl = slice(k * C, (k + 1) * C)
        xi, xj = hi[ei[0], sl], hj[ei[1], sl]
        a = F.leaky_relu(xi @ att_i[k] + xj @ att_j[k], 0.2)
        m = torch.full((n,), -1e9, dtype=a.dtype).scatter_reduce(0, ei[0], a.detach(), "amax", include_self=True)
        ex = torch.exp(a - m[ei[0]])
        den = torch.zeros(n, dtype=a.dtype).index_add(0, ei[0], ex)
        alpha = ex / den[ei[0]]
        outs.append(torch.zeros((n, C), dtype=a.dtype).index_add(0, ei[0], xj * alpha[:, None]))
    return torch.cat(outs, 1)


@pytest.mark.parametrize("self_loops", [False, True])
def test_two_layer_gat_over_gcn_dataflow_blocks(self_loops):
    """GCNDataFlow -> get_dense_feature -> Linear -> gat_aggregate, twice -> loss -> backward, against the float64
    restatement; with self loops the targets arrive unsorted"""
    import euler_b200
    from euler_b200 import convolution as conv
    from euler_b200.dataflow import GCNDataFlow
    D, H, C1, C2 = 16, 2, 8, 4
    g = graphs.random_graph(seed=8, n=3000, T=1, avg_deg=4, feat_dim=D, hub=500)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    rs = np.random.RandomState(21)
    roots = torch.from_numpy(g["ids"][rs.randint(0, 3000, size=100)].astype(np.int64)).cuda()
    flow = GCNDataFlow([[0], [0]], add_self_loops=self_loops)(roots)
    torch.manual_seed(0)
    params = [torch.nn.Linear(D, H * C1, bias=False).cuda(), torch.randn(H, C1, device="cuda") * 0.3,
              torch.randn(H, C1, device="cuda") * 0.3,
              torch.nn.Linear(H * C1, H * C2, bias=False).cuda(), torch.randn(H, C2, device="cuda") * 0.3,
              torch.randn(H, C2, device="cuda") * 0.3]
    for p in params[1:3] + params[4:6]:
        p.requires_grad_(True)
    layers = [params[:3], params[3:]]
    x0 = euler_b200.get_dense_feature(flow[0].n_id, [0], [D])[0]
    x = x0
    for i, (blk, (lin, ai, aj)) in enumerate(zip(flow, layers)):
        hx = lin(x)
        x = conv.gat_aggregate((hx[blk.res_n_id], hx), blk.edge_index, blk.size, ai, aj)
        if i == 0:
            x = torch.relu(x)
    wl = torch.from_numpy(rs.randn(*x.shape).astype(np.float32)).cuda()
    (x * wl).sum().backward()

    ref = [torch.nn.Parameter(p.weight.detach().cpu().double()) if isinstance(p, torch.nn.Linear) else
           p.detach().cpu().double().requires_grad_(True) for p in params]
    xr = x0.cpu().double()
    for i, blk in enumerate(flow):
        w, ai, aj = ref[3 * i: 3 * i + 3]
        xr = restated_gat_layer(xr[blk.res_n_id.cpu()], xr, blk.edge_index.cpu(), blk.size, w, ai, aj)
        if i == 0:
            xr = torch.relu(xr)
    (xr * wl.cpu().double()).sum().backward()
    close(x, xr, "output")
    for p, r, nm in zip(params, ref, ("W1", "att1_i", "att1_j", "W2", "att2_i", "att2_j")):
        got = p.weight.grad if isinstance(p, torch.nn.Linear) else p.grad
        close(got, r.grad, "grad " + nm)


def test_fused_forward_matches_the_composition_on_a_dataflow_block():
    """the deeper block of a GCNDataFlow without self loops has sorted targets: bit-exact"""
    import euler_b200
    from euler_b200.dataflow import GCNDataFlow
    g = graphs.random_graph(seed=4, n=5000, T=1, avg_deg=6, hub=2000)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    rs = np.random.RandomState(2)
    roots = torch.from_numpy(g["ids"][rs.randint(0, 5000, size=300)].astype(np.int64)).cuda()
    for blk in GCNDataFlow([[0], [0]], add_self_loops=False)(roots):
        ei = blk.edge_index.to(torch.int32)
        h, sd, ss = inputs(rs, blk.size[0], blk.size[1], 4, 8)
        out, alpha = fused(h, sd, ss, ei[0], ei[1], blk.size[0])
        want_out, want_alpha = composition(h, sd, ss, ei[0], ei[1], blk.size[0])
        bits_equal(out, want_out, "out")
        bits_equal(alpha, want_alpha, "alpha")


def test_bad_arguments_raise():
    import euler_b200
    from euler_b200 import _lib, ops
    from euler_b200 import convolution as conv
    h, sd, ss = torch.randn(5, 8, device="cuda"), torch.randn(3, 2, device="cuda"), torch.randn(5, 2, device="cuda")
    ei = torch.tensor([[0, 1], [2, 3]], device="cuda")
    with pytest.raises(euler_b200.EulerError):
        ops.gat_attention_aggregate(h, sd, torch.randn(5, 3, device="cuda"), ei, (3, 5))   # heads disagree
    with pytest.raises(euler_b200.EulerError):
        ops.gat_attention_aggregate(torch.randn(5, 7, device="cuda"), sd, ss, ei, (3, 5))  # H*C not a multiple of H
    with pytest.raises(euler_b200.EulerError):
        ops.gat_attention_aggregate(h, sd, ss, ei[0], (3, 5))                               # edge_index not [2, E]
    with pytest.raises(euler_b200.EulerError):
        ops.gat_attention_aggregate(h, sd[:, 0], ss, ei, (3, 5))                           # 1-D scores
    att = torch.randn(2, 4, device="cuda")
    with pytest.raises(euler_b200.EulerError):
        conv.gat_aggregate((h[:3, :6], h), ei, (3, 5), att, att)                            # width is not H*C
    with pytest.raises(euler_b200.EulerError):
        conv.gat_aggregate((h[:3], h), ei, (3, 5), att, torch.randn(2, 3, device="cuda"))   # att_j is not [H, C]
    wide = torch.randn(5, 16, device="cuda")
    out_slice = conv.gat_aggregate((wide[:3, :8], wide[:, :8]), ei, (3, 5), att, att)       # column slices: not contiguous
    out_copy = conv.gat_aggregate((wide[:3, :8].contiguous(), wide[:, :8].contiguous()), ei, (3, 5), att, att)
    assert torch.equal(out_slice, out_copy)
    with pytest.raises(euler_b200.EulerError):
        conv.gat_aggregate((h[:3], h), ei, (3, 5), torch.randn(2, 4, device="cuda"), torch.randn(2, 4, device="cuda"), aggr="mean")
    lib, ctx = _lib.load(), euler_b200.context()
    dst, src = ei[0].to(torch.int32), ei[1].to(torch.int32)
    out = torch.empty(3, 8, device="cuda")
    args = (h.data_ptr(), sd.data_ptr(), ss.data_ptr(), dst.data_ptr(), src.data_ptr())
    assert lib.eu_gat_aggregate(ctx._h, *args, 2, 3, 5, 0, 4, out.data_ptr(), None) == 1          # heads < 1
    assert lib.eu_gat_aggregate(ctx._h, *args, 2, 3, 5, 2, 0, out.data_ptr(), None) == 1          # head_dim < 1
    assert lib.eu_gat_aggregate(ctx._h, *args, -1, 3, 5, 2, 4, out.data_ptr(), None) == 1         # negative E
    assert lib.eu_gat_aggregate(ctx._h, None, *args[1:], 2, 3, 5, 2, 4, out.data_ptr(), None) == 1  # null h_src
    assert lib.eu_gat_aggregate(ctx._h, *args, 2, 3, 5, 2, 4, None, None) == 1                    # null out
    gh, gsd, gss = torch.empty(5, 8, device="cuda"), torch.empty(3, 2, device="cuda"), torch.empty(5, 2, device="cuda")
    assert lib.eu_gat_aggregate_backward(ctx._h, out.data_ptr(), h.data_ptr(), None, sd.data_ptr(), ss.data_ptr(), dst.data_ptr(),
                                         src.data_ptr(), 2, 3, 5, 2, 4, gh.data_ptr(), gsd.data_ptr(), gss.data_ptr()) == 1  # null alpha
    assert lib.eu_gat_aggregate(ctx._h, *args, 2, 3, 5, 2, 4, out.data_ptr(), None) == 0
