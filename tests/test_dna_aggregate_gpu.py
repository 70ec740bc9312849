"""DNAConv's fused attention aggregation (eu_dna_aggregate / eu_dna_aggregate_backward, euler_b200/csrc/dna.cu) on the GPU.

Forward: on dyadic inputs with k = 0 (every score 0, a = 1/(H+1)) bit for bit equal to the literal composition of
dna_conv.py over the mp ops and to float64; for H = 1 and sorted targets of at most 256 edges, given the op's alpha, equal to
gather -> multiply -> norm product -> scatter_mean; on random inputs within rounding of float64 and of the f32 composition.
Unsorted targets give the bits of the stably sorted edge list.  Backward: against float64 and autograd through the
composition, identical from run to run, exact zeros for unused rows.  End to end: two DNA layers over GCNDataFlow blocks with
self loops against a float64 restatement of dna_conv.py and BaseGNNNet's loop."""
import ctypes as C

import numpy as np
import pytest
import torch

import dna_reference as ref
import graphs

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _graph():
    import euler_b200
    g = graphs.random_graph(seed=5, n=200, T=1, avg_deg=3)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    yield
    torch.cuda.synchronize()


def cuda(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float32)).cuda()


def bits_equal(a, b, what):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    assert a.shape == b.shape, "%s: shapes %s vs %s" % (what, tuple(a.shape), tuple(b.shape))
    bad = (a.view(torch.int32) != b.view(torch.int32)).sum().item()
    assert bad == 0, "%s: %d of %d values differ" % (what, bad, a.numel())


def close(got, want, what, rtol=1e-4):
    """within rtol relative, with an absolute floor of rtol times the largest magnitude"""
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else got
    want = want.detach().cpu().double().numpy() if torch.is_tensor(want) else want
    floor = rtol * max(float(np.abs(want).max()) if want.size else 0.0, 1e-30)
    assert np.allclose(got, want, rtol=rtol, atol=floor), "%s: max abs diff %g (largest %g)" % (
        what, float(np.abs(got - want).max()) if want.size else 0.0, floor / rtol)


def edge_list(rs, n_dst, n_src, E, hub=0, hub_src=0, empty_frac=0.3):
    """(dst, src) int32 on the device, sorted by dst (stably): empty targets, multi-edges, optionally a hub target of `hub`
    extra edges and a hub source of `hub_src` extra edges"""
    live = rs.choice(n_dst, size=max(1, int(n_dst * (1 - empty_frac))), replace=False)
    dst = rs.choice(live, size=E) if E else np.zeros(0, np.int64)
    src = rs.randint(0, n_src, size=E)
    if E >= 4:
        dst[1], src[1] = dst[0], src[0]                         # a multi-edge
    if hub:
        dst = np.concatenate([dst, np.full(hub, live[0])])
        src = np.concatenate([src, rs.randint(0, n_src, size=hub)])
    if hub_src:
        dst = np.concatenate([dst, rs.choice(live, size=hub_src)])
        src = np.concatenate([src, np.full(hub_src, 1 % n_src)])
    order = np.argsort(dst, kind="stable")
    return tuple(torch.from_numpy(a[order].astype(np.int32)).cuda() for a in (dst, src))


def dyadic(rs, shape, lo, hi, scale):
    return cuda(rs.randint(lo, hi + 1, size=shape) * scale)


def norms(rs, n):
    return cuda(rs.choice([0.5, 1.0, 2.0], size=n))


def fused(q, k, v, n0, n1, dst, src, H, alpha=False):
    from euler_b200 import ops
    if alpha:
        return ops._raw_dna(q, k, v, n0, n1, dst, src, q.shape[0], H, True)
    return ops.dna_attention_aggregate(q, k, v, n0, n1, torch.stack([dst, src]), (q.shape[0], k.shape[0]), H)


def composition(q, k, v, n0, n1, dst, src, H):
    """dna_conv.py's apply_edge and scatter_mean literally, in f32 over the mp ops, from the per-node q, k, v: gather the
    rows and norms of every edge, the reshapes and transposes of multi_head / attention, restricted_softmax,
    norm_i * norm_j * out, scatter_mean"""
    from euler_b200 import ops
    n_dst, dim = q.shape[0], q.shape[1]
    C_ = dim // H
    qe, ke, ve = ops.gather(q, dst), ops.gather(k, src), ops.gather(v, src)
    ni, nj = ops.gather(n0.reshape(-1, 1), dst), ops.gather(n1.reshape(-1, 1), src)
    qh, kh, vh = (t.reshape(-1, 1, H, C_).permute(1, 0, 2, 3) for t in (qe, ke, ve))
    out = ref.literal_attention(qh, kh, vh).permute(1, 0, 2, 3).reshape(-1, qh.shape[1], dim).squeeze(0)
    return ops.scatter_mean(ni * nj * out, dst, n_dst)


def reference64(q, k, v, n0, n1, dst, src, H, exact_sums=True):
    """the closed form in float64 on the CPU.  exact_sums: the sums are f32-exact, so the f32 mean's divisor and division
    are applied to the float64 sum rounded to f32 (as the op and the composition do)"""
    q, k, v, n0, n1 = (t.detach().cpu().double() for t in (q, k, v, n0, n1))
    d, s = dst.cpu().long(), src.cpu().long()
    msg, _ = ref.closed_form_messages(q[d], k[s], v[s], n0.reshape(-1)[d] * n1.reshape(-1)[s], H)
    n = q.shape[0]
    tot = torch.zeros((n, q.shape[1]), dtype=torch.float64).index_add(0, d, msg)
    if not exact_sums:
        return tot / (torch.bincount(d, minlength=n).double()[:, None] + 1e-7)
    cnt = torch.bincount(d, minlength=n).float() + np.float32(1e-7)
    return tot.float() / cnt[:, None]


HC_CASES = [(1, 1), (1, 4), (1, 32), (3, 3), (3, 32), (7, 4), (7, 1)]


@pytest.mark.parametrize("H,C_", HC_CASES)
def test_forward_is_bit_exact_on_dyadic_inputs(H, C_):
    """k = 0: every score is 0, a = 1/(H+1) (dyadic for H = 1, 3, 7); v in {-4..4}/4, norms in {1/2, 1, 2}: every
    message and sum is exact, so any summation order gives the same bits"""
    rs = np.random.RandomState(H * 100 + C_)
    dim = H * C_
    for n_dst, n_src, E, hub in ((7, 5, 1, 0), (50, 40, 300, 0), (300, 2000, 5000, 1500)):
        dst, src = edge_list(rs, n_dst, n_src, E, hub=hub)
        q = cuda(rs.randn(n_dst, dim))
        k = torch.zeros(n_src, dim, device="cuda")
        v = dyadic(rs, (n_src, dim), -4, 4, 0.25)
        n0, n1 = norms(rs, n_dst), norms(rs, n_src)
        out, alpha = fused(q, k, v, n0, n1, dst, src, H, alpha=True)
        what = "H=%d C=%d E=%d" % (H, C_, dst.numel())
        assert (alpha == 1.0 / (H + 1)).all(), what
        bits_equal(out, composition(q, k, v, n0, n1, dst, src, H), "vs composition " + what)
        bits_equal(out, reference64(q, k, v, n0, n1, dst, src, H), "vs float64 " + what)
        bits_equal(fused(q, k, v, n0, n1, dst, src, H), out, "autograd entry " + what)
        counts = torch.bincount(dst.long(), minlength=n_dst)
        assert (out[counts == 0] == 0).all() and not torch.signbit(out[counts == 0]).any(), what


@pytest.mark.parametrize("H,C_", [(1, 32), (3, 4), (3, 3), (7, 1)])
def test_unaligned_rows_give_the_same_bits(H, C_):
    """q, k and v at a 4-byte offset: no float4 loads, the same bits"""
    rs = np.random.RandomState(3 + H + C_)
    n_dst, n_src, dim = 300, 900, H * C_
    dst, src = edge_list(rs, n_dst, n_src, 5000, hub=700)
    t = [cuda(rs.randn(n, dim) * 0.5) for n in (n_dst, n_src, n_src)]
    n0, n1 = cuda(rs.rand(n_dst) + 0.1), cuda(rs.rand(n_src) + 0.1)
    un = []
    for x in t:
        buf = torch.empty(x.numel() + 1, device="cuda")
        xu = buf[1:].view(x.shape)
        xu.copy_(x)
        assert xu.data_ptr() % 16 != 0
        un.append(xu)
    a = fused(*t, n0, n1, dst, src, H, alpha=True)
    b = fused(*un, n0, n1, dst, src, H, alpha=True)
    bits_equal(b[0], a[0], "out unaligned vs aligned")
    bits_equal(b[1], a[1], "alpha unaligned vs aligned")


def test_h1_equals_gather_multiply_norm_scatter_mean_given_alpha():
    """H = 1, sorted targets of at most 256 edges each: given the op's alpha, out is the composition's bits"""
    from euler_b200 import ops
    rs = np.random.RandomState(12)
    n_dst, n_src = 400, 3000
    for dim in (32, 3, 128):
        dst, src = edge_list(rs, n_dst, n_src, 20_000)
        assert torch.bincount(dst.long()).max() <= 256
        q, k, v = cuda(rs.randn(n_dst, dim)), cuda(rs.randn(n_src, dim)), cuda(rs.randn(n_src, dim))
        n0, n1 = cuda(rs.rand(n_dst) + 0.1), cuda(rs.rand(n_src) + 0.1)
        out, alpha = fused(q, k, v, n0, n1, dst, src, 1, alpha=True)
        msg = (ops.gather(n0.view(-1, 1), dst) * ops.gather(n1.view(-1, 1), src)) * (ops.gather(v, src) * alpha.view(-1, 1))
        bits_equal(out, ops.scatter_mean(msg, dst, n_dst), "dim = %d" % dim)


@pytest.mark.parametrize("H,C_", [(1, 32), (1, 128), (4, 32), (2, 3), (8, 4)])
def test_random_inputs_within_rounding(H, C_):
    rs = np.random.RandomState(40 + H * C_)
    n_dst, n_src, dim = 500, 4000, H * C_
    dst, src = edge_list(rs, n_dst, n_src, 30_000, hub=2000, hub_src=2000)
    q, k, v = (cuda(rs.randn(n, dim)) for n in (n_dst, n_src, n_src))
    n0, n1 = cuda(rs.rand(n_dst) + 0.1), cuda(rs.rand(n_src) + 0.1)
    out = fused(q, k, v, n0, n1, dst, src, H)
    close(out, reference64(q, k, v, n0, n1, dst, src, H, exact_sums=False), "vs float64", rtol=1e-5)
    close(out, composition(q, k, v, n0, n1, dst, src, H), "vs composition", rtol=1e-4)


def test_edge_cases():
    from euler_b200 import ops
    rs = np.random.RandomState(11)
    H, C_ = 2, 4
    dim = H * C_
    q, k, v = cuda(rs.randn(4, dim)), cuda(rs.randn(30, dim)), cuda(rs.randn(30, dim))
    n0, n1 = cuda(rs.rand(4) + 0.5), cuda(rs.rand(30) + 0.5)
    # E = 0: zero rows
    e0 = torch.zeros((2, 0), dtype=torch.int32, device="cuda")
    out = ops.dna_attention_aggregate(q, k, v, n0, n1, e0, (4, 30), H)
    assert out.shape == (4, dim) and (out == 0).all()
    # E = 1
    dst, src = (torch.tensor([x], dtype=torch.int32, device="cuda") for x in (2, 7))
    out = fused(q, k, v, n0, n1, dst, src, H)
    close(out, reference64(q, k, v, n0, n1, dst, src, H, exact_sums=False), "E = 1", rtol=1e-5)
    assert (out[[0, 1, 3]] == 0).all()
    # a 10^5-edge hub target and a 10^5-edge hub source (391 chunks each), dyadic so the bits are exact: H = 3 and k = 0
    # make a = 1/4, v in {-1, 0, 1}/4 and norms in {1, 2} keep every sum far below 2^24 of its last bit
    n_dst, n_src, H3 = 300, 5000, 3
    dst, src = edge_list(rs, n_dst, n_src, 3000, hub=100_000, hub_src=100_000)
    qd, kd = cuda(rs.randn(n_dst, H3 * C_)), torch.zeros(n_src, H3 * C_, device="cuda")
    vd = dyadic(rs, (n_src, H3 * C_), -1, 1, 0.25)
    n0d, n1d = cuda(rs.choice([1.0, 2.0], size=n_dst)), cuda(rs.choice([1.0, 2.0], size=n_src))
    out = fused(qd, kd, vd, n0d, n1d, dst, src, H3)
    bits_equal(out, reference64(qd, kd, vd, n0d, n1d, dst, src, H3), "hubs vs float64")
    bits_equal(out, composition(qd, kd, vd, n0d, n1d, dst, src, H3), "hubs vs composition")
    # large positive logits (every s >= 120: exp(-m) underflows) and large negative ones (every s <= -200: every exp(s)
    # underflows, a = 0).  A score of magnitude s carries a rounding error of about s * 2^-24, which the softmax turns into a
    # relative error of that size: hence 1e-3 here
    dst, src = edge_list(rs, 50, 40, 600)
    for scale in (60.0, -100.0):
        qb = cuda(np.abs(rs.randn(50, dim)) + 1.0)
        kb = cuda(np.abs(rs.randn(40, dim)) + 1.0) * scale
        vb = cuda(rs.randn(40, dim))
        n0b, n1b = cuda(rs.rand(50) + 0.5), cuda(rs.rand(40) + 0.5)
        out, alpha = fused(qb, kb, vb, n0b, n1b, dst, src, H, alpha=True)
        assert torch.isfinite(out).all() and torch.isfinite(alpha).all()
        if scale < 0:
            assert (alpha == 0).all() and (out == 0).all()
        close(out, reference64(qb, kb, vb, n0b, n1b, dst, src, H, exact_sums=False), "logits x %g" % scale, rtol=1e-3)


@pytest.mark.parametrize("H,C_", [(1, 32), (4, 8), (3, 3)])
def test_unsorted_targets_equal_the_stably_sorted_list(H, C_):
    rs = np.random.RandomState(17 + H)
    n_dst, n_src, dim = 500, 700, H * C_
    dst, src = edge_list(rs, n_dst, n_src, 8000, hub=3000)
    perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
    ud, us = dst[perm].contiguous(), src[perm].contiguous()
    order = torch.sort(ud, stable=True)[1]
    q, k, v = (cuda(rs.randn(n, dim)) for n in (n_dst, n_src, n_src))
    n0, n1 = cuda(rs.rand(n_dst) + 0.1), cuda(rs.rand(n_src) + 0.1)
    out, alpha = fused(q, k, v, n0, n1, ud, us, H, alpha=True)
    o2, a2 = fused(q, k, v, n0, n1, ud[order].contiguous(), us[order].contiguous(), H, alpha=True)
    bits_equal(out, o2, "unsorted vs the stably sorted list")
    bits_equal(alpha[order], a2, "alpha unsorted vs sorted")
    close(out, reference64(q, k, v, n0, n1, ud, us, H, exact_sums=False), "unsorted vs float64", rtol=1e-5)


def kernel_names(fn):
    """the kernels (eu_ctx_profile names) that fn() runs on this thread's Context"""
    from euler_b200 import _lib, ops
    torch.cuda.synchronize()
    ctx = ops._ctx_on_stream()
    lib = _lib.load()
    lib.eu_ctx_profile(ctx._h, 1)
    try:
        fn()
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 16)
        lib.eu_ctx_profile_read(ctx._h, buf, len(buf))
    finally:
        lib.eu_ctx_profile(ctx._h, 0)
    return {line.split(",")[0] for line in buf.value.decode().splitlines() if line}


def test_sorted_targets_take_no_sort():
    rs = np.random.RandomState(5)
    dst, src = edge_list(rs, 100, 100, 2000)
    q, k, v = (cuda(rs.randn(100, 16)) for _ in range(3))
    n0, n1 = cuda(rs.rand(100) + 0.1), cuda(rs.rand(100) + 0.1)
    names = kernel_names(lambda: fused(q, k, v, n0, n1, dst, src, 2, alpha=True))
    assert "dna_scores" in names and "dna_sums" in names and "dna_sort" not in names, names
    perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
    names = kernel_names(lambda: fused(q, k, v, n0, n1, dst[perm].contiguous(), src[perm].contiguous(), 2, alpha=True))
    assert "dna_sort" in names, names


def backward64(q, k, v, n0, n1, dst, src, H, g):
    """autograd of the float64 closed form on the CPU"""
    leaves = [t.detach().cpu().double().requires_grad_(True) for t in (q, k, v)]
    d, s = dst.cpu().long(), src.cpu().long()
    w = (n0.cpu().double().reshape(-1)[d] * n1.cpu().double().reshape(-1)[s])
    msg, _ = ref.closed_form_messages(leaves[0][d], leaves[1][s], leaves[2][s], w, H)
    ref.scatter_mean(msg, d, q.shape[0]).backward(g.cpu().double())
    return [t.grad for t in leaves]


def fused_grads(q, k, v, n0, n1, dst, src, H, g):
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    fused(*leaves, n0, n1, dst, src, H).backward(g)
    return [t.grad for t in leaves]


@pytest.mark.parametrize("H,C_", [(1, 32), (4, 8), (2, 3), (8, 4)])
@pytest.mark.parametrize("unsorted", [False, True])
def test_backward_against_float64_and_autograd(H, C_, unsorted):
    rs = np.random.RandomState(H * 7 + C_ + (100 if unsorted else 0))
    n_dst, n_src, dim = 400, 20_000, H * C_                   # more sources than edges: unused rows
    dst, src = edge_list(rs, n_dst, n_src, 6000, hub=3000, hub_src=1000)
    if unsorted:
        perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
        dst, src = dst[perm].contiguous(), src[perm].contiguous()
    q, k, v = (cuda(rs.randn(n, dim)) for n in (n_dst, n_src, n_src))
    n0, n1 = cuda(rs.rand(n_dst) + 0.1), cuda(rs.rand(n_src) + 0.1)
    g = cuda(rs.randn(n_dst, dim))
    grads = fused_grads(q, k, v, n0, n1, dst, src, H, g)
    want = backward64(q, k, v, n0, n1, dst, src, H, g)
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    composition(*leaves, n0, n1, dst, src, H).backward(g)
    for nm, a, w, c in zip(("grad_q", "grad_k", "grad_v"), grads, want, leaves):
        close(a, w, nm + " vs float64")
        close(a, c.grad, nm + " vs autograd through the composition")
    again = fused_grads(q, k, v, n0, n1, dst, src, H, g)
    for nm, a, b in zip(("grad_q", "grad_k", "grad_v"), grads, again):
        assert torch.equal(a, b), nm + " differs between two runs"
    dst_used = torch.bincount(dst.long(), minlength=n_dst) > 0
    src_used = torch.bincount(src.long(), minlength=n_src) > 0
    assert (~dst_used).any() and (~src_used).any()
    assert (grads[0][~dst_used] == 0).all() and (grads[1][~src_used] == 0).all() and (grads[2][~src_used] == 0).all()


def test_backward_without_edges_is_zero():
    from euler_b200 import ops
    q, k, v = (torch.randn(n, 8, device="cuda", requires_grad=True) for n in (3, 5, 5))
    out = ops.dna_attention_aggregate(q, k, v, torch.ones(3, device="cuda"), torch.ones(5, device="cuda"),
                                      torch.zeros((2, 0), dtype=torch.int64, device="cuda"), (3, 5), 2)
    assert out.shape == (3, 8) and (out == 0).all()
    out.sum().backward()
    assert (q.grad == 0).all() and (k.grad == 0).all() and (v.grad == 0).all()


@pytest.mark.parametrize("H", [1, 4])
def test_two_layer_dna_over_gcn_dataflow_blocks(H):
    """GCNDataFlow with self loops (the dna example's setting: the targets arrive unsorted) -> get_dense_feature -> two DNA
    layers (BaseGNNNet's loop: x_target = x[res_n_id], conv, relu; groups = 8) -> loss -> backward, against the float64
    restatement of dna_conv.py; gradients to the features, in_fc, lin_q, lin_k and lin_v"""
    import euler_b200
    from euler_b200 import convolution as conv
    from euler_b200.dataflow import GCNDataFlow
    D0, dim, groups = 24, 32, 8
    g = graphs.random_graph(seed=8, n=3000, T=1, avg_deg=4, feat_dim=D0, hub=500)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    rs = np.random.RandomState(21 + H)
    roots = torch.from_numpy(g["ids"][rs.randint(0, 3000, size=100)].astype(np.int64)).cuda()
    flow = GCNDataFlow([[0], [0]], add_self_loops=True)(roots)
    assert any((blk.edge_index[0][1:] < blk.edge_index[0][:-1]).any().item() for blk in flow)
    x0 = euler_b200.get_dense_feature(flow[0].n_id, [0], [D0])[0].clone().requires_grad_(True)
    params = []
    for d_in in (D0, dim):
        fc = cuda(rs.randn(dim, d_in) * 0.3).requires_grad_(True)
        lins = [(cuda(rs.randn(groups, dim // groups, dim // groups) * 0.5).requires_grad_(True),
                 cuda(rs.randn(dim) * 0.1).requires_grad_(True)) for _ in range(3)]
        params.append((fc, lins))
    x = x0
    for blk, (fc, lins) in zip(flow, params):
        xt = x[blk.res_n_id]
        x = torch.relu(conv.dna_aggregate((xt @ fc.T, x @ fc.T), blk.edge_index, blk.size, *lins, H))
    wl = cuda(rs.randn(*x.shape))
    (x * wl).sum().backward()

    xr0 = x0.detach().cpu().double().requires_grad_(True)
    rparams = [(fc.detach().cpu().double().requires_grad_(True),
                [tuple(t.detach().cpu().double().requires_grad_(True) for t in p) for p in lins]) for fc, lins in params]
    xr = xr0
    for blk, (fc, lins) in zip(flow, rparams):
        xr = torch.relu(ref.literal_dna_layer(xr[blk.res_n_id.cpu()], xr, blk.edge_index.cpu().long(), blk.size, fc, *lins,
                                              H, groups))
    (xr * wl.cpu().double()).sum().backward()
    close(x, xr, "output")
    close(x0.grad, xr0.grad, "grad x")
    for i, ((fc, lins), (rfc, rlins)) in enumerate(zip(params, rparams)):
        close(fc.grad, rfc.grad, "grad in_fc %d" % i)
        for nm, p, r in zip(("lin_q", "lin_k", "lin_v"), lins, rlins):
            close(p[0].grad, r[0].grad, "grad %s kernel %d" % (nm, i))
            close(p[1].grad, r[1].grad, "grad %s bias %d" % (nm, i))


def test_bad_arguments_raise():
    import euler_b200
    from euler_b200 import _lib, ops
    from euler_b200 import convolution as conv
    q, k, v = torch.randn(3, 8, device="cuda"), torch.randn(5, 8, device="cuda"), torch.randn(5, 8, device="cuda")
    n0, n1 = torch.ones(3, device="cuda"), torch.ones(5, device="cuda")
    ei = torch.tensor([[0, 1], [2, 3]], device="cuda")
    E = euler_b200.EulerError
    bad = [
        ((q, k, v[:, :7], n0, n1, ei), 2),                            # widths disagree
        ((q[:2], k, v, n0, n1, ei), 2),                               # q rows != n_dst
        ((q, k, v, n0[:2], n1, ei), 2),                               # n0 rows != n_dst
        ((q, k, v, n0, n1.view(5, 1, 1), ei), 2),                     # n1 not [n] or [n, 1]
        ((q.double(), k, v, n0, n1, ei), 2),                          # not f32
        ((q, k, v, n0.double(), n1, ei), 2),                          # norms not f32
        ((q, k, v, n0, n1, ei[0]), 2),                                # edge_index not [2, E]
        ((q[:, 0], k, v, n0, n1, ei), 2),                             # 1-D rows
        ((q, k, v, n0, n1, ei), 3),                                   # dim % heads
        ((q, k, v, n0, n1, ei), 0),                                   # heads < 1
    ]
    for args, H in bad:
        with pytest.raises(E):
            ops.dna_attention_aggregate(*args, (3, 5), H)
    q16 = torch.randn(3, 16, device="cuda")
    k16 = torch.randn(5, 16, device="cuda")
    with pytest.raises(E, match="heads"):
        ops.dna_attention_aggregate(q16, k16, k16, n0, n1, ei, (3, 5), 16)   # more heads than the op holds
    x = torch.randn(5, 8, device="cuda")
    lin = (torch.randn(2, 4, 4, device="cuda"), torch.randn(8, device="cuda"))
    with pytest.raises(E):
        conv.dna_aggregate(x, ei, (3, 5), lin, lin, lin, 2)                  # not (x_target, x_source)
    with pytest.raises(E):
        conv.dna_aggregate((x[:3], x), ei, (3, 5), lin, lin, lin[0], 2)      # lin_v not a pair
    with pytest.raises(E):
        conv.dna_aggregate((x[:3], x), ei, (3, 5), lin, lin, lin, 3)         # dim % heads
    with pytest.raises(E):
        conv.group_dense(x, torch.randn(3, 2, 2, device="cuda"))             # dim % groups
    lib, ctx = _lib.load(), euler_b200.context()
    dst, src = ei[0].to(torch.int32), ei[1].to(torch.int32)
    out = torch.empty(3, 8, device="cuda")
    a = (q.data_ptr(), k.data_ptr(), v.data_ptr(), n0.data_ptr(), n1.data_ptr(), dst.data_ptr(), src.data_ptr())
    assert lib.eu_dna_aggregate(ctx._h, *a, 2, 3, 5, 0, 8, out.data_ptr(), None) == 1            # heads < 1
    assert lib.eu_dna_aggregate(ctx._h, *a, 2, 3, 5, 2, 0, out.data_ptr(), None) == 1            # head_dim < 1
    assert lib.eu_dna_aggregate(ctx._h, *a, -1, 3, 5, 2, 4, out.data_ptr(), None) == 1           # negative E
    assert lib.eu_dna_aggregate(ctx._h, *a, 2, 0, 5, 2, 4, out.data_ptr(), None) == 1            # edges, no targets
    assert lib.eu_dna_aggregate(ctx._h, None, *a[1:], 2, 3, 5, 2, 4, out.data_ptr(), None) == 1  # null q
    assert lib.eu_dna_aggregate(ctx._h, *a, 2, 3, 5, 2, 4, None, None) == 1                      # null out
    assert lib.eu_dna_aggregate(ctx._h, *a, 2, 3, 5, 16, 1, out.data_ptr(), None) == 4           # heads > 8
    assert lib.eu_dna_aggregate(ctx._h, *a, 1 << 31, 3, 5, 2, 4, out.data_ptr(), None) == 4      # 2^31 edges
    al = torch.empty(2, 2, 2, device="cuda")
    gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    bwd = [out.data_ptr(), *a[:5], al.data_ptr(), *a[5:], 2, 3, 5, 2, 4, gq.data_ptr(), gk.data_ptr(), gv.data_ptr()]
    for i in (0, 6, 14, 16):                                                                     # null grad_out, alpha, grad_q, grad_v
        assert lib.eu_dna_aggregate_backward(ctx._h, *bwd[:i], None, *bwd[i + 1:]) == 1
    assert lib.eu_dna_aggregate(ctx._h, *a, 2, 3, 5, 2, 4, out.data_ptr(), al.data_ptr()) == 0
    close(out, reference64(q, k, v, n0, n1, dst, src, 2, exact_sums=False), "after the refusals", rtol=1e-5)
