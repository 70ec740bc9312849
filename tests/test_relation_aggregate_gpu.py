"""RelationConv's fused typed mean aggregation (eu_relation_aggregate / eu_relation_aggregate_backward,
euler_b200/csrc/relation.cu) on the GPU.

Forward: on dyadic inputs (every sum exact in any order) bit for bit equal to convolution.relation_aggregate (the literal
restatement of relation_conv.py, one matvec per edge) and to a float64 restatement; on random inputs within rounding of both.
Unsorted (target, relation) keys give the bits of the stably sorted edge list.  Backward: against a float64 restatement and
autograd through relation_aggregate, identical from run to run, exact zeros where nothing flows.  End to end: RelationDataFlow
blocks (which arrive with sorted keys) through a two-layer RGCN against a float64 restatement of relation_conv.py and
BaseGNNNet's loop."""
import ctypes as C

import numpy as np
import pytest
import torch

import graphs

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _graph():
    import euler_b200
    g = graphs.random_graph(seed=5, n=200, T=1, avg_deg=3)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    yield
    torch.cuda.synchronize()


def bits_equal(a, b, what):
    a, b = a.detach().cpu(), b.detach().cpu()
    assert a.shape == b.shape, what
    bad = (a.view(torch.int32) != b.view(torch.int32)).sum().item()
    assert bad == 0, "%s: %d of %d values differ" % (what, bad, a.numel())


def close(got, want, what, rtol=1e-4):
    """within rtol relative, with an absolute floor of rtol times the largest magnitude"""
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else got
    want = want.detach().cpu().double().numpy() if torch.is_tensor(want) else want
    floor = rtol * max(float(np.abs(want).max()) if want.size else 0.0, 1e-30)
    assert np.allclose(got, want, rtol=rtol, atol=floor), "%s: max abs diff %g (largest %g)" % (
        what, float(np.abs(got - want).max()) if want.size else 0.0, floor / rtol)


def edge_list(rs, n_dst, n_src, E, R, hub=0, hub_rel=None, empty_frac=0.3, used_rel=None):
    """(dst, rel, src) int32 on the device, sorted by (dst, rel), stably: empty targets, multi-edges and optionally one hub
    target of `hub` extra edges (all of relation hub_rel when given)"""
    live = rs.choice(n_dst, size=max(1, int(n_dst * (1 - empty_frac))), replace=False)
    rels = np.arange(R) if used_rel is None else np.asarray(used_rel)
    dst = rs.choice(live, size=E) if E else np.zeros(0, np.int64)
    rel = rs.choice(rels, size=E) if E else np.zeros(0, np.int64)
    src = rs.randint(0, n_src, size=E)
    if E >= 4:
        dst[1], rel[1], src[1] = dst[0], rel[0], src[0]          # a multi-edge
    if hub:
        dst = np.concatenate([dst, np.full(hub, live[0])])
        rel = np.concatenate([rel, np.full(hub, hub_rel) if hub_rel is not None else rs.choice(rels, size=hub)])
        src = np.concatenate([src, rs.randint(0, n_src, size=hub)])
    order = np.lexsort((rel, dst))
    return tuple(torch.from_numpy(a[order].astype(np.int32)).cuda() for a in (dst, rel, src))


def dyadic(rs, shape, lo, hi, scale):
    return torch.from_numpy((rs.randint(lo, hi + 1, size=shape) * scale).astype(np.float32)).cuda()


def denominators(dst, n_dst):
    """scatter_mean's divisor as the f32 arithmetic gives it: fl(fl(count) + 1e-7f)"""
    cnt = np.bincount(dst, minlength=n_dst).astype(np.float32)
    return (cnt + np.float32(1e-7)).astype(np.float32)


def reference64(x, W, rel, dst, src, n_dst):
    """relation_conv.py:53-70 in float64 on the CPU, the per-edge matvec summed per target; the f32 mean's divisor and
    division (exact for inputs whose float64 sums are representable in f32)"""
    x, W = x.detach().cpu().double().numpy(), W.detach().cpu().double().numpy()
    rel, dst, src = (t.cpu().numpy().astype(np.int64) for t in (rel, dst, src))
    s = np.zeros((n_dst, W.shape[1]))
    if dst.size:
        np.add.at(s, dst, np.einsum("edf,ef->ed", W[rel], x[src]))
    return torch.from_numpy((s.astype(np.float32) / denominators(dst, n_dst)[:, None]).astype(np.float32))


def reference64_real(x, W, rel, dst, src, n_dst):
    """the same in float64 throughout (for random inputs)"""
    x, W = x.detach().cpu().double().numpy(), W.detach().cpu().double().numpy()
    rel, dst, src = (t.cpu().numpy().astype(np.int64) for t in (rel, dst, src))
    s = np.zeros((n_dst, W.shape[1]))
    if dst.size:
        np.add.at(s, dst, np.einsum("edf,ef->ed", W[rel], x[src]))
    return s / (np.bincount(dst, minlength=n_dst)[:, None] + 1e-7)


def fused(x, W, rel, dst, src, n_dst):
    from euler_b200 import ops
    return ops.relation_mean_aggregate(x, W, rel, torch.stack([dst, src]), (n_dst, x.shape[0]))


def composed(x, W, rel, dst, src, n_dst):
    from euler_b200 import convolution as conv
    return conv.relation_aggregate((None, x), torch.stack([dst, src]), (n_dst, x.shape[0]), rel, W)


FD_CASES = [(1, 1), (3, 5), (16, 32), (32, 32), (64, 128), (128, 128)]


@pytest.mark.parametrize("F,D", FD_CASES)
@pytest.mark.parametrize("R", [1, 18, 300])
def test_forward_is_bit_exact_on_dyadic_inputs(F, D, R):
    """x in {-4..4}/4, W in {-4..4}/8: every product is a multiple of 2^-5 and every sum stays far below 2^24 of them"""
    rs = np.random.RandomState(F * 1000 + D * 10 + R)
    E = 20_000 if F * D <= 1024 else 3000
    for n_dst, n_src, e in ((7, 5, 1), (50, 40, 3), (400, 3000, E)):
        dst, rel, src = edge_list(rs, n_dst, n_src, e, R)
        x = dyadic(rs, (n_src, F), -4, 4, 0.25)
        W = dyadic(rs, (R, D, F), -4, 4, 0.125)
        out = fused(x, W, rel, dst, src, n_dst)
        what = "F=%d D=%d R=%d E=%d" % (F, D, R, e)
        bits_equal(out, composed(x, W, rel, dst, src, n_dst), "vs relation_aggregate " + what)
        bits_equal(out, reference64(x, W, rel, dst, src, n_dst), "vs float64 " + what)
        counts = torch.bincount(dst.long(), minlength=n_dst)
        assert (out[counts == 0] == 0).all() and not torch.signbit(out[counts == 0]).any(), what


@pytest.mark.parametrize("F,D", [(16, 32), (3, 5), (128, 128)])
def test_unaligned_rows_give_the_same_bits(F, D):
    """x_src at a 4-byte offset: no float4 loads, the same bits"""
    rs = np.random.RandomState(3 + F)
    n_dst, n_src, R = 300, 900, 18
    dst, rel, src = edge_list(rs, n_dst, n_src, 5000, R)
    x = torch.from_numpy(rs.randn(n_src, F).astype(np.float32)).cuda()
    W = torch.from_numpy(rs.randn(R, D, F).astype(np.float32)).cuda()
    buf = torch.empty(n_src * F + 1, device="cuda")
    xu = buf[1:].view(n_src, F)
    xu.copy_(x)
    assert xu.data_ptr() % 16 != 0
    bits_equal(fused(xu, W, rel, dst, src, n_dst), fused(x, W, rel, dst, src, n_dst), "unaligned vs aligned")
    xd, Wd = dyadic(rs, (n_src, F), -4, 4, 0.25), dyadic(rs, (R, D, F), -4, 4, 0.125)
    xu.copy_(xd)
    bits_equal(fused(xu, Wd, rel, dst, src, n_dst), reference64(xd, Wd, rel, dst, src, n_dst), "unaligned dyadic vs float64")


@pytest.mark.parametrize("F,D", [(16, 32), (3, 5), (64, 128)])
def test_random_inputs_within_rounding(F, D):
    rs = np.random.RandomState(40 + F)
    n_dst, n_src, R = 500, 4000, 18
    dst, rel, src = edge_list(rs, n_dst, n_src, 30_000, R, hub=20_000)
    x = torch.from_numpy(rs.randn(n_src, F).astype(np.float32)).cuda()
    W = torch.from_numpy(rs.randn(R, D, F).astype(np.float32)).cuda()
    out = fused(x, W, rel, dst, src, n_dst)
    close(out, reference64_real(x, W, rel, dst, src, n_dst), "vs float64", rtol=1e-5)
    close(out, composed(x, W, rel, dst, src, n_dst), "vs relation_aggregate", rtol=1e-4)


def test_edge_cases():
    from euler_b200 import ops
    rs = np.random.RandomState(11)
    F, D, R = 8, 12, 5
    W = dyadic(rs, (R, D, F), -4, 4, 0.125)
    x = dyadic(rs, (30, F), -4, 4, 0.25)
    # E = 0: zero rows
    e0 = torch.zeros((2, 0), dtype=torch.int32, device="cuda")
    out = ops.relation_mean_aggregate(x, W, torch.zeros(0, dtype=torch.int32, device="cuda"), e0, (4, 30))
    assert out.shape == (4, D) and (out == 0).all()
    # E = 1
    dst, rel, src = (torch.tensor([v], dtype=torch.int32, device="cuda") for v in (2, 3, 7))
    out = fused(x, W, rel, dst, src, 4)
    bits_equal(out, reference64(x, W, rel, dst, src, 4), "E = 1")
    assert (out[[0, 1, 3]] == 0).all()
    # a single relation; relations never used (R = 300, only 3 used)
    for R2, used in ((1, None), (300, [0, 150, 299])):
        W2 = dyadic(rs, (R2, D, F), -4, 4, 0.125)
        dst, rel, src = edge_list(rs, 60, 30, 2000, R2, used_rel=used)
        bits_equal(fused(x, W2, rel, dst, src, 60), reference64(x, W2, rel, dst, src, 60), "R = %d" % R2)
    # a 10^5-edge hub target whose edges are one pair (391 chunks) and a hub spread over all relations
    x3 = dyadic(rs, (5000, 4), -1, 1, 0.25)
    W3 = dyadic(rs, (R, 8, 4), -2, 2, 0.125)
    for hub_rel in (2, None):
        dst, rel, src = edge_list(rs, 300, 5000, 3000, R, hub=100_000, hub_rel=hub_rel)
        out = fused(x3, W3, rel, dst, src, 300)
        bits_equal(out, reference64(x3, W3, rel, dst, src, 300), "hub, relation %s" % hub_rel)
        bits_equal(out, composed(x3, W3, rel, dst, src, 300), "hub vs relation_aggregate")


@pytest.mark.parametrize("F,D", [(16, 32), (3, 5)])
def test_unsorted_keys_equal_the_stably_sorted_list(F, D):
    rs = np.random.RandomState(17 + F)
    n_dst, n_src, R = 500, 700, 18
    dst, rel, src = edge_list(rs, n_dst, n_src, 8000, R, hub=3000)
    perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
    ud, ur, us = dst[perm].contiguous(), rel[perm].contiguous(), src[perm].contiguous()
    order = torch.from_numpy(np.lexsort((ur.cpu().numpy(), ud.cpu().numpy()))).cuda()   # stable
    x = torch.from_numpy(rs.randn(n_src, F).astype(np.float32)).cuda()
    W = torch.from_numpy(rs.randn(R, D, F).astype(np.float32)).cuda()
    out = fused(x, W, ur, ud, us, n_dst)
    bits_equal(out, fused(x, W, ur[order], ud[order], us[order], n_dst), "unsorted vs the stably sorted list")
    close(out, reference64_real(x, W, ur, ud, us, n_dst), "unsorted vs float64", rtol=1e-5)
    # sorted targets with relations out of order within a target take the sort as well
    flip = torch.from_numpy(np.lexsort((-rel.cpu().numpy(), dst.cpu().numpy()))).cuda()
    fd, fr, fs = dst[flip].contiguous(), rel[flip].contiguous(), src[flip].contiguous()
    o2 = torch.from_numpy(np.lexsort((fr.cpu().numpy(), fd.cpu().numpy()))).cuda()
    bits_equal(fused(x, W, fr, fd, fs, n_dst), fused(x, W, fr[o2], fd[o2], fs[o2], n_dst), "relations descending")


def test_relations_out_of_range_raise():
    import euler_b200
    rs = np.random.RandomState(2)
    R = 4
    dst, rel, src = edge_list(rs, 10, 10, 50, R)
    x = torch.randn(10, 3, device="cuda")
    W = torch.randn(R, 5, 3, device="cuda")
    for bad in (-1, R):
        r2 = rel.clone()
        r2[17] = bad
        with pytest.raises(euler_b200.EulerError, match="outside"):
            fused(x, W, r2, dst, src, 10)
        r3 = r2[torch.randperm(r2.numel(), device="cuda")]   # unsorted keys: checked in the same pass
        with pytest.raises(euler_b200.EulerError, match="outside"):
            fused(x, W, r3, dst, src, 10)
    fused(x, W, rel, dst, src, 10)                           # the ctx still works


def reference_backward(x, W, rel, dst, src, n_dst, g):
    """float64 restatement of the gradients of out = mean_e W[rel_e] x[src_e] with respect to x and W"""
    x, W, g = (t.detach().cpu().double().numpy() for t in (x, W, g))
    rel, dst, src = (t.cpu().numpy().astype(np.int64) for t in (rel, dst, src))
    gm = g / (np.bincount(dst, minlength=n_dst)[:, None] + 1e-7)
    gx, gW = np.zeros_like(x), np.zeros_like(W)
    np.add.at(gx, src, np.einsum("edf,ed->ef", W[rel], gm[dst]))
    np.add.at(gW, rel, np.einsum("ed,ef->edf", gm[dst], x[src]))
    return gx, gW


def fused_grads(x, W, rel, dst, src, n_dst, g):
    from euler_b200 import ops
    leaves = [t.clone().requires_grad_(True) for t in (x, W)]
    out = ops.relation_mean_aggregate(*leaves, rel, torch.stack([dst, src]), (n_dst, x.shape[0]))
    out.backward(g)
    return [t.grad for t in leaves]


@pytest.mark.parametrize("F,D", [(16, 32), (3, 5), (128, 128)])
@pytest.mark.parametrize("unsorted", [False, True])
def test_backward_against_float64_and_autograd(F, D, unsorted):
    rs = np.random.RandomState(F * 7 + D + (100 if unsorted else 0))
    n_dst, n_src, R = 400, 20_000, 300                       # more sources than edges and relations never used
    E = 6000 if F * D <= 1024 else 2000
    dst, rel, src = edge_list(rs, n_dst, n_src, E, R, hub=5000, used_rel=rs.choice(R, size=40, replace=False))
    if unsorted:
        perm = torch.from_numpy(rs.permutation(dst.numel())).cuda()
        dst, rel, src = dst[perm].contiguous(), rel[perm].contiguous(), src[perm].contiguous()
    x = torch.from_numpy(rs.randn(n_src, F).astype(np.float32)).cuda()
    W = torch.from_numpy(rs.randn(R, D, F).astype(np.float32)).cuda()
    g = torch.from_numpy(rs.randn(n_dst, D).astype(np.float32)).cuda()
    grads = fused_grads(x, W, rel, dst, src, n_dst, g)
    want = reference_backward(x, W, rel, dst, src, n_dst, g)
    leaves = [t.clone().requires_grad_(True) for t in (x, W)]
    composed(*leaves, rel, dst, src, n_dst).backward(g)
    for nm, a, w, c in zip(("grad_x_src", "grad_matrix"), grads, want, leaves):
        close(a, w, nm + " vs float64")
        close(a, c.grad, nm + " vs autograd through relation_aggregate")
    again = fused_grads(x, W, rel, dst, src, n_dst, g)
    for nm, a, b in zip(("grad_x_src", "grad_matrix"), grads, again):
        assert torch.equal(a, b), nm + " differs between two runs"
    src_used = torch.bincount(src.long(), minlength=n_src) > 0
    rel_used = torch.bincount(rel.long(), minlength=R) > 0
    assert (~src_used).any() and (~rel_used).any()
    assert (grads[0][~src_used] == 0).all() and (grads[1][~rel_used] == 0).all()


def test_backward_without_edges_is_zero():
    from euler_b200 import ops
    x = torch.randn(5, 8, device="cuda", requires_grad=True)
    W = torch.randn(3, 4, 8, device="cuda", requires_grad=True)
    out = ops.relation_mean_aggregate(x, W, torch.zeros(0, dtype=torch.int64, device="cuda"),
                                      torch.zeros((2, 0), dtype=torch.int64, device="cuda"), (3, 5))
    assert out.shape == (3, 4) and (out == 0).all()
    out.sum().backward()
    assert (x.grad == 0).all() and (W.grad == 0).all()


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


def hetero_flow(T, roots_n=64, seed=3):
    import euler_b200
    from euler_b200.dataflow import RelationDataFlow
    gr = euler_b200.Graph.rmat_hetero(20_000, 200_000, T, 2, seed=44)
    euler_b200.set_graph(gr, seed=1)
    roots = torch.from_numpy(np.random.RandomState(seed).randint(1, 20_001, size=roots_n).astype(np.int64)).cuda()
    types = list(range(T))
    return RelationDataFlow([5, 5], [types, types])(roots)


def test_relation_dataflow_blocks_arrive_sorted():
    """with rel = e_id and an ascending type list the (dst, rel) keys are non-decreasing: no sort runs"""
    from euler_b200 import ops
    T = 6
    flow = hetero_flow(T)
    rs = np.random.RandomState(0)
    for blk in flow:
        d, r = blk.edge_index[0].cpu().numpy(), blk.e_id.cpu().numpy()
        assert d.size > 100
        key = d.astype(np.int64) * T + r
        assert (np.diff(key) >= 0).all()
        x = dyadic(rs, (blk.size[1], 16), -4, 4, 0.25)
        W = dyadic(rs, (T, 32, 16), -4, 4, 0.125)
        names = kernel_names(lambda: ops._raw_relation(x, W, blk.e_id.to(torch.int32).contiguous(),
                                                       blk.edge_index[0].to(torch.int32).contiguous(),
                                                       blk.edge_index[1].to(torch.int32).contiguous(), blk.size[0]))
        assert "rel_heads" in names and "rel_out" in names and "rel_sort" not in names, names
        ei = blk.edge_index.to(torch.int32)
        bits_equal(fused(x, W, blk.e_id, ei[0], ei[1], blk.size[0]), composed(x, W, blk.e_id, ei[0], ei[1], blk.size[0]),
                   "block")


def restated_rgcn_layer(x_tgt, x_src, ei, size, attr, W, fc):
    """relation_conv.py:53-73 literally, in float64 torch on the CPU: gather x_j, unique + gather of the matrices, matmul,
    scatter_mean (count + 1e-7), plus fc(x_target)"""
    x_j = x_src[ei[1]]
    u, inv = torch.unique(attr, return_inverse=True)
    m = W[u][inv]
    msg = torch.matmul(m, x_j.unsqueeze(-1)).squeeze(-1)
    n = size[0]
    s = torch.zeros((n, W.shape[1]), dtype=msg.dtype).index_add(0, ei[0], msg)
    cnt = torch.zeros(n, dtype=msg.dtype).index_add(0, ei[0], torch.ones(ei.shape[1], dtype=msg.dtype))
    return x_tgt @ fc.T + s / (cnt[:, None] + 1e-7)


def test_two_layer_rgcn_over_relation_dataflow_blocks():
    """RelationDataFlow -> embeddings -> two RelationConv layers (BaseGNNNet's loop: x_target = x[res_n_id], conv, relu) ->
    the final Dense -> loss -> backward, against the float64 restatement; gradients to the embeddings, matrices and fcs"""
    from euler_b200 import convolution as conv
    T, F0, D1, D2, OUT = 5, 16, 32, 24, 8
    flow = hetero_flow(T, roots_n=100, seed=9)
    torch.manual_seed(0)
    emb = (torch.randn(20_001, F0, device="cuda") * 0.5).requires_grad_(True)
    mats = [(torch.randn(T, D1, F0, device="cuda") * 0.2).requires_grad_(True),
            (torch.randn(T, D2, D1, device="cuda") * 0.2).requires_grad_(True)]
    fcs = [torch.nn.Linear(F0, D1, bias=False).cuda(), torch.nn.Linear(D1, D2, bias=False).cuda()]
    head = torch.nn.Linear(D2, OUT).cuda()
    x = emb[flow[0].n_id]
    for blk, W, fc in zip(flow, mats, fcs):
        x_tgt = x[blk.res_n_id]
        x = torch.relu(fc(x_tgt) + conv.relation_aggregate_fused((x_tgt, x), blk.edge_index, blk.size, blk.e_id, W))
    y = head(x)
    wl = torch.randn(*y.shape, device="cuda")
    (y * wl).sum().backward()

    emb_r = emb.detach().cpu().double().requires_grad_(True)
    mats_r = [W.detach().cpu().double().requires_grad_(True) for W in mats]
    fcs_r = [fc.weight.detach().cpu().double().requires_grad_(True) for fc in fcs]
    head_w = head.weight.detach().cpu().double().requires_grad_(True)
    head_b = head.bias.detach().cpu().double().requires_grad_(True)
    xr = emb_r[flow[0].n_id.cpu()]
    for blk, W, fc in zip(flow, mats_r, fcs_r):
        xr = torch.relu(restated_rgcn_layer(xr[blk.res_n_id.cpu()], xr, blk.edge_index.cpu(), blk.size, blk.e_id.cpu().long(),
                                            W, fc))
    yr = xr @ head_w.T + head_b
    (yr * wl.cpu().double()).sum().backward()
    close(y, yr, "output")
    close(emb.grad, emb_r.grad, "grad embeddings")
    for i in range(2):
        close(mats[i].grad, mats_r[i].grad, "grad matrix %d" % i)
        close(fcs[i].weight.grad, fcs_r[i].grad, "grad fc %d" % i)
    close(head.weight.grad, head_w.grad, "grad head")


def test_bad_arguments_raise():
    import euler_b200
    from euler_b200 import _lib, ops
    from euler_b200 import convolution as conv
    x, W = torch.randn(5, 4, device="cuda"), torch.randn(3, 6, 4, device="cuda")
    ei = torch.tensor([[0, 1], [2, 3]], device="cuda")
    rel = torch.tensor([0, 2], device="cuda")
    E = euler_b200.EulerError
    with pytest.raises(E):
        ops.relation_mean_aggregate(x, W[0], rel, ei, (3, 5))                          # 2-D matrix
    with pytest.raises(E):
        ops.relation_mean_aggregate(x, W[None], rel, ei, (3, 5))                       # 4-D matrix
    with pytest.raises(E):
        ops.relation_mean_aggregate(x[:, :3], W, rel, ei, (3, 5))                      # F disagrees
    with pytest.raises(E):
        ops.relation_mean_aggregate(x[:4], W, rel, ei, (3, 5))                         # n_src disagrees
    with pytest.raises(E):
        ops.relation_mean_aggregate(x.double(), W, rel, ei, (3, 5))                    # not f32
    with pytest.raises(E):
        ops.relation_mean_aggregate(x, W.half(), rel, ei, (3, 5))                      # not f32
    with pytest.raises(E):
        ops.relation_mean_aggregate(x, W, rel.float(), ei, (3, 5))                     # float relations
    with pytest.raises(E):
        ops.relation_mean_aggregate(x, W, rel[:1], ei, (3, 5))                         # one relation for two edges
    with pytest.raises(E):
        ops.relation_mean_aggregate(x, W, rel, ei[0], (3, 5))                          # edge_index not [2, E]
    with pytest.raises(E):
        conv.relation_aggregate_fused((None, x), ei, (3, 5), torch.tensor([0, 3], device="cuda"), W)   # rel = R
    lib, ctx = _lib.load(), euler_b200.context()
    d, s, r = ei[0].to(torch.int32), ei[1].to(torch.int32), rel.to(torch.int32)
    out = torch.empty(3, 6, device="cuda")
    a = (x.data_ptr(), W.data_ptr(), r.data_ptr(), d.data_ptr(), s.data_ptr())
    assert lib.eu_relation_aggregate(ctx._h, *a, 2, 3, 5, 0, 6, 4, out.data_ptr()) == 1            # R < 1
    assert lib.eu_relation_aggregate(ctx._h, *a, 2, 3, 5, 3, 0, 4, out.data_ptr()) == 1            # D < 1
    assert lib.eu_relation_aggregate(ctx._h, *a, -1, 3, 5, 3, 6, 4, out.data_ptr()) == 1           # negative E
    assert lib.eu_relation_aggregate(ctx._h, None, *a[1:], 2, 3, 5, 3, 6, 4, out.data_ptr()) == 1  # null x_src
    assert lib.eu_relation_aggregate(ctx._h, *a, 2, 3, 5, 3, 6, 4, None) == 1                      # null out
    assert lib.eu_relation_aggregate(ctx._h, *a, 2, 3, 5, 1 << 20, 1 << 10, 4, out.data_ptr()) == 4  # R*D*F >= 2^31
    gx, gW = torch.empty_like(x), torch.empty_like(W)
    assert lib.eu_relation_aggregate_backward(ctx._h, out.data_ptr(), *a, 2, 3, 5, 3, 6, 4, gx.data_ptr(), None) == 1
    assert lib.eu_relation_aggregate(ctx._h, *a, 2, 3, 5, 3, 6, 4, out.data_ptr()) == 0
    close(out, reference64_real(x, W, r, d, s, 3), "after the refusals", rtol=1e-5)
