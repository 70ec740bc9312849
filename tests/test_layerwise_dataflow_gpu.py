"""The sparse batch adjacency (eu_sparse_get_adj_coo, euler_b200/csrc/layerwise.cu), sample_neighbor_layerwise_coo and the
layer-wise dataflows on the GPU: the adjacency bit-exact against the numpy restatement of sparse_get_adj_op.cc and equal to
the dense op's nonzero entries plus the filler; the draws those of sample_neighbor_layerwise; the device dataflows equal to
the same flows driven by the CPU stand-in of tests/test_layerwise_dataflow_cpu.py replaying the device's draws."""
import numpy as np
import pytest
import torch

import cases
import graphs
from test_layerwise_dataflow_cpu import ABSENT, CpuLayerwiseSampler, eq_flow, hub_of, np_sparse_get_adj

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def dense_coo(adj):
    """the SparseTensor of a dense [batch, N, M] 0/1 view: its nonzero entries plus the filler of every batch row whose
    (N-1, M-1) is 0"""
    keep = adj != 0
    keep[:, -1, -1] = True
    return np.argwhere(keep).astype(np.int64), (adj[keep] != 0).astype(np.int64)


def _inputs(g, og, rs, batch, N, M):
    """nodes with the hub, absent and repeated nodes; neighbors drawn mostly from the nodes' own listings (many hits),
    repeated, absent, and the extreme id -1"""
    nodes = g["ids"][rs.randint(0, len(g["ids"]), size=(batch, N))].astype(np.int64)
    nodes.reshape(-1)[::11] = ABSENT
    nodes.reshape(-1)[3::17] = nodes.reshape(-1)[0]
    nodes[:, 0] = hub_of(g)
    lens, ids, _, _ = og.get_full_neighbor(nodes.reshape(-1).astype(np.uint64), [0])
    pool = np.concatenate([ids.astype(np.int64), g["ids"].astype(np.int64), [ABSENT, -1]])
    nb = pool[rs.randint(0, len(pool), size=(batch, M))]
    nb.reshape(-1)[5::9] = nb.reshape(-1)[0]
    nb[:, -1] = nb[:, 0]
    return nodes, nb


@pytest.mark.parametrize("T,stride", [(1, 1), (3, 7)])
def test_coo_adjacency_equals_the_restatement_and_the_dense_op(T, stride):
    """random multigraphs with a 4000-edge hub, batch 1..64, N and M up to a few thousand, edge-type lists with repeats,
    out-of-range types and none"""
    import euler_b200
    g = graphs.random_graph(seed=50 + T, n=20_000, T=T, avg_deg=5, id_stride=stride, id_base=3, hub=4000)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    og = graphs.oracle_graph(g)
    rs = np.random.RandomState(T)
    most = 0
    for batch, N, M in [(1, 1, 1), (1, 3000, 2500), (7, 200, 300), (64, 40, 50), (3, 1, 4000), (2, 2000, 1), (64, 1, 1)]:
        nodes, nb = _inputs(g, og, rs, batch, N, M)
        for et in ([0], [T - 1, 0, T - 1], [], [9, 0]):
            idx, val, shape = euler_b200.sparse_get_adj_coo(torch.from_numpy(nodes).cuda(), torch.from_numpy(nb).cuda(), et, N, M)
            w_idx, w_val, w_shape = np_sparse_get_adj(og, nodes, nb, et)
            most = max(most, int(w_val.sum()))
            what = "batch=%d N=%d M=%d et=%s" % (batch, N, M, et)
            cases.eq(idx.cpu().numpy(), w_idx, "indices " + what)
            cases.eq(val.cpu().numpy(), w_val, "values " + what)
            assert shape == w_shape
            d_idx, d_val = dense_coo(euler_b200.sparse_get_adj(nodes.reshape(-1), nb.reshape(-1), et, N, M).cpu().numpy())
            cases.eq(idx.cpu().numpy(), d_idx, "dense indices " + what)
            cases.eq(val.cpu().numpy(), d_val, "dense values " + what)
    assert most > 1000                  # the neighbors are drawn from the listings: the large cases hit often


def test_coo_adjacency_ids_zero_and_minus_one_and_empty_inputs():
    import euler_b200
    from test_full_dataflow_cpu import extreme_id_graph
    g = extreme_id_graph()
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    og = graphs.oracle_graph(g)
    e = int(np.flatnonzero(g["nbr"] == np.uint64(2 ** 64 - 1))[0])
    lists_minus_one = g["ids"][(np.searchsorted(g["grp_ptr"], e, side="right") - 1) // g["T"]].astype(np.int64)
    nodes = np.asarray([[0, -1, -1, 0, 5, ABSENT, lists_minus_one, 7]], np.int64)
    lens, ids, _, _ = og.get_full_neighbor(nodes.reshape(-1).astype(np.uint64), [0, 1])
    nb = np.concatenate([ids.astype(np.int64)[:20], [-1, 0, -1, ABSENT]]).reshape(1, -1)
    for et in ([0, 1], [1, 1]):
        idx, val, _ = euler_b200.sparse_get_adj_coo(nodes, nb, et, nodes.shape[1], nb.shape[1])
        w_idx, w_val, _ = np_sparse_get_adj(og, nodes, nb, et)
        cases.eq(idx.cpu().numpy(), w_idx, "extreme ids")
        cases.eq(val.cpu().numpy(), w_val, "extreme ids")
        if et == [0, 1]:
            assert (nb[0, w_idx[w_val == 1, 2]] == -1).any()        # 2^64-1 is a listed neighbor here
    for n, m, nd, nbs in [(3, 4, 0, 0), (0, 4, 0, 8), (3, 0, 6, 0)]:
        idx, val, shape = euler_b200.sparse_get_adj_coo(np.ones(nd, np.int64), np.ones(nbs, np.int64), [0], n, m)
        assert idx.shape == (0, 3) and val.numel() == 0 and shape[1:] == (n, m)
    out, (idx, val, shape) = euler_b200.sample_neighbor_layerwise_coo(np.ones((2, 0), np.int64), [0], 3, default_node=-5)
    assert out.cpu().tolist() == [[-5] * 3] * 2 and idx.shape == (0, 3) and shape == (2, 0, 3)


@pytest.mark.parametrize("rng", ["minstd", "philox"])
@pytest.mark.parametrize("weight_func", ["", "sqrt"])
def test_coo_sampling_draws_what_the_dense_sampler_draws(rng, weight_func):
    """under one seed sample_neighbor_layerwise_coo draws exactly what sample_neighbor_layerwise draws, and the call after it
    draws identically too (the same engine state is consumed); its adjacency is the dense one's entries plus the filler"""
    import euler_b200
    g = graphs.random_graph(seed=77, n=5000, T=2, avg_deg=5, hub=4000, zero_w_frac=0.1, empty_frac=0.2)
    euler_b200.set_graph(graphs.cuda_graph(g), rng=rng, seed=9)
    og = graphs.oracle_graph(g)
    rs = np.random.RandomState(1)
    nodes = g["ids"][rs.randint(0, 5000, size=(16, 30))].astype(np.int64)
    nodes[3] = ABSENT                                         # a batch row without candidates
    nodes[0, 0] = hub_of(g)
    d_nodes = torch.from_numpy(nodes).cuda()
    seq = []
    for fn in (euler_b200.sample_neighbor_layerwise, euler_b200.sample_neighbor_layerwise_coo):
        euler_b200.seed(21)
        first = fn(d_nodes, [0, 1], 700, -3, weight_func)
        second = fn(d_nodes[2:], [1], 300, -3, weight_func)
        seq.append((first, second))
    (f_dense, s_dense), (f_coo, s_coo) = seq
    for dense, coo in ((f_dense, f_coo), (s_dense, s_coo)):
        cases.eq(coo[0].cpu().numpy(), dense[0].cpu().numpy(), "draws")
        d_idx, d_val = dense_coo(dense[1].cpu().numpy())
        cases.eq(coo[1][0].cpu().numpy(), d_idx, "adjacency vs dense")
        cases.eq(coo[1][1].cpu().numpy(), d_val, "values vs dense")
    w_idx, w_val, _ = np_sparse_get_adj(og, nodes, f_coo[0].cpu().numpy(), [0, 1])
    cases.eq(f_coo[1][0].cpu().numpy(), w_idx, "adjacency vs restatement")
    cases.eq(f_coo[1][1].cpu().numpy(), w_val, "values vs restatement")
    assert (f_coo[0][3] == -3).all() and len(np.unique(f_coo[0][0].cpu().numpy())) < 700     # default fill; repeated draws


class Recorder:
    """euler_b200 with every draw recorded (host copies), for the stand-in to replay"""

    def __init__(self):
        import euler_b200
        self.mod, self.draws = euler_b200, []

    def sample_neighbor(self, *a, **kw):
        r = self.mod.sample_neighbor(*a, **kw)
        self.draws.append(r[0].cpu().numpy())
        return r

    def sample_neighbor_layerwise_coo(self, *a, **kw):
        r = self.mod.sample_neighbor_layerwise_coo(*a, **kw)
        self.draws.append(r[0].cpu().numpy())
        return r

    def __getattr__(self, name):
        return getattr(self.mod, name)


def test_device_dataflows_equal_the_stand_in_replaying_the_draws():
    import euler_b200
    from euler_b200.dataflow import LayerwiseDataFlow, LayerwiseEachDataFlow
    g = graphs.random_graph(seed=12, n=20_000, T=2, avg_deg=6, hub=4000)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=4)
    rs = np.random.RandomState(2)
    roots = g["ids"][rs.randint(0, 20_000, size=512)].astype(np.int64)
    roots[::13] = ABSENT
    roots[1] = hub_of(g)
    flows = [(LayerwiseDataFlow, ([400, 400], [[0], [0]]), {}), (LayerwiseDataFlow, ([50, 60, 0], [[0, 1], [1], [0, 1]]), {}),
             (LayerwiseEachDataFlow, ([10, 20], [[0], [1]]), {"max_id": 10 ** 9}),
             (LayerwiseEachDataFlow, ([5, 1, 7], [[0, 1], [0], [1]]), {})]
    for cls, args, kw in flows:
        for self_loops in (True, False):
            for r in (roots, roots[:1], np.full(3, ABSENT, np.int64)):
                rec = Recorder()
                flow = cls(*args, add_self_loops=self_loops, sampler=rec, **kw)(torch.from_numpy(r).cuda())
                cpu = CpuLayerwiseSampler(g, replay=rec.draws)
                want = cls(*args, add_self_loops=self_loops, sampler=cpu, **kw)(torch.from_numpy(r))
                assert not cpu.replay
                eq_flow(flow, [(b.n_id.numpy(), b.res_n_id.numpy(), b.edge_index.numpy(), b.size) for b in want])
                assert all(b.edge_index.is_cuda and b.n_id.is_cuda for b in flow)


def test_adapt_block_feeds_gcn_aggregate():
    """one LayerwiseDataFlow ('adapt') block -> get_dense_feature -> gcn_aggregate against numpy over the same block"""
    import euler_b200
    from euler_b200 import convolution as conv
    from euler_b200.dataflow import LayerwiseDataFlow
    D = 32
    g = graphs.random_graph(seed=8, n=3000, T=2, avg_deg=4, feat_dim=D, hub=500)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    roots = torch.from_numpy(g["ids"][np.random.RandomState(6).randint(0, 3000, size=200)].astype(np.int64)).cuda()
    flow = LayerwiseDataFlow([100, 100], [[0, 1], [1]])(roots)
    for blk in flow:
        x = euler_b200.get_dense_feature(blk.n_id, [0], [D])[0]
        got = conv.gcn_aggregate((None, x), blk.edge_index, blk.size).cpu().numpy()
        e0, e1 = blk.edge_index.cpu().numpy()
        x1 = x.cpu().numpy().astype(np.float64)
        deg0 = np.bincount(e0, minlength=blk.size[0]).astype(np.float64)
        deg1 = np.bincount(e1, minlength=blk.size[1]).astype(np.float64)
        want = np.zeros((blk.size[0], D))
        np.add.at(want, e0, ((deg0[e0] ** -0.5) * (deg1[e1] ** -0.5))[:, None] * x1[e1])
        assert np.allclose(got, want, rtol=1e-5, atol=1e-5)
        assert e0.size > blk.size[0]


def test_coo_argument_checks():
    """a cap that is not the entry count and negative sizes are refused"""
    import euler_b200
    from euler_b200 import _lib
    g = graphs.random_graph(seed=2, n=100, T=1)
    euler_b200.set_graph(graphs.cuda_graph(g))
    lib, ctx = _lib.load(), euler_b200.context()
    nodes = torch.arange(1, 11, dtype=torch.int64, device="cuda")
    ptr = torch.empty(11, dtype=torch.int64, device="cuda")
    idx = torch.empty((1000, 3), dtype=torch.int64, device="cuda")
    val = torch.empty(1000, dtype=torch.int64, device="cuda")
    et = np.zeros(1, np.int32)
    args = (ctx._h, nodes.data_ptr(), nodes.data_ptr(), 2, 5, 5, et.ctypes.data, 1)
    assert lib.eu_sparse_get_adj_coo(*args, 0, ptr.data_ptr(), None, None) == 0
    nnz = int(ptr[-1].item())
    assert nnz >= 2
    assert lib.eu_sparse_get_adj_coo(*args, nnz + 1, ptr.data_ptr(), idx.data_ptr(), val.data_ptr()) == 1
    assert lib.eu_sparse_get_adj_coo(*args, nnz, ptr.data_ptr(), idx.data_ptr(), val.data_ptr()) == 0
    assert lib.eu_sparse_get_adj_coo(ctx._h, nodes.data_ptr(), nodes.data_ptr(), 2, -1, 5, et.ctypes.data, 1, 0, ptr.data_ptr(),
                                     None, None) == 1
