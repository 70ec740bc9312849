"""The fused full-neighbor hop (eu_full_neighbor_hop, euler_b200/csrc/full_hop.cu) on the GPU: bit-exact against the CPU
stand-in of tests/test_full_dataflow_cpu.py for every integer output and weight, equal to the composition of the existing
ops on an R-MAT graph, and GCNDataFlow / RelationDataFlow blocks feeding the convolutions end to end."""
import os
import sys

import numpy as np
import pytest
import torch

import cases
import graphs
from test_full_dataflow_cpu import CpuFullSampler, extreme_id_graph

pytestmark = pytest.mark.gpu
RTOL = 1e-5


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def _frontiers(g, rs):
    """frontier sizes 0, 1, 31 and ~10^5 (warp, CTA and grid-stride boundaries), the hub in each non-empty one, absent and
    repeated nodes"""
    hub = g["ids"][int(np.argmax(np.diff(g["grp_ptr"]))) // g["T"]].astype(np.int64)
    out = []
    for n in (0, 1, 31, 1000, 100_003):
        f = g["ids"][rs.randint(0, len(g["ids"]), size=n)].astype(np.int64)
        if n:
            f[0] = hub
            f[5::13] = 10 ** 15
        out.append(f)
    return out


def _hop_case(g, metapath_types):
    import euler_b200
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    cpu = CpuFullSampler(g)
    rs = np.random.RandomState(4)
    for nodes in _frontiers(g, rs):
        d_nodes = torch.from_numpy(nodes).cuda()
        for et in metapath_types:
            for self_loops in (True, False):
                got = euler_b200.full_neighbor_hop(d_nodes, et, self_loops, True)
                want = cpu.full_neighbor_hop(torch.from_numpy(nodes), et, self_loops, True)
                for nm, a, b in zip(("n_id", "res_n_id", "edge_index", "types"), got, want):
                    cases.eq(a.cpu().numpy(), b.numpy(), "%s n=%d et=%s self_loops=%s" % (nm, len(nodes), et, self_loops))
            got = euler_b200.full_neighbor_adjacency(d_nodes, et)
            want = cpu.full_neighbor_adjacency(torch.from_numpy(nodes), et)
            for nm, a, b in zip(("next", "indptr", "cols", "weights"), got, want):
                cases.eq(a.cpu().numpy(), b.numpy(), "adjacency %s n=%d et=%s" % (nm, len(nodes), et))


@pytest.mark.parametrize("T,stride", [(1, 1), (3, 7)])
def test_device_hop_equals_the_cpu_stand_in(T, stride):
    """dense ids (T=1) and hashed sparse ids (T=3) with a 4000-edge hub; every flag combination the Python layers use"""
    g = graphs.random_graph(seed=31 + T, n=20_000, T=T, avg_deg=5, id_stride=stride, id_base=3, hub=4000, zero_w_frac=0.1)
    _hop_case(g, [[0], list(range(T))[::-1], [T - 1, 0, T - 1], [], [9, 0]])


def test_device_hop_with_ids_zero_and_minus_one():
    g = extreme_id_graph()
    import euler_b200
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    cpu = CpuFullSampler(g)
    nodes = np.asarray([0, -1, -1, 0, 5, 10 ** 15, 7], np.int64)
    for et in ([0, 1], [1, 1]):
        got = euler_b200.full_neighbor_hop(torch.from_numpy(nodes).cuda(), et, True, True)
        want = cpu.full_neighbor_hop(torch.from_numpy(nodes), et, True, True)
        for a, b in zip(got, want):
            cases.eq(a.cpu().numpy(), b.numpy(), "extreme ids et=%s" % et)
        got = euler_b200.get_multi_hop_neighbor(nodes, [et, et])
        want = euler_b200.get_multi_hop_neighbor(torch.from_numpy(nodes), [et, et], sampler=cpu)
        for a, b in zip(got[0], want[0]):
            cases.eq(a.cpu().numpy(), b.numpy(), "multi-hop nodes")
        for a, b in zip(got[1], want[1]):
            for x, y in zip(a, b):
                cases.eq(x.cpu().numpy(), y.numpy(), "multi-hop adjacency")


def test_dataflows_equal_the_composition_of_existing_ops_on_rmat():
    """GCNDataFlow on a 1M-node R-MAT graph, 2 hops == the composition timed by benchmarks/full_dataflow.py
    (get_full_neighbor + cat / repeat_interleave + unique once per hop); RelationDataFlow's blocks are the same without the
    self loops, e_id = the listed types"""
    import euler_b200
    from euler_b200.dataflow import GCNDataFlow, RelationDataFlow
    sys.path.insert(0, os.path.join(graphs.ROOT, "benchmarks"))
    from full_dataflow import composed_gcn_flow
    gr = euler_b200.Graph.rmat(1_000_000, 10_000_000, seed=42)
    euler_b200.set_graph(gr, seed=1)
    seeds = torch.from_numpy(np.random.RandomState(3).randint(1, 1_000_001, size=512).astype(np.int64)).cuda()
    for self_loops in (True, False):
        flow = GCNDataFlow([[0], [0]], add_self_loops=self_loops)(seeds)
        comp = composed_gcn_flow(euler_b200, seeds, [[0], [0]], self_loops)
        assert len(flow) == 2
        for blk, (n_id, res, ei) in zip(flow.blocks, comp):
            assert torch.equal(blk.n_id, n_id) and torch.equal(blk.res_n_id, res) and torch.equal(blk.edge_index, ei)
            assert blk.e_id is None and blk.size == (res.numel(), n_id.numel())
    rflow = RelationDataFlow([10, 10], [[0], [0]])(seeds)
    comp = composed_gcn_flow(euler_b200, seeds, [[0], [0]], False)
    cur = seeds
    for blk, (n_id, res, ei) in zip(rflow.blocks, comp):
        assert torch.equal(blk.n_id, n_id) and torch.equal(blk.res_n_id, res) and torch.equal(blk.edge_index, ei)
        _, _, _, t = euler_b200.get_full_neighbor(cur, [0])
        assert torch.equal(blk.e_id, t)
        cur = n_id
    assert comp[1][2].shape[1] > 100_000        # hop 2 spans many CTAs and grid-stride rounds


def test_gcn_and_relation_blocks_feed_the_convolutions():
    """GCNDataFlow -> get_dense_feature -> gcn_aggregate and RelationDataFlow -> relation_aggregate against numpy over the
    same blocks (1e-5 relative: the aggregation scatters atomically)"""
    import euler_b200
    from euler_b200 import convolution as conv
    from euler_b200.dataflow import GCNDataFlow, RelationDataFlow
    D = 32
    g = graphs.random_graph(seed=8, n=3000, T=2, avg_deg=4, feat_dim=D, hub=500)
    euler_b200.set_graph(graphs.cuda_graph(g), seed=1)
    rs = np.random.RandomState(6)
    roots = torch.from_numpy(g["ids"][rs.randint(0, 3000, size=200)].astype(np.int64)).cuda()
    flow = GCNDataFlow([[0, 1], [1]])(roots)
    for blk in flow:
        x = euler_b200.get_dense_feature(blk.n_id, [0], [D])[0]
        got = conv.gcn_aggregate((None, x), blk.edge_index, blk.size).cpu().numpy()
        e0, e1 = blk.edge_index.cpu().numpy()
        x1 = x.cpu().numpy().astype(np.float64)
        deg0 = np.bincount(e0, minlength=blk.size[0]).astype(np.float64)
        deg1 = np.bincount(e1, minlength=blk.size[1]).astype(np.float64)
        want = np.zeros((blk.size[0], D))
        np.add.at(want, e0, ((deg0[e0] ** -0.5) * (deg1[e1] ** -0.5))[:, None] * x1[e1])
        assert np.allclose(got, want, rtol=RTOL, atol=1e-5)
    R, dim = 2, 16
    mat = torch.from_numpy(rs.randn(R, dim, D).astype(np.float32) * 0.1).cuda()
    rflow = RelationDataFlow([5, 5], [[0, 1], [1, 0]])(roots)
    for blk in rflow:
        x = euler_b200.get_dense_feature(blk.n_id, [0], [D])[0]
        got = conv.relation_aggregate((None, x), blk.edge_index, blk.size, blk.e_id, mat).cpu().numpy()
        e0, e1 = blk.edge_index.cpu().numpy()
        attr = blk.e_id.cpu().numpy()
        msg = np.einsum("eij,ej->ei", mat.cpu().numpy()[attr].astype(np.float64), x.cpu().numpy()[e1].astype(np.float64))
        s = np.zeros((blk.size[0], dim))
        np.add.at(s, e0, msg)
        want = s / (np.bincount(e0, minlength=blk.size[0])[:, None] + 1e-7)
        assert np.allclose(got, want, rtol=RTOL, atol=1e-4)


def test_hop_argument_checks():
    """flag combinations outside the contract are refused before any work"""
    import euler_b200
    from euler_b200 import _lib
    g = graphs.random_graph(seed=2, n=100, T=1)
    euler_b200.set_graph(graphs.cuda_graph(g))
    lib, ctx = _lib.load(), euler_b200.context()
    nodes = torch.arange(1, 11, dtype=torch.int64, device="cuda")
    ptr = torch.empty(11, dtype=torch.int64, device="cuda")
    et = np.zeros(1, np.int32)
    for flags in (2, 6, 8):              # self loops without the frontier, self loops with sorting, an unknown flag
        assert lib.eu_full_neighbor_hop(ctx._h, nodes.data_ptr(), 10, et.ctypes.data, 1, flags, 0, ptr.data_ptr(),
                                        None, None, None, None, None, None, None) == 1
    assert lib.eu_full_neighbor_hop(ctx._h, nodes.data_ptr(), 10, et.ctypes.data, 1, 1, 0, ptr.data_ptr(),
                                    None, None, None, None, None, None, None) == 0
    assert torch.equal(ptr.cpu()[1:] - ptr.cpu()[:-1], torch.from_numpy(np.diff(g["grp_ptr"])[:10]))
