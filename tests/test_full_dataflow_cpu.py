"""euler_b200/dataflow.py GCNDataFlow / RelationDataFlow and ops.get_multi_hop_neighbor against literal numpy restatements
of tf_euler/python/dataflow/gcn_dataflow.py + neighbor_dataflow.py:84-110 (double unique included), relation_dataflow.py
and neighbor_ops.py:209-242 + tf.sparse_reorder, driven by a CPU stand-in for the fused device hop (the oracle's full
listing + numpy first-occurrence unique).  The device hop itself is compared with this stand-in in
tests/test_full_dataflow_gpu.py."""
import numpy as np
import pytest
import torch

import graphs
from test_dataflow_cpu import np_unique_first

U64_MAX = np.uint64(2 ** 64 - 1)


class CpuFullSampler:
    """full_neighbor_hop / full_neighbor_adjacency of euler_b200.ops, restated on the host"""

    def __init__(self, g):
        self.og = graphs.oracle_graph(g)

    def _listing(self, nodes, edge_types):
        nodes = np.asarray(nodes.numpy() if torch.is_tensor(nodes) else nodes, np.int64).reshape(-1)
        lens, ids, w, t = self.og.get_full_neighbor(nodes.astype(np.uint64), list(edge_types))
        lens = np.asarray(lens, np.int64)
        return nodes, lens, ids.astype(np.int64), w, t

    def full_neighbor_hop(self, nodes, edge_types, self_loops=True, with_types=False):
        nodes, lens, vals, _w, t = self._listing(nodes, edge_types)
        n, E = len(nodes), len(vals)
        rows = np.repeat(np.arange(n, dtype=np.int64), lens)
        uniq, inv = np_unique_first(np.concatenate([vals, nodes]))
        inv = inv.astype(np.int64)
        res = inv[E:]
        if self_loops:
            ei = np.stack([np.concatenate([rows, np.arange(n, dtype=np.int64)]), inv])
        else:
            ei = np.stack([rows, inv[:E]])
        return (torch.from_numpy(uniq.astype(np.int64)), torch.from_numpy(res), torch.from_numpy(ei),
                torch.from_numpy(t.astype(np.int32)) if with_types else None)

    def full_neighbor_adjacency(self, nodes, edge_types):
        nodes, lens, vals, w, _t = self._listing(nodes, edge_types)
        nxt, col = np_unique_first(vals)
        indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        rows = np.repeat(np.arange(len(nodes)), lens)
        order = np.lexsort((col, rows))          # stable: equal (row, col) pairs keep the listing order
        return (torch.from_numpy(nxt.astype(np.int64)), torch.from_numpy(indptr), torch.from_numpy(col[order].astype(np.int64)),
                torch.from_numpy(w[order]))


# ------------------------------------------------------------------------------------------ literal restatements
def reference_gcn_flow(og, n_id, metapath, add_self_loops):
    """gcn_dataflow.py:34-48 (get_neighbors), then neighbor_dataflow.py:84-110 (UniqueDataFlow.produce_subgraph)"""
    neighbors, srcs = [], []
    cur = n_id.reshape(-1)
    for et in metapath:
        lens, ids, _, _ = og.get_full_neighbor(cur.astype(np.uint64), et)
        one = ids.astype(np.int64)
        neighbors.append(one)
        srcs.append(np.repeat(np.arange(len(cur)), lens).astype(np.int32))      # indices[:, 0], cast to int32
        cur, _ = np_unique_first(np.concatenate([one, cur]))
    blocks = []
    cur = n_id.reshape(-1)
    last_idx = np.arange(len(cur))
    for i in range(len(metapath)):
        new_u, inv = np_unique_first(np.concatenate([neighbors[i], cur]))     # the second unique of the same input
        res = inv[len(inv) - len(cur):]
        src = srcs[i]
        if add_self_loops:
            src = np.concatenate([src, last_idx])
            last_idx = np.arange(len(new_u))
            dst = inv
        else:
            dst = inv[:len(inv) - len(cur)]
            last_idx = dst
        blocks.append((new_u, res, None, np.stack([src, dst]).astype(np.int64), (len(cur), len(new_u))))
        cur = new_u
    return blocks[::-1]


def reference_relation_flow(og, n_id, metapath):
    """relation_dataflow.py:31-71: no self loops whatever add_self_loops says; e_id = the listed types"""
    neighbors, types, srcs = [], [], []
    cur = n_id.reshape(-1)
    for et in metapath:
        lens, ids, _, t = og.get_full_neighbor(cur.astype(np.uint64), et)
        neighbors.append(ids.astype(np.int64))
        types.append(t)
        srcs.append(np.repeat(np.arange(len(cur)), lens).astype(np.int32))
        cur, _ = np_unique_first(np.concatenate([neighbors[-1], cur]))
    blocks = []
    cur = n_id.reshape(-1)
    for i in range(len(metapath)):
        new_u, inv = np_unique_first(np.concatenate([neighbors[i], cur]))
        res = inv[len(inv) - len(cur):]
        dst = inv[:len(inv) - len(cur)]
        blocks.append((new_u, res, types[i], np.stack([srcs[i], dst]).astype(np.int64), (len(cur), len(new_u))))
        cur = new_u
    return blocks[::-1]


def reference_multi_hop(og, nodes, metapath):
    """neighbor_ops.py:209-242: per hop unique(listing) and the SparseTensor (indices, values, shape) after sparse_reorder"""
    nodes = nodes.reshape(-1)
    nodes_list, adj_list = [nodes], []
    for et in metapath:
        lens, ids, w, _ = og.get_full_neighbor(nodes.astype(np.uint64), et)
        nxt, idx = np_unique_first(ids.astype(np.int64))
        indices = np.stack([np.repeat(np.arange(len(nodes)), lens), idx], 1).astype(np.int64)
        order = np.lexsort((indices[:, 1], indices[:, 0]))        # sparse_reorder: row-major (ties: any order)
        adj_list.append((indices[order], w[order], (len(nodes), len(nxt))))
        nodes_list.append(nxt)
        nodes = nxt
    return nodes_list, adj_list


def same_multiset_per_pair(indices, got_w, want_w):
    """weights of equal (row, col) pairs compared as multisets: sparse_reorder promises no order among them"""
    key = np.lexsort((got_w, indices[:, 1], indices[:, 0]))
    key2 = np.lexsort((want_w, indices[:, 1], indices[:, 0]))
    return np.array_equal(got_w[key], want_w[key2])


# ------------------------------------------------------------------------------------------ cases
def make_graph(T, **kw):
    args = dict(seed=20 + T, n=600, T=T, avg_deg=4, id_stride=1, id_base=1, hub=120)
    args.update(kw)
    return graphs.random_graph(**args)


def extreme_id_graph():
    """node ids 0 .. n-1 (id 0 is a node) and edges to 2^64-1 (-1 as int64), an id no node can have: listed, never expanded"""
    g = graphs.random_graph(seed=9, n=300, T=2, avg_deg=5, id_base=0, hub=60, sorted_adj=False)
    g["nbr"][g["nbr"] == g["ids"][-1]] = U64_MAX
    return g


def roots_of(g, seed, size=48):
    rs = np.random.RandomState(seed)
    roots = g["ids"][rs.randint(0, len(g["ids"]), size=size)].astype(np.int64)
    roots[::7] = 10 ** 12                                   # absent
    roots[3::11] = roots[1]                                 # repeated
    hub = int(np.argmax(np.diff(g["grp_ptr"]))) // g["T"]
    roots[2] = np.int64(g["ids"][hub].astype(np.int64))
    return roots


GRAPHS = {
    "T1": lambda: make_graph(1),
    "T3-sparse-ids": lambda: make_graph(3, id_stride=5, id_base=7),
    "extreme-ids": extreme_id_graph,
}
# repeated types, an empty type list, out-of-range types (every type >= T of a graph lists nothing)
METAPATHS = [[[0], [0]], [[1, 0, 1], [0]], [[0], []], [[7, 0], [-1]], [[2], [0, 2]]]


def _roots_sets(g):
    roots = roots_of(g, 5)
    out = [roots, roots[:1], np.zeros(0, np.int64), np.full(5, 10 ** 12, np.int64)]    # empty input; a hop listing nothing
    if g["ids"][0] == 0:
        out.append(np.asarray([0, -1, -1, 0, 5], np.int64))
    return out


def _eq_flow(flow, want):
    assert len(flow) == len(want)
    for blk, (n_id, res, e_id, ei, size) in zip(flow, want):
        assert np.array_equal(blk.n_id.numpy(), n_id)
        assert np.array_equal(blk.res_n_id.numpy(), res)
        assert np.array_equal(blk.edge_index.numpy(), ei)
        assert blk.edge_index.dtype == torch.int64
        assert blk.size == size
        if e_id is None:
            assert blk.e_id is None
        else:
            assert np.array_equal(blk.e_id.numpy(), e_id)


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_gcn_dataflow_blocks_equal_the_reference_construction(gname):
    from euler_b200.dataflow import GCNDataFlow
    g = GRAPHS[gname]()
    og = graphs.oracle_graph(g)
    sampler = CpuFullSampler(g)
    for mp in METAPATHS:
        for roots in _roots_sets(g):
            for self_loops in (True, False):
                flow = GCNDataFlow(mp, add_self_loops=self_loops, sampler=sampler)(torch.from_numpy(roots))
                _eq_flow(flow, reference_gcn_flow(og, roots, mp, self_loops))


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_relation_dataflow_blocks_equal_the_reference_construction(gname):
    from euler_b200.dataflow import RelationDataFlow
    g = GRAPHS[gname]()
    og = graphs.oracle_graph(g)
    sampler = CpuFullSampler(g)
    for mp in METAPATHS:
        for roots in _roots_sets(g):
            for self_loops in (True, False):           # ignored, as in the reference
                flow = RelationDataFlow([5] * len(mp), mp, add_self_loops=self_loops, sampler=sampler)(torch.from_numpy(roots))
                _eq_flow(flow, reference_relation_flow(og, roots, mp))


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_get_multi_hop_neighbor_equals_the_reference_op(gname):
    from euler_b200.ops import get_multi_hop_neighbor
    g = GRAPHS[gname]()
    og = graphs.oracle_graph(g)
    sampler = CpuFullSampler(g)
    for mp in METAPATHS + [[[0]] * 3]:
        for roots in _roots_sets(g):
            nodes_list, adj_list = get_multi_hop_neighbor(torch.from_numpy(roots.reshape(-1, 1)), mp, sampler=sampler)
            w_nodes, w_adj = reference_multi_hop(og, roots, mp)
            assert len(nodes_list) == len(w_nodes) == len(mp) + 1
            assert np.array_equal(nodes_list[0].numpy(), roots)                  # the input, flattened, not uniqued
            for got, want in zip(nodes_list[1:], w_nodes[1:]):
                assert np.array_equal(got.numpy(), want)
            for (indptr, cols, w), (indices, values, shape) in zip(adj_list, w_adj):
                indptr = indptr.numpy()
                assert len(indptr) == shape[0] + 1
                rows = np.repeat(np.arange(shape[0]), np.diff(indptr))
                got_idx = np.stack([rows, cols.numpy()], 1)
                assert np.array_equal(got_idx, indices)
                assert same_multiset_per_pair(indices, w.numpy(), values)
                assert cols.numel() == 0 or cols.max().item() < shape[1]

