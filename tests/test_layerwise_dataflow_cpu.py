"""euler_b200/dataflow.py LayerwiseDataFlow ('adapt') / LayerwiseEachDataFlow ('layerwise') against literal numpy restatements
of tf_euler/python/dataflow/layerwise_dataflow.py + neighbor_dataflow.py, driven by a CPU stand-in sampler: the oracle's full
listing, seeded numpy draws from the (dst, type) candidate set and a numpy restatement of the SparseTensor that
tf_euler/kernels/sparse_get_adj_op.cc:84-117 builds (filler entry included).  The device op eu_sparse_get_adj_coo and the
device dataflows are compared with this stand-in in tests/test_layerwise_dataflow_gpu.py."""
import numpy as np
import pytest
import torch

import graphs
from test_dataflow_cpu import np_unique_first
from test_full_dataflow_cpu import extreme_id_graph

ABSENT = 10 ** 12


# ------------------------------------------------------------------------------------------ the adjacency builder
def literal_sparse_get_adj(og, nodes, nb, edge_types):
    """sparse_get_adj_op.cc:84-117 line by line: per batch row the set of (src, dst) pairs listed by its nodes, then every
    (j, k) in row-major order -- 1 if (nodes[b, j], nb[b, k]) is in the set, else 0 at (N-1, M-1) only"""
    batch, N = nodes.shape
    M = nb.shape[1]
    flat = nodes.reshape(-1)
    lens, ids, _, _ = og.get_full_neighbor(flat.astype(np.uint64), list(edge_types))
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = ids.astype(np.int64)
    idx, val = [], []
    for i in range(batch):
        relation = set()
        for j in range(N * i, N * (i + 1)):
            for k in range(ptr[j], ptr[j + 1]):
                relation.add((int(flat[j]), int(ids[k])))
        for j in range(N):
            for k in range(M):
                if (int(nodes[i, j]), int(nb[i, k])) in relation:
                    idx.append((i, j, k))
                    val.append(1)
                elif j == N - 1 and k == M - 1:
                    idx.append((i, j, k))
                    val.append(0)
    return np.asarray(idx, np.int64).reshape(-1, 3), np.asarray(val, np.int64), (batch, N, M)


def np_sparse_get_adj(og, nodes, nb, edge_types):
    """the same SparseTensor, vectorised for large batches: membership of (b, nodes[b, j], nb[b, k]) among the batch row's
    listed (b, src, dst) triples, over ids renumbered densely"""
    batch, N = nodes.shape
    M = nb.shape[1]
    if batch * N == 0 or M == 0:
        return np.zeros((0, 3), np.int64), np.zeros(0, np.int64), (batch, N, M)
    flat = nodes.reshape(-1)
    lens, ids, _, _ = og.get_full_neighbor(flat.astype(np.uint64), list(edge_types))
    ids = ids.astype(np.int64)
    vocab = np.unique(np.concatenate([flat, ids, nb.reshape(-1)]))
    U = np.int64(len(vocab))
    code = lambda x: np.searchsorted(vocab, x).astype(np.int64)          # noqa: E731
    row = np.repeat(np.arange(batch * N), lens)
    listed = ((row // N) * U + code(flat[row])) * U + code(ids)
    b = np.arange(batch, dtype=np.int64)[:, None, None]
    query = (b * U + code(nodes)[:, :, None]) * U + code(nb)[:, None, :]
    hit = np.isin(query, listed)
    keep = hit.copy()
    keep[:, N - 1, M - 1] = True
    return np.argwhere(keep).astype(np.int64), hit[keep].astype(np.int64), (batch, N, M)


# ------------------------------------------------------------------------------------------ CPU stand-in
class CpuLayerwiseSampler:
    """sample_neighbor / sample_neighbor_layerwise_coo / get_full_neighbor / unique of euler_b200.ops on the host.  Draws are
    seeded numpy draws (sample_neighbor: uniform over the node's listing; layer-wise: weighted over the batch row's (dst, type)
    candidates), or with `replay` the given arrays in call order.  Every draw is logged with the nodes it was drawn for."""

    def __init__(self, g, seed=0, replay=None):
        self.og = graphs.oracle_graph(g)
        self.rs = np.random.RandomState(seed)
        self.replay = None if replay is None else list(replay)
        self.log = []

    @staticmethod
    def _np(x):
        return np.asarray(x.numpy() if torch.is_tensor(x) else x, np.int64)

    def _next(self, nodes, draw):
        out = self.replay.pop(0) if self.replay is not None else draw()
        self.log.append((nodes, out))
        return out

    def get_full_neighbor(self, nodes, edge_types):
        lens, ids, w, t = self.og.get_full_neighbor(self._np(nodes).reshape(-1).astype(np.uint64), list(edge_types))
        indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        return torch.from_numpy(indptr), torch.from_numpy(ids.astype(np.int64)), torch.from_numpy(w), torch.from_numpy(t)

    def unique(self, ids):
        v, inv = np_unique_first(self._np(ids))
        return torch.from_numpy(v.astype(np.int64)), torch.from_numpy(inv.astype(np.int32))

    def sample_neighbor(self, nodes, edge_types, count, default_node=-1):
        nodes = self._np(nodes).reshape(-1)

        def draw():
            lens, ids, _, _ = self.og.get_full_neighbor(nodes.astype(np.uint64), list(edge_types))
            ptr = np.concatenate([[0], np.cumsum(lens)])
            out = np.full((len(nodes), count), default_node, np.int64)
            for i in range(len(nodes)):
                if lens[i]:
                    out[i] = ids[ptr[i] + self.rs.randint(0, lens[i], size=count)].astype(np.int64)
            return out
        out = self._next(nodes, draw)
        return torch.from_numpy(out), None, None

    def sample_neighbor_layerwise_coo(self, nodes, edge_types, count, default_node=-1, weight_func=''):
        nodes = self._np(nodes)
        batch, n = nodes.shape

        def draw():
            out = np.full((batch, count), default_node, np.int64)
            if n == 0:
                return out
            lens, ids, w, t = self.og.get_full_neighbor(nodes.reshape(-1).astype(np.uint64), list(edge_types))
            ptr = np.concatenate([[0], np.cumsum(lens)])
            for b in range(batch):
                lo, hi = ptr[b * n], ptr[(b + 1) * n]
                cand = {}
                for k in range(lo, hi):
                    key = (int(ids[k].astype(np.int64)), int(t[k]))
                    cand[key] = cand.get(key, 0.0) + float(w[k])
                wt = np.asarray(list(cand.values()), np.float64)
                if weight_func == 'sqrt':
                    wt = np.sqrt(wt)
                if len(cand) and wt.sum() > 0:
                    dst = np.asarray([d for d, _ in cand], np.int64)
                    out[b] = dst[self.rs.choice(len(dst), size=count, p=wt / wt.sum())]
            return out
        out = self._next(nodes, draw)
        idx, val, shape = np_sparse_get_adj(self.og, nodes, out, edge_types)
        return torch.from_numpy(out), (torch.from_numpy(idx), torch.from_numpy(val), shape)


# ------------------------------------------------------------------------------------------ literal restatements
def _draws(log):
    """the stand-in's draws in call order, checking that the restatement asks for them with the same nodes"""
    it = iter(log)

    def take(nodes):
        got_nodes, out = next(it)
        assert np.array_equal(got_nodes, nodes)
        return out
    return take


def unique_produce_subgraph(n_id, neighbors, srcs, add_self_loops):
    """neighbor_dataflow.py:84-110 (UniqueDataFlow.produce_subgraph)"""
    blocks = []
    cur = n_id.reshape(-1)
    last_idx = np.arange(len(cur))
    for i in range(len(neighbors)):
        new_u, inv = np_unique_first(np.concatenate([neighbors[i], cur]))
        res = inv[len(inv) - len(cur):]
        src = srcs[i]
        if add_self_loops:
            src = np.concatenate([src, last_idx])
            last_idx = np.arange(len(new_u))
            dst = inv
        else:
            dst = inv[:len(inv) - len(cur)]
            last_idx = dst
        blocks.append((new_u, res, np.stack([src, dst]).astype(np.int64), (len(cur), len(new_u))))
        cur = new_u
    return blocks[::-1]


def neighbor_produce_subgraph(n_id, neighbors, srcs, add_self_loops):
    """neighbor_dataflow.py:45-68 (NeighborDataFlow.produce_subgraph, no unique; TF's [-0:] / [:-0] slices kept)"""
    blocks = []
    cur = n_id.reshape(-1)
    last_idx = np.arange(len(cur))
    for i in range(len(neighbors)):
        new = np.concatenate([neighbors[i], cur])
        new_inv = np.arange(len(new))
        res = new_inv[-len(cur):]
        src = srcs[i]
        if add_self_loops:
            src = np.concatenate([src, last_idx])
            last_idx = new_inv
        else:
            new_inv = new_inv[:-len(cur)]
            last_idx = new_inv
        blocks.append((new, res, np.stack([src, new_inv]).astype(np.int64), (len(cur), len(new))))
        cur = new
    return blocks[::-1]


def reference_layerwise_flow(og, n_id, metapath, fanouts, add_self_loops, take):
    """layerwise_dataflow.py:35-62 (LayerwiseDataFlow.get_neighbors), then UniqueDataFlow.produce_subgraph"""
    neighbors, srcs = [], []
    cur = n_id.reshape(-1)
    total_fanout = 0
    for i in range(len(metapath)):
        if i == len(metapath) - 1:
            lens, ids, _, _ = og.get_full_neighbor(cur.astype(np.uint64), metapath[i])
            one_indices = np.repeat(np.arange(len(cur)), lens)
            one = ids.astype(np.int64)
        else:
            total_fanout += fanouts[i]
            last_count = len(cur)
            unique_neighbor = take(cur.reshape(1, last_count))
            assert unique_neighbor.shape == (1, total_fanout)
            idx, _, _ = literal_sparse_get_adj(og, cur.reshape(1, last_count), unique_neighbor, metapath[i])
            one = unique_neighbor.reshape(-1)[idx[:, 2]]
            one_indices = idx[:, 1]
        neighbors.append(one.reshape(-1))
        srcs.append(one_indices.astype(np.int32))
        cur, _ = np_unique_first(np.concatenate([one.reshape(-1), cur]))
    return unique_produce_subgraph(n_id, neighbors, srcs, add_self_loops)


def reference_layerwise_each_flow(og, n_id, metapath, fanouts, add_self_loops, take):
    """layerwise_dataflow.py:79-119 (get_neighbors_sage + get_neighbors_layer), then NeighborDataFlow.produce_subgraph"""
    cur = n_id.reshape(-1)
    count = fanouts[0]
    one = take(cur)
    neighbors = [one.reshape(-1)]
    srcs = [np.tile(np.arange(len(cur)).reshape(-1, 1), [1, count]).reshape(-1)]
    cur, last_count = neighbors[-1], fanouts[0]
    for et, count in zip(metapath[1:], fanouts[1:]):
        nodes2d = cur.reshape(-1, last_count)
        unique_neighbor = take(nodes2d)
        idx, _, _ = literal_sparse_get_adj(og, nodes2d, unique_neighbor, et)
        one = unique_neighbor.reshape(-1)[idx[:, 2] + idx[:, 0] * count]
        neighbors.append(one.reshape(-1))
        srcs.append((idx[:, 1] + idx[:, 0] * last_count).astype(np.int32))
        cur, last_count = one, count
    return neighbor_produce_subgraph(n_id, neighbors, srcs, add_self_loops)


def eq_flow(flow, want):
    assert len(flow) == len(want)
    for blk, (n_id, res, ei, size) in zip(flow, want):
        assert np.array_equal(np.asarray(blk.n_id.cpu()), n_id)
        assert np.array_equal(np.asarray(blk.res_n_id.cpu()), res)
        assert np.array_equal(np.asarray(blk.edge_index.cpu()), ei)
        assert blk.edge_index.dtype == torch.int64
        assert blk.size == size and blk.e_id is None


# ------------------------------------------------------------------------------------------ cases
def make_graph(T, **kw):
    args = dict(seed=40 + T, n=500, T=T, avg_deg=4, id_stride=1, id_base=1, hub=150)
    args.update(kw)
    return graphs.random_graph(**args)


GRAPHS = {
    "T1": lambda: make_graph(1),
    "T3-sparse-ids": lambda: make_graph(3, id_stride=5, id_base=7),
    "extreme-ids": extreme_id_graph,
}


def hub_of(g):
    return np.int64(g["ids"][int(np.argmax(np.diff(g["grp_ptr"]))) // g["T"]].astype(np.int64))


def roots_sets(g):
    rs = np.random.RandomState(5)
    roots = g["ids"][rs.randint(0, len(g["ids"]), size=24)].astype(np.int64)
    roots[::7] = ABSENT                                     # absent
    roots[3::8] = roots[1]                                  # repeated
    roots[2] = hub_of(g)
    out = [roots, roots[2:3], np.zeros(0, np.int64), np.full(4, ABSENT, np.int64)]   # one root; empty; no candidates at all
    if g["ids"][0] == 0:
        out.append(np.asarray([0, -1, -1, 0, 5], np.int64))
    return out


def test_vectorised_adjacency_equals_the_literal_loop():
    """np_sparse_get_adj (the stand-in's and the GPU tests' restatement) == the loop of sparse_get_adj_op.cc, on multi-edges,
    one and three edge types, a hub, absent and repeated nodes and neighbors, ids 0 and 2^64-1, N = 1, M = 1, empty inputs"""
    for gname in sorted(GRAPHS):
        g = GRAPHS[gname]()
        og = graphs.oracle_graph(g)
        rs = np.random.RandomState(8)
        for batch, N, M in [(1, 1, 1), (3, 1, 5), (2, 6, 1), (4, 7, 9), (1, 30, 40), (0, 3, 3), (2, 0, 4), (2, 3, 0)]:
            nodes = g["ids"][rs.randint(0, len(g["ids"]), size=(batch, N))].astype(np.int64)
            if nodes.size:
                nodes.reshape(-1)[::5] = ABSENT
                nodes[0, 0] = hub_of(g)
                nodes[-1, -1] = nodes[0, 0]
            lens, ids, _, _ = og.get_full_neighbor(nodes.reshape(-1).astype(np.uint64), [0])
            pool = np.concatenate([ids.astype(np.int64), g["ids"][:50].astype(np.int64), [ABSENT, -1, 0]])
            nb = pool[rs.randint(0, len(pool), size=(batch, M))]
            if nb.size:
                nb.reshape(-1)[1::4] = nb.reshape(-1)[0]         # a neighbor repeated in nb
            for et in ([0], [0, 0], [], [9], list(range(g["T"]))[::-1]):
                a = literal_sparse_get_adj(og, nodes, nb, et)
                b = np_sparse_get_adj(og, nodes, nb, et)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2], (gname, batch, N, M, et)
                if batch * N and M:
                    assert len(set(a[0][:, 0].tolist())) == batch          # every batch row has an entry: a 1 or the filler


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_layerwise_dataflow_blocks_equal_the_reference_construction(gname):
    from euler_b200.dataflow import LayerwiseDataFlow
    g = GRAPHS[gname]()
    og = graphs.oracle_graph(g)
    for metapath, fanouts in [([[0], [0]], [6, 6]), ([[0, 1], [1], [0]], [3, 4, 0]), ([[0]], [5]), ([[1], [1, 0]], [1, 1])]:
        for roots in roots_sets(g):
            for self_loops in (True, False):
                sampler = CpuLayerwiseSampler(g, seed=len(roots))
                flow = LayerwiseDataFlow(fanouts, metapath, add_self_loops=self_loops, sampler=sampler)(torch.from_numpy(roots))
                want = reference_layerwise_flow(og, roots, metapath, fanouts, self_loops, _draws(sampler.log))
                eq_flow(flow, want)


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_layerwise_each_dataflow_blocks_equal_the_reference_construction(gname):
    from euler_b200.dataflow import LayerwiseEachDataFlow
    g = GRAPHS[gname]()
    og = graphs.oracle_graph(g)
    # a third hop reshapes the second hop's edges into rows of fanouts[1]: fanouts[1] = 1 always divides
    for metapath, fanouts in [([[0], [0]], [3, 4]), ([[0, 1], [1], [0]], [2, 1, 3]), ([[0]], [2])]:
        for roots in roots_sets(g):
            for self_loops in (True, False):
                sampler = CpuLayerwiseSampler(g, seed=7 + len(roots))
                flow = LayerwiseEachDataFlow(fanouts, metapath, add_self_loops=self_loops, max_id=10 ** 7,
                                             sampler=sampler)(torch.from_numpy(roots))
                want = reference_layerwise_each_flow(og, roots, metapath, fanouts, self_loops, _draws(sampler.log))
                eq_flow(flow, want)


def test_empty_frontier_brings_the_default_node_in():
    """a frontier without candidates draws default_node (-1) only; the filler entry makes it an edge and a node of the
    next frontier, as upstream"""
    from euler_b200.dataflow import LayerwiseDataFlow
    g = make_graph(1)
    sampler = CpuLayerwiseSampler(g)
    roots = np.full(3, ABSENT, np.int64)
    flow = LayerwiseDataFlow([4, 4], [[0], [0]], sampler=sampler)(torch.from_numpy(roots))
    hop1 = flow.blocks[0]
    assert hop1.n_id.tolist() == [-1, ABSENT]
    assert hop1.edge_index.tolist() == [[2, 0, 1, 2], [0, 1, 1, 1]]      # the filler (row 2 -> draw 3 = -1), then self loops
