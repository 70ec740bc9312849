"""Minibatch subgraph construction for the message-passing convolutions: the reference's NeighborDataFlow /
UniqueDataFlow / SageDataFlow / GCNDataFlow / RelationDataFlow / LayerwiseDataFlow / LayerwiseEachDataFlow
(tf_euler/python/dataflow/{base,neighbor,sage,gcn,relation,layerwise}_dataflow.py) over this package's ops.

A DataFlow is the list of Blocks a convolution stack consumes, deepest hop first (base_dataflow.py:19-52):
    block.n_id        node ids of the block's source side (hop l+1 frontier [+ the destination nodes])
    block.res_n_id    positions of the destination nodes inside n_id
    block.edge_index  [2, E]: edge_index[0] = index into the destination nodes, edge_index[1] = index into n_id
    block.size        (number of destination nodes, number of source nodes)

Tensors stay on the device; the only host syncs are shapes, as in TF: the unique count of UniqueDataFlow, per hop of
GCNDataFlow / RelationDataFlow the listing total and the unique count, and per layer-wise hop the adjacency's entry count.
`sampler` is any object with sample_neighbor(nodes, edge_types, count, default_node) -> (ids[B, count], w, t),
unique(ids) -> (values, inverse), full_neighbor_hop(nodes, edge_types, self_loops, with_types) -> (n_id, res_n_id,
edge_index, types), get_full_neighbor(nodes, edge_types) -> (indptr, ids, w, t) and
sample_neighbor_layerwise_coo(nodes[batch, n], edge_types, count) -> (ids[batch, count], (indices[nnz, 3], values, shape)):
euler_b200 itself on the GPU, or a CPU stand-in in the tests."""
import torch


class Block:
    def __init__(self, n_id, res_n_id, e_id, edge_index, size):
        self.n_id, self.res_n_id, self.e_id, self.edge_index, self.size = n_id, res_n_id, e_id, edge_index, size


class DataFlow:
    """base_dataflow.py:31-52"""

    def __init__(self, n_id):
        self.n_id = n_id
        self._last = n_id
        self.blocks = []

    def append(self, n_id, res_n_id, e_id, edge_index):
        self.blocks.append(Block(n_id, res_n_id, e_id, edge_index, (int(self._last.numel()), int(n_id.numel()))))
        self._last = n_id

    def __len__(self):
        return len(self.blocks)

    def __getitem__(self, idx):
        return self.blocks[::-1][idx]

    def __iter__(self):
        return iter(self.blocks[::-1])


def _default_sampler():
    import euler_b200
    return euler_b200


class NeighborDataFlow:
    """neighbor_dataflow.py:24-73: no de-duplication; block l's sources are [hop-l neighbors, destinations]."""

    def __init__(self, num_hops, add_self_loops=True, sampler=None):
        self.num_hops, self.add_self_loops = num_hops, add_self_loops
        self.sampler = sampler or _default_sampler()

    def get_neighbors(self, n_id):
        raise NotImplementedError

    def _merge(self, new_n_id):
        """identity numbering (no unique): values, inverse"""
        return new_n_id, torch.arange(new_n_id.numel(), device=new_n_id.device)

    def produce_subgraph(self, n_id):
        n_id = n_id.reshape(-1)
        last_idx = torch.arange(n_id.numel(), device=n_id.device)
        flow = DataFlow(n_id)
        neighbors, edge_srcs = self.get_neighbors(n_id)
        for i in range(self.num_hops):
            n_prev = n_id.numel()
            cat = torch.cat([neighbors[i], n_id])
            new_n_id, new_inv = self._merge(cat)
            res_n_id = new_inv[-n_prev:]
            edge_src = edge_srcs[i]
            if self.add_self_loops:
                edge_src = torch.cat([edge_src, last_idx])
                last_idx = torch.arange(new_n_id.numel(), device=n_id.device)
                edge_dst = new_inv
            else:
                edge_dst = new_inv[:-n_prev]
                last_idx = edge_dst
            n_id = new_n_id
            flow.append(new_n_id, res_n_id, None, torch.stack([edge_src.to(torch.int64), edge_dst.to(torch.int64)]))
        return flow

    __call__ = produce_subgraph


class UniqueDataFlow(NeighborDataFlow):
    """neighbor_dataflow.py:76-109: every block's source side is tf.unique'd (first-occurrence order)."""

    def _merge(self, new_n_id):
        values, inverse = self.sampler.unique(new_n_id)
        return values, inverse.to(torch.int64)


class SageDataFlow(UniqueDataFlow):
    """sage_dataflow.py:24-50: fixed-fanout sample_neighbor per hop; the next hop samples from unique(neighbors + nodes)."""

    def __init__(self, fanouts, metapath, add_self_loops=True, max_id=-1, sampler=None):
        super().__init__(num_hops=len(metapath), add_self_loops=add_self_loops, sampler=sampler)
        self.fanouts, self.metapath, self.max_id = fanouts, metapath, max_id

    def get_neighbors(self, n_id):
        neighbors, neighbor_src = [], []
        for hop_edge_types, count in zip(self.metapath, self.fanouts):
            n_id = n_id.reshape(-1)
            one, _w, _t = self.sampler.sample_neighbor(n_id, hop_edge_types, count, default_node=self.max_id + 1)
            one = one.reshape(-1)
            neighbors.append(one)
            neighbor_src.append(torch.arange(n_id.numel(), device=n_id.device).repeat_interleave(count))
            n_id, _ = self.sampler.unique(torch.cat([one, n_id]))
        return neighbors, neighbor_src


class GCNDataFlow:
    """gcn_dataflow.py:26-48 over UniqueDataFlow.produce_subgraph (neighbor_dataflow.py:84-110): every hop lists the full
    neighborhood of its frontier (metapath[h]'s edge types) and the next frontier is unique(concat(neighbors, frontier)).
    The reference computes that unique twice per hop (in get_neighbors and again in produce_subgraph, on the same input);
    here one fused hop (sampler.full_neighbor_hop) lists, renumbers and emits the block's edges.  e_id is None."""
    with_types = False     # e_id = the listed edge types

    def __init__(self, metapath, add_self_loops=True, sampler=None):
        self.metapath, self.add_self_loops = metapath, add_self_loops
        self.sampler = sampler or _default_sampler()

    def produce_subgraph(self, n_id):
        n_id = n_id.reshape(-1)
        flow = DataFlow(n_id)
        for hop_edge_types in self.metapath:
            n_id, res_n_id, edge_index, types = self.sampler.full_neighbor_hop(n_id, hop_edge_types, self.add_self_loops,
                                                                                self.with_types)
            flow.append(n_id, res_n_id, types, edge_index)
        return flow

    __call__ = produce_subgraph


class RelationDataFlow(GCNDataFlow):
    """relation_dataflow.py:25-71: GCNDataFlow's blocks without self loops -- whatever add_self_loops says, as in the
    reference -- and with e_id = the edge type of every listed edge (i32), for RelationConv.  fanouts is accepted and
    unused, as there."""
    with_types = True

    def __init__(self, fanouts, metapath, add_self_loops=True, sampler=None):
        super().__init__(metapath, add_self_loops=False, sampler=sampler)
        self.fanouts = fanouts


def _full_listing(sampler, n_id, edge_types):
    """get_full_neighbor(n_id)[0] as (values, indices[:, 0]): the listed ids and the row of each"""
    indptr, ids, _w, _t = sampler.get_full_neighbor(n_id, edge_types)
    rows = torch.arange(n_id.numel(), device=n_id.device).repeat_interleave(indptr[1:] - indptr[:-1], output_size=ids.numel())
    return ids, rows


class LayerwiseDataFlow(UniqueDataFlow):
    """layerwise_dataflow.py:26-62 ('adapt', AdaptiveGCN): every hop but the last draws total_fanout = the sum of the fanouts so
    far from the union of the whole frontier's neighbors (one batch row), and its edges are the adjacency's entries (row j ->
    the k-th draw); the last hop lists the frontier's full neighborhoods.  As upstream, the adjacency's filler entry (value 0,
    sparse_get_adj_coo) is an edge too, and a frontier without candidates brings default_node (-1) into n_id."""

    def __init__(self, fanouts, metapath, add_self_loops=True, sampler=None):
        super().__init__(num_hops=len(metapath), add_self_loops=add_self_loops, sampler=sampler)
        self.fanouts, self.metapath = fanouts, metapath

    def get_neighbors(self, n_id):
        neighbors, neighbor_src = [], []
        total_fanout = 0
        for i, hop_edge_types in enumerate(self.metapath):
            n_id = n_id.reshape(-1)
            if i == len(self.metapath) - 1:
                one, src = _full_listing(self.sampler, n_id, hop_edge_types)
            else:
                total_fanout += self.fanouts[i]
                drawn, (indices, _v, _shape) = self.sampler.sample_neighbor_layerwise_coo(n_id.reshape(1, -1), hop_edge_types,
                                                                                          total_fanout)
                one = drawn.reshape(-1)[indices[:, 2]]
                src = indices[:, 1]
            neighbors.append(one)
            neighbor_src.append(src)
            n_id, _ = self.sampler.unique(torch.cat([one, n_id]))
        return neighbors, neighbor_src


class LayerwiseEachDataFlow(NeighborDataFlow):
    """layerwise_dataflow.py:65-119 ('layerwise'), no de-duplication: hop 1 is sample_neighbor(fanouts[0]) with default_node =
    max_id + 1; every later hop reshapes the previous hop's neighbors into rows of the previous fanout, draws fanouts[h] per row
    from the row's union of neighbors, and takes the adjacency's entries (fillers included) as edges, numbered across rows:
    neighbor indices[:, 2] + indices[:, 0] * count, source indices[:, 1] + indices[:, 0] * last_count.  As upstream, a third
    hop needs the second hop's edge count to be a multiple of fanouts[1].  Upstream passes `defulat_node=` to sample_neighbor
    and so raises TypeError; here the keyword is spelled right."""

    def __init__(self, fanouts, metapath, add_self_loops=True, max_id=-1, sampler=None):
        super().__init__(num_hops=len(metapath), add_self_loops=add_self_loops, sampler=sampler)
        self.fanouts, self.metapath, self.max_id = fanouts, metapath, max_id

    def get_neighbors(self, n_id):
        n_id = n_id.reshape(-1)
        count = self.fanouts[0]
        one, _w, _t = self.sampler.sample_neighbor(n_id, self.metapath[0], count, default_node=self.max_id + 1)
        neighbors = [one.reshape(-1)]
        neighbor_src = [torch.arange(n_id.numel(), device=n_id.device).repeat_interleave(count)]
        cur, last_count = neighbors[0], count
        for hop_edge_types, count in zip(self.metapath[1:], self.fanouts[1:]):
            drawn, (indices, _v, _shape) = self.sampler.sample_neighbor_layerwise_coo(cur.reshape(-1, last_count), hop_edge_types,
                                                                                      count)
            one = drawn.reshape(-1)[indices[:, 2] + indices[:, 0] * count]
            neighbors.append(one)
            neighbor_src.append(indices[:, 1] + indices[:, 0] * last_count)
            cur, last_count = one, count
        return neighbors, neighbor_src
