"""CPU: the layer / hop plan of GCNEncoder.infer (encoders.infer_plan), its table computation (_infer_layers, fused=False)
on CPU tensors in float64 over a hand-built whole-graph adjacency against forward's composition (_layers over
get_multi_hop_neighbor's hops) on the same tiny graph, and argument errors."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200.encoders import GCNEncoder, GenieEncoder, infer_plan

# a tiny graph of 13 nodes (id = row) with two edge types; id 20 is listed but is not a node.  Row 4 lists nothing.
N_NODES, ABSENT = 13, 20
LISTS = {0: {v: [(3 * v + k) % 13 for k in range(v % 4)] + ([(3 * v) % 13] if v % 4 == 3 else []) for v in range(13)},
         1: {v: [(5 * v + 1) % 13, ABSENT] if v % 3 == 0 else [(v + 2) % 13] for v in range(13)}}
LISTS[0][4] = LISTS[1][4] = []


def _listing(v, types):
    return [x for t in types for x in (LISTS[t].get(v, []) if v < N_NODES else [])]


def _column(v):
    return v if v < N_NODES else N_NODES      # the absent id is the one row after the nodes


def _whole(types, rows):
    """graph_adjacency's (indptr, cols) over `rows` (ids = rows; the absent id's row lists nothing), listing order"""
    lists = [[_column(x) for x in _listing(v, types)] for v in rows]
    indptr = torch.as_tensor(np.r_[0, np.cumsum([len(r) for r in lists])], dtype=torch.int64)
    return indptr, torch.as_tensor([c for r in lists for c in r], dtype=torch.int64)


def _multi_hop(nodes, metapath):
    """get_multi_hop_neighbor's hops: next nodes in first-occurrence order, each row's entries ordered by column"""
    nodes_list, adjs = [list(nodes)], []
    for types in metapath:
        listing = [_listing(v, types) for v in nodes_list[-1]]
        uniq = list(dict.fromkeys(x for row in listing for x in row))
        pos = {v: i for i, v in enumerate(uniq)}
        rows = [sorted(pos[x] for x in row) for row in listing]
        indptr = torch.as_tensor(np.r_[0, np.cumsum([len(r) for r in rows])], dtype=torch.int64)
        adjs.append((indptr, torch.as_tensor([c for r in rows for c in r], dtype=torch.int64)))
        nodes_list.append(uniq)
    return nodes_list, adjs


def test_plan_shares_the_tables_of_equal_windows():
    assert infer_plan([[0]]) == []
    assert infer_plan([[0], [0]]) == [{((0,),): [0, 1]}]
    assert infer_plan([[0], [1]]) == [{((0,),): [0], ((1,),): [1]}]
    assert infer_plan([[0, 1], [1]]) == [{((0, 1),): [0], ((1,),): [1]}]
    assert infer_plan([[1, 0], [0, 1]]) == [{((1, 0),): [0], ((0, 1),): [1]}]   # the listing order is part of the window
    assert infer_plan([[0]] * 3) == [{((0,),): [0, 1, 2]}, {((0,), (0,)): [0, 1]}]
    assert infer_plan([[0], [1], [0]]) == [{((0,),): [0, 2], ((1,),): [1]}, {((0,), (1,)): [0], ((1,), (0,)): [1]}]
    assert infer_plan(np.array([[0], [0]])) == [{((0,),): [0, 1]}]


KW = dict(feature_idx='f1', feature_dim=6, head_num=2, fused=False)


@pytest.mark.parametrize("use_residual", (False, True))
@pytest.mark.parametrize("metapath", ([[0]], [[0], [0]], [[0], [1]], [[0, 1], [1]], [[1], [0], [1]]))
@pytest.mark.parametrize("aggregator", ("gcn", "mean", "attention"))
def test_infer_layers_equal_forwards_composition(aggregator, metapath, use_residual):
    torch.manual_seed(0)
    enc = GCNEncoder(metapath, 8, aggregator, use_residual=use_residual, **KW).double().requires_grad_(False)
    width = enc.dims[0]
    table = torch.randn(N_NODES + 1, width, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    ids = [3, 4, ABSENT, 9, 3, 0, 12]
    N = N_NODES + 1
    adjs = [_whole(types, range(N)) for types in metapath]
    final = _whole(metapath[0], ids)
    self_cols = torch.as_tensor([_column(v) for v in ids])
    seen = []
    got = enc._infer_layers(table, adjs, final, self_cols, 3, lambda layer, rows: seen.append(rows))
    nodes, hops = _multi_hop(ids, metapath)
    hidden = [table[torch.as_tensor([_column(v) for v in hop])] for hop in nodes]
    want_seen = [hidden[0]]
    want = enc._layers(hidden, hops, lambda layer, h: want_seen.append(h))
    assert got.dtype == torch.float64 and got.shape == want.shape == (len(ids), enc.dims[-1])
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-12, atol=1e-12)
    assert len(seen) == len(want_seen) == len(metapath) + 1
    for a, b in zip(seen, want_seen):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-12, atol=1e-12)
    # every node in row order (self_cols None): the first N_NODES rows of the whole adjacency of hop 0
    every = enc._infer_layers(table, adjs, (adjs[0][0][:N_NODES + 1], adjs[0][1]), None, 5)
    np.testing.assert_allclose(every[torch.as_tensor([3, 0, 12])].numpy(), want[[0, 5, 6]].numpy(), rtol=1e-12, atol=1e-12)


def test_genie_steps_are_forwards():
    torch.manual_seed(0)
    enc = GenieEncoder([[0], [1]], 8, **KW).double()
    h_t = [torch.randn(5, d, dtype=torch.float64) for d in enc.dims]
    with torch.no_grad():
        h_t = [fc(h) for fc, h in zip(enc.depth_fc, h_t)]
        out = enc._steps(h_t)
        first = enc.lstm_cell(h_t[0], (torch.zeros_like(out), torch.zeros_like(out)))[0]
    assert out.shape == (5, 8)
    np.testing.assert_allclose(out.numpy(), first.numpy())


def test_argument_errors():
    enc = GCNEncoder([[0]], 8, 'gcn', **KW)
    for chunk_rows in (0, -4):
        with pytest.raises(ValueError, match="chunk_rows"):
            enc.infer(torch.as_tensor([1, 2]), chunk_rows=chunk_rows)
