"""Rows of the fanout sampler that cannot draw, bit-exact against the oracle: k_prepare writes their default entries with the
warp's lanes striding over the warp's output slots, and enters their id 0 into the next hop's table once per block, at the
block's smallest index."""
import numpy as np
import pytest
import torch

import cases
import graphs
from oracle import pyoracle as po
from test_gpu_parity import _oracle_fanout

pytestmark = pytest.mark.gpu

# hops of at least this many seeds copy their duplicates' draws (kRepeatMinRows); smaller ones draw them again
REPEAT_MIN_ROWS = 1 << 17


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def _give_edges(g, rows, k, seed):
    """g with `k` edges (to random nodes, positive weights) in every edge group of each row of `rows` that has none there."""
    n, T = len(g["ids"]), g["T"]
    rs = np.random.RandomState(seed)
    want = np.zeros(n, bool)
    want[rows] = True
    gp = g["grp_ptr"]
    nbr, w, ptr = [], [], [0]
    for q in range(n * T):
        b, e = gp[q], gp[q + 1]
        if e == b and want[q // T]:
            nbr.append(np.sort(g["ids"][rs.randint(0, n, size=k)]))
            w.append((1 + rs.randint(0, 100, size=k)).astype(np.float32) / np.float32(10))
        else:
            nbr.append(g["nbr"][b:e])
            w.append(g["w"][b:e])
        ptr.append(ptr[-1] + len(nbr[-1]))
    g = dict(g, grp_ptr=np.asarray(ptr, np.int64), nbr=np.concatenate(nbr).astype(np.uint64),
             w=np.concatenate(w).astype(np.float32))
    g["cum_w"], g["grp_cum"] = po.build_cum(g["grp_ptr"], g["w"], n, T)
    return g


def _check_fanout(ids, ws, ts, o, counts, what):
    o_ids, o_ws, o_ts = o
    for l in range(len(counts)):
        cases.eq(ids[l + 1].cpu().numpy(), o_ids[l], "%s ids hop %d" % (what, l))
        cases.eq(ws[l].cpu().numpy(), o_ws[l], "%s w hop %d" % (what, l))
        cases.eq(ts[l].cpu().numpy(), o_ts[l], "%s t hop %d" % (what, l))


@pytest.mark.parametrize("kind", ["none_draw", "all_draw"])
def test_hops_where_every_row_or_no_row_cannot_draw(kind):
    """Every seed absent (no row of any hop draws: all default entries, id 0 fills the chained frontier), or every node with
    edges (every row of every hop draws: no default entry).  The last hop has more than REPEAT_MIN_ROWS seeds."""
    import euler_b200
    n = 3000
    g = graphs.random_graph(seed=17, n=n, T=1, avg_deg=4, empty_frac=0.0 if kind == "all_draw" else 0.3)
    if kind == "all_draw":
        g = _give_edges(g, np.arange(n), 2, seed=18)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=5)
    og = graphs.oracle_graph(g)
    rs = np.random.RandomState(2)
    if kind == "none_draw":
        seeds = np.full(2000, 123456789012, dtype=np.int64)
        seeds[::3] = -1
    else:
        seeds = g["ids"][rs.randint(0, n, size=2000)].astype(np.int64)
    ets, counts = [[0], [0], [0]], [10, 8, 2]
    for rep in range(2):   # back to back: the tables and counters must be left clean
        ids, ws, ts = euler_b200.sample_fanout(seeds, ets, counts, -1)
        if rep == 0:
            po.seed(5)
        o = og.op_sample_fanout(seeds, ets, counts, -1)
        _check_fanout(ids, ws, ts, o, counts, "%s rep %d" % (kind, rep))
        for l in range(len(counts)):
            out = ids[l + 1].cpu().numpy()
            assert (out == -1).all() if kind == "none_draw" else (out != -1).all(), "hop %d" % l


@pytest.mark.parametrize("nb,node0", [(1, False), (3, False), (1, True), (3, True)])
def test_chained_fanout_with_many_placeholder_rows(nb, node0):
    """Most rows of every hop cannot draw: each enters `count` zeros into the next hop's table, from many blocks of every
    batch.  With node0, id 0 is a node with edges of every type: the next hop's placeholder rows draw, and the smallest index
    of id 0 decides which of them is the first occurrence -- its place in the serial draw order, and in the last hop
    (REPEAT_MIN_ROWS seeds or more) the row whose draws the others copy.  Batches are independent engines and tables."""
    import euler_b200
    n = 1500
    g = graphs.random_graph(seed=23 + nb, n=n, T=2, avg_deg=1, empty_frac=0.7, hub=30, id_base=0 if node0 else 1)
    if node0:
        g = _give_edges(g, [0], 3, seed=29)
        assert g["ids"][0] == 0 and (np.diff(g["grp_ptr"][:3]) > 0).all()
    gr = graphs.cuda_graph(g)
    og = graphs.oracle_graph(g)
    euler_b200.set_graph(gr)
    ctx = euler_b200.Context(gr, "minstd", 1)
    seeds_e = [900 + 13 * b for b in range(nb)]
    ctx.set_engines(nb, seeds_e)
    rs = np.random.RandomState(nb)
    nodes = g["ids"][rs.randint(0, n, size=(nb, 3000))].astype(np.int64)
    nodes[:, 5::7] = 0           # placeholders among the seeds (node 0 itself when node0)
    nodes[:, 300:700] = 55555555
    ets, counts = [[0, 1], [1, 0], [0, 1]], [9, 6, 4]
    assert nb * 3000 * 9 * 6 >= REPEAT_MIN_ROWS
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    ids, ws, ts = euler_b200.sample_fanout_batched(nodes, ets, counts, -1, ctx=ctx)
    for b in range(nb):
        po.seed(seeds_e[b])
        o_ids, o_ws, o_ts = _oracle_fanout(og, nodes[b], ets, counts)
        for l in range(len(counts)):
            cases.eq(ids[l + 1][b].cpu().numpy(), o_ids[l], "batch %d ids hop %d" % (b, l))
            cases.eq(ws[l][b].cpu().numpy(), o_ws[l], "batch %d w hop %d" % (b, l))
            cases.eq(ts[l][b].cpu().numpy(), o_ts[l], "batch %d t hop %d" % (b, l))
        # rows that cannot draw are spread over most 256-row blocks of the two chaining hops
        for l in range(2):
            cannot = o_ids[l].reshape(-1, counts[l])[:, 0] == -1
            assert cannot.mean() > 0.1 and cannot[:len(cannot) // 256 * 256].reshape(-1, 256).any(1).mean() > 0.5, "hop %d" % l
