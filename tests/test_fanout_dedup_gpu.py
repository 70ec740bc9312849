"""Repeated work in the fanout path, bit-exact against the oracle: the fused SAGE aggregation reduces each distinct segment
once and copies it to the rows that repeat it; the sampler draws each eligible seed once and copies its outputs to the
seed's later occurrences."""
import numpy as np
import pytest
import torch

import cases
import graphs
from oracle import pyoracle as po
from test_gpu_parity import _oracle_fanout

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def _segments(g, count, rs, n_rows):
    """[n_rows, count] ids: many exact copies of a few segments, segments that differ only in their last id, the same ids in
    another order, rows whose ids are all absent, and a tail of distinct segments."""
    n = len(g["ids"])
    base = g["ids"][rs.randint(0, n, size=(12, count))].astype(np.int64)
    base[1, :-1] = base[0, :-1]                           # differs from segment 0 only in the last id
    base[2] = base[0, ::-1]                               # segment 0 reversed
    base[3] = np.roll(base[0], 1)                         # segment 0 rotated
    base[4, count // 2:] = -1                             # half default-filled
    base[5] = -1                                          # no neighbor at all
    base[6] = 987654321012                                # an id the graph does not have
    base[7, ::2] = -1
    rows = base[rs.randint(0, len(base), size=n_rows)]
    tail = g["ids"][rs.randint(0, n, size=(n_rows // 4, count))].astype(np.int64)
    out = np.concatenate([rows, tail])
    return out[rs.permutation(len(out))]


# calls of at least this many rows reduce each distinct segment once (kRepeatMinRows); smaller ones reduce every row
REPEAT_MIN_ROWS = 1 << 17


@pytest.mark.parametrize("D,count", [(256, 2), (128, 3), (64, 10), (3, 6), (4, 40)])
def test_fused_aggregate_with_repeated_segments_matches_oracle(D, count):
    import euler_b200
    from euler_b200 import _lib
    n = 3000
    g = graphs.random_graph(seed=131 + D, n=n, T=1, feat_dim=D, id_stride=5 if D == 64 else 1)
    cases.CudaBackend(g, g["ids"])
    og = graphs.oracle_graph(g)
    lib = _lib.load()
    ctx = euler_b200.context()
    rs = np.random.RandomState(D + count)
    # calls of different sizes back to back: each must find the table all-free, whatever the call before it claimed
    for n_rows in (140000, 110000, 37, 120000, 2000):
        seg = _segments(g, count, rs, n_rows)
        rows = len(seg)
        assert (rows >= REPEAT_MIN_ROWS) == (n_rows >= 110000)
        ids = seg.reshape(-1)
        feat = og.op_get_dense_feature(ids, D)
        src = np.repeat(np.arange(rows, dtype=np.int32), count)
        d_ids = torch.from_numpy(ids).cuda()
        for mean, fn in ((True, lib.eu_sage_mean_aggregate), (False, lib.eu_sage_add_aggregate)):
            out = torch.full((rows, D), float("nan"), dtype=torch.float32, device="cuda")
            _lib.check(fn(ctx._h, d_ids.data_ptr(), rows, count, D, out.data_ptr()))
            want = po.scatter_mean(feat, src, rows) if mean else po.scatter_add(feat, src, rows)
            cases.eq(out.cpu().numpy(), want, "%s rows=%d" % ("mean" if mean else "add", rows))


def test_reordered_segments_are_not_merged():
    """The same ids in another order sum in another order: the outputs differ in their last bits and neither may take the
    other's result."""
    import euler_b200
    from euler_b200 import _lib
    D, count, n = 16, 10, 500
    g = graphs.random_graph(seed=5, n=n, T=1, feat_dim=D)
    g["feat"] *= np.float32(1) + np.random.RandomState(6).uniform(0, 1000, size=(n, 1)).astype(np.float32)   # mixed magnitudes
    cases.CudaBackend(g, g["ids"])
    og = graphs.oracle_graph(g)
    rs = np.random.RandomState(7)
    seg = g["ids"][rs.randint(0, n, size=count)].astype(np.int64)
    perms = [seg] + [seg[rs.permutation(count)] for _ in range(15)]
    ids = np.concatenate([perms[i % len(perms)] for i in range(REPEAT_MIN_ROWS + 1000)])
    rows = len(ids) // count
    src = np.repeat(np.arange(rows, dtype=np.int32), count)
    want = po.scatter_add(og.op_get_dense_feature(ids, D), src, rows)
    assert len({want[i].tobytes() for i in range(len(perms))}) > 1, "the permutations must sum to different bits"
    out = torch.empty((rows, D), dtype=torch.float32, device="cuda")
    d_ids = torch.from_numpy(ids).cuda()
    _lib.check(_lib.load().eu_sage_add_aggregate(euler_b200.context()._h, d_ids.data_ptr(), rows, count, D, out.data_ptr()))
    cases.eq(out.cpu().numpy(), want, "permuted segments")


@pytest.mark.parametrize("nb,B,T", [(1, 4000, 1), (6, 700, 3), (12, 350, 2)])
def test_batched_fanout_with_heavily_repeated_seeds(nb, B, T):
    """A low-degree graph: every hop repeats most of its seeds, within a batch and across batches.  Batch b == one
    sample_fanout call on an engine seeded like engine b, over three hops and two consecutive calls.  The last hop has
    more than REPEAT_MIN_ROWS seeds: its duplicates copy their first occurrence's draws; the first two draw again."""
    import euler_b200
    n = 400
    g = graphs.random_graph(seed=300 + nb, n=n, T=T, avg_deg=2, empty_frac=0.3, hub=40, id_stride=7, zero_w_frac=0.1)
    gr = graphs.cuda_graph(g)
    og = graphs.oracle_graph(g)
    euler_b200.set_graph(gr)
    ctx = euler_b200.Context(gr, "minstd", 1)
    seeds_e = [500 + 31 * b for b in range(nb)]
    ctx.set_engines(nb, seeds_e)
    rs = np.random.RandomState(nb)
    pool = g["ids"][rs.randint(0, n, size=20)].astype(np.int64)       # few distinct seeds, shared by every batch
    nodes = pool[rs.randint(0, len(pool), size=(nb, B))]
    nodes[:, ::11] = 77777777
    nodes[:, 1::13] = -1
    nodes[0, :30] = nodes[0, 0]
    # one edge type (T = 1), a strict subset of the types (T = 3) and all of them (T = 2): the three draw modes
    ets = {1: [[0], [0], [0]], 2: [[0, 1], [1, 0], [0, 1]], 3: [[0, 2], [2, 0], [1, 2]]}[T]
    counts = [7, 5, 3]
    states = {}
    for rep in range(2):
        ctx.set_stream(torch.cuda.current_stream().cuda_stream)
        ids, ws, ts = euler_b200.sample_fanout_batched(nodes, ets, counts, -1, ctx=ctx)
        for b in range(nb):
            if rep == 0:
                po.seed(seeds_e[b])
            else:
                po.set_state(states[b])
            o_ids, o_ws, o_ts = _oracle_fanout(og, nodes[b], ets, counts)
            states[b] = po.get_state()
            for l in range(len(counts)):
                cases.eq(ids[l + 1][b].cpu().numpy(), o_ids[l], "batch %d rep %d ids hop %d" % (b, rep, l))
                cases.eq(ws[l][b].cpu().numpy(), o_ws[l], "batch %d rep %d w hop %d" % (b, rep, l))
                cases.eq(ts[l][b].cpu().numpy(), o_ts[l], "batch %d rep %d t hop %d" % (b, rep, l))


def test_fanout_of_a_low_degree_graph_matches_oracle():
    """sample_fanout (one batch, default ctx) on a graph where most hop-1 nodes have one or two neighbors; the third hop
    (614400 seeds) copies its duplicates' draws."""
    import euler_b200
    n = 2000
    g = graphs.random_graph(seed=41, n=n, T=2, avg_deg=1, empty_frac=0.2, hub=200)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=99)
    og = graphs.oracle_graph(g)
    seeds = g["ids"][np.random.RandomState(1).randint(0, 60, size=4096)].astype(np.int64)
    ets = [[0, 1], [1, 0], [0, 1]]
    ids, ws, ts = euler_b200.sample_fanout(seeds, ets, [15, 10, 4])
    po.seed(99)
    o_ids, o_ws, o_ts = og.op_sample_fanout(seeds, ets, [15, 10, 4])
    for l in range(3):
        cases.eq(ids[l + 1].cpu().numpy(), o_ids[l], "ids hop %d" % l)
        cases.eq(ws[l].cpu().numpy(), o_ws[l], "weights hop %d" % l)
        cases.eq(ts[l].cpu().numpy(), o_ts[l], "types hop %d" % l)
