"""Every device hash table on keys built to collide (tests/collision_cases.py): id chains that wrap past the last slot, absent
ids whose search walks the whole chain, a repeated id far down it, dedup regions that wrap inside themselves, ids 0 and
2^64-1, SAGE segments that share a 32-bit tag and a home slot, and edges whose hashes share one home.  Each op is compared
with a plain reference: a dict for lookups and first occurrence, the oracle for exact-mode draws and f32-order reductions,
float64 as a bound.  tests/test_hash_collisions_cpu.py counts the collisions each case really contains."""
import ctypes as C

import numpy as np
import pytest
import torch

import bf16_reference as bf
import cases
import collision_cases as cc
import graphs
import mp_ops_reference as ref
from oracle import pyoracle as po
from test_full_dataflow_cpu import CpuFullSampler
from test_gpu_parity import _oracle_fanout

pytestmark = pytest.mark.gpu
INT32_MIN = np.iinfo(np.int32).min
ETS = [[0, 1], [1, 0]]


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def _rows(q):
    """the row of each query id (a dict: the later row of a repeated id), -1 when absent"""
    m = cc.row_of_id()
    return np.asarray([m.get(int(k), -1) for k in np.asarray(q, np.int64).view(np.uint64)], np.int64)


# ------------------------------------------------------------------------------------------------ node id table
def test_node_table_lookups():
    import euler_b200 as eb
    g = cc.collision_graph(16)
    eb.set_graph(graphs.cuda_graph(g), rng="minstd", seed=11)
    og = graphs.oracle_graph(g)
    q = cc.node_queries()
    rows = _rows(q)
    assert rows[q == cc.cluster()[cc.DUP_OF]].min() == len(g["ids"]) - 1, "the repeated id is its later row"
    assert (rows[q == 0] >= 0).all() and (rows[q == -1] < 0).all()
    d_q = torch.from_numpy(q).cuda()
    cases.eq(eb.get_node_type(d_q).cpu().numpy(), np.where(rows >= 0, g["node_type"][rows], INT32_MIN), "node types")
    cases.eq(eb.get_dense_feature(d_q, [0], [16])[0].cpu().numpy(), ref.dense_feature(g["feat"], [16], rows, 0, 16),
             "dense features")
    indptr, nb, w, t = (x.cpu().numpy() for x in eb.get_full_neighbor(d_q, [0, 1]))
    deg = np.diff(g["grp_ptr"]).reshape(-1, 2).sum(1)
    cases.eq(np.diff(indptr), np.where(rows >= 0, deg[rows], 0), "full neighbor lengths")
    lens, o_nb, o_w, o_t = og.get_full_neighbor(q.view(np.uint64), [0, 1])
    cases.eq(np.diff(indptr), lens.astype(np.int64), "full neighbor lengths vs oracle")
    cases.eq(nb, o_nb.astype(np.int64), "full neighbor ids")
    cases.eq(w, o_w, "full neighbor weights")
    cases.eq(t, o_t, "full neighbor types")
    got = [x.cpu().numpy() for x in eb.sample_neighbor(d_q, [0, 1], 7)]
    po.seed(11)
    for nm, a, b in zip(("ids", "weights", "types"), got, og.op_sample_neighbor(q, [0, 1], 7)):
        cases.eq(a, b, "sample_neighbor " + nm)


# ------------------------------------------------------------------------------------------------ fanout dedup tables
@pytest.mark.parametrize("B,counts", [(3000, [5, 3]), (140_000, [3, 2])])
def test_fanout_on_cluster_seeds_matches_oracle(B, counts):
    """seeds and most neighbours from the cluster; hops of 3000 / 15000 seeds, and of 140000 / 420000 (the duplicate-list
    path)"""
    import euler_b200 as eb
    g = cc.collision_graph()
    eb.set_graph(graphs.cuda_graph(g), rng="minstd", seed=21)
    og = graphs.oracle_graph(g)
    seeds = cc.fanout_seeds(B, np.random.RandomState(B))
    ids, ws, ts = eb.sample_fanout(seeds, ETS, counts)
    po.seed(21)
    o_ids, o_ws, o_ts = og.op_sample_fanout(seeds, ETS, counts)
    for l in range(len(counts)):
        cases.eq(ids[l + 1].cpu().numpy(), o_ids[l], "ids hop %d" % l)
        cases.eq(ws[l].cpu().numpy(), o_ws[l], "weights hop %d" % l)
        cases.eq(ts[l].cpu().numpy(), o_ts[l], "types hop %d" % l)


@pytest.mark.parametrize("nb,B", [(4, 3000), (3, 50_000)])
def test_batched_fanout_regions_wrap_inside_themselves(nb, B):
    """every batch's seeds home at the last slot of its own region: each region's chain wraps to the region's slot 0 and
    must not spill into the next batch's region (the second hop of (3, 50000) has 200000 seeds per batch)"""
    import euler_b200 as eb
    g = cc.collision_graph()
    gr = graphs.cuda_graph(g)
    og = graphs.oracle_graph(g)
    eb.set_graph(gr)
    ctx = eb.Context(gr, "minstd", 1)
    seeds_e = [700 + 13 * b for b in range(nb)]
    ctx.set_engines(nb, seeds_e)
    rs = np.random.RandomState(nb)
    nodes = np.stack([cc.fanout_seeds(B, rs) for _ in range(nb)])
    counts = [4, 3]
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    ids, ws, ts = eb.sample_fanout_batched(nodes, ETS, counts, -1, ctx=ctx)
    for b in range(nb):
        po.seed(seeds_e[b])
        o_ids, o_ws, o_ts = _oracle_fanout(og, nodes[b], ETS, counts)
        for l in range(len(counts)):
            cases.eq(ids[l + 1][b].cpu().numpy(), o_ids[l], "batch %d ids hop %d" % (b, l))
            cases.eq(ws[l][b].cpu().numpy(), o_ws[l], "batch %d weights hop %d" % (b, l))
            cases.eq(ts[l][b].cpu().numpy(), o_ts[l], "batch %d types hop %d" % (b, l))


@pytest.mark.parametrize("B", (3000, 140_000))
def test_philox_fanout_gives_repeated_seeds_one_row(B):
    import euler_b200 as eb
    g = cc.collision_graph()
    eb.set_graph(graphs.cuda_graph(g), rng="philox", seed=5)
    seeds = cc.fanout_seeds(B, np.random.RandomState(B + 1))
    counts = [4, 3]
    ids, ws, ts = eb.sample_fanout(seeds, ETS, counts)
    frontier = seeds
    for l, c in enumerate(counts):
        # an output row of -1 may stand for draws whose first is node 0 (the next hop samples those): hop 0 keeps every row,
        # later hops the rows whose seed is an id
        keep = np.flatnonzero(frontier != -1) if l else np.arange(len(frontier))
        _, first, inv = np.unique(frontier[keep], return_index=True, return_inverse=True)
        for nm, x in (("ids", ids[l + 1]), ("weights", ws[l]), ("types", ts[l])):
            x = x.cpu().numpy().reshape(len(frontier), c)[keep]
            cases.eq(x, x[first[inv]], "philox hop %d %s of repeated seeds" % (l, nm))
        frontier = ids[l + 1].cpu().numpy()
    absent = _rows(seeds) < 0
    assert (ids[1].cpu().numpy().reshape(B, -1)[absent] == -1).all()


# ------------------------------------------------------------------------------------------------ first-occurrence tables
def _unique_first(x):
    u, first = np.unique(x, return_index=True)
    order = np.argsort(first, kind="stable")
    pos = np.empty(len(u), np.int64)
    pos[order] = np.arange(len(u))
    return u[order], pos[np.searchsorted(u, x)].astype(np.int32)


def test_unique_on_cluster_runs():
    import euler_b200 as eb
    eb.set_graph(graphs.cuda_graph(cc.collision_graph()))
    x = cc.unique_input(np.random.RandomState(3))
    for n in (40, 300, 5000, len(x)):
        vals, inv = eb.unique(torch.from_numpy(x[:n]).cuda())
        want_v, want_i = _unique_first(x[:n])
        cases.eq(vals.cpu().numpy(), want_v, "unique values n=%d" % n)
        cases.eq(inv.cpu().numpy(), want_i, "unique inverse n=%d" % n)


@pytest.mark.parametrize("n", (31, 2000, 60_000))
def test_full_hop_and_multi_hop_on_cluster(n):
    import euler_b200 as eb
    g = cc.collision_graph()
    eb.set_graph(graphs.cuda_graph(g), seed=1)
    cpu = CpuFullSampler(g)
    nodes = cc.fanout_seeds(n, np.random.RandomState(n))
    d_nodes = torch.from_numpy(nodes).cuda()
    for et in ([0, 1], [1]):
        for self_loops in (True, False):
            got = eb.full_neighbor_hop(d_nodes, et, self_loops, True)
            want = cpu.full_neighbor_hop(torch.from_numpy(nodes), et, self_loops, True)
            for nm, a, b in zip(("n_id", "res_n_id", "edge_index", "types"), got, want):
                cases.eq(a.cpu().numpy(), b.numpy(), "%s n=%d et=%s self_loops=%s" % (nm, n, et, self_loops))
    got = eb.get_multi_hop_neighbor(nodes, [[0, 1], [1, 0]])
    want = eb.get_multi_hop_neighbor(torch.from_numpy(nodes), [[0, 1], [1, 0]], sampler=cpu)
    for a, b in zip(got[0], want[0]):
        cases.eq(a.cpu().numpy(), b.numpy(), "multi-hop nodes n=%d" % n)
    for a, b in zip(got[1], want[1]):
        for x, y in zip(a, b):
            cases.eq(x.cpu().numpy(), y.numpy(), "multi-hop adjacency n=%d" % n)


# ------------------------------------------------------------------------------------------------ SAGE segment table
def _sage_graph(D, feat_dtype="float32", place="device"):
    """the collision graph with D-wide features stored as feat_dtype at place, and the f32 table those bits widen to"""
    import euler_b200 as eb
    g = cc.collision_graph(D)
    feat = bf.rounded(g["feat"]) if feat_dtype == "bfloat16" else g["feat"]
    gr = eb.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], cum_w=g["cum_w"], grp_cum=g["grp_cum"],
                           node_type=g["node_type"], node_w=g["node_w"], n_node_types=g["n_node_types"], feat=g["feat"],
                           feat_dtype=feat_dtype, feat_place=place, feat_cache_rows=len(g["ids"]) // 3 if place == "host" else 0)
    eb.set_graph(gr)
    return gr, dict(g, feat=feat)


def _fused(ids, rows, count, D, mean, out_dtype):
    """eu_sage_{mean,add}_aggregate_out_dtype over device ids [rows * count]"""
    from euler_b200 import _lib, ops
    out = torch.full((rows, D), float("nan"), dtype=out_dtype, device="cuda")
    name = "eu_sage_%s_aggregate_out_dtype" % ("mean" if mean else "add")
    _lib.check(getattr(_lib.load(), name)(ops._ctx_on_stream()._h, ids.data_ptr(), rows, count, D, _lib.TORCH_DTYPES[out_dtype],
                                          out.data_ptr()))
    return out


def _bits(out):
    return out.view(torch.int16).cpu().numpy().view(np.uint16) if out.dtype == torch.bfloat16 else out.cpu().numpy()


def _pool_reference(g, pool, count, D, mean):
    """the pool's outputs in the reference's f32 order: get_dense_feature then scatter_mean / scatter_add"""
    og = graphs.oracle_graph(g)
    x = og.op_get_dense_feature(pool.reshape(-1), D)
    src = np.repeat(np.arange(len(pool), dtype=np.int32), count)
    want = (po.scatter_mean if mean else po.scatter_add)(x, src, len(pool))
    # float64 bound: a sum of `count` f32 terms in any order, then one division
    x64 = x.astype(np.float64).reshape(len(pool), count, D)
    s64 = x64.sum(1) / ((count + 1e-7) if mean else 1.0)
    tol = (count + 2) * 2.0 ** -24 * np.abs(x64).sum(1) / ((count + 1e-7) if mean else 1.0) + 2.0 ** -149
    assert (np.abs(want - s64) <= tol).all(), "f32 reference vs float64"
    return want


@pytest.mark.parametrize("place", ("device", "host"))
@pytest.mark.parametrize("feat_dtype", ("float32", "bfloat16"))
@pytest.mark.parametrize("D", (128, 256, 64, 3))
def test_sage_twins_are_not_merged(D, feat_dtype, place):
    """twin segments -- same tag, same home slot, different last id -- in calls past 2^17 rows, bit-equal to the reference and
    to the single-pass call over the distinct segments, for f32 and bf16 outputs"""
    _, g = _sage_graph(D, feat_dtype, place)
    for count in cc.SAGE_COUNTS:
        pool, groups, _ = cc.sage_pool(count)
        idx = cc.sage_rows(count, cc.SAGE_ROWS, count)
        d_big = torch.from_numpy(pool[idx].reshape(-1)).cuda()
        d_pool = torch.from_numpy(pool.reshape(-1)).cuda()
        for mean in (True, False):
            want = _pool_reference(g, pool, count, D, mean)
            for grp in groups:   # twins differ: a merge would show
                assert len({want[i].tobytes() for i in grp}) == len(grp), "twins with equal outputs"
            for out_dtype in (torch.float32, torch.bfloat16):
                what = "D=%d %s %s count=%d %s out %s" % (D, feat_dtype, place, count, "mean" if mean else "add", out_dtype)
                w = bf.round_bits(want) if out_dtype == torch.bfloat16 else want
                single = _bits(_fused(d_pool, len(pool), count, D, mean, out_dtype))
                cases.eq(single, w, what + " single pass")
                cases.eq(_bits(_fused(d_big, len(idx), count, D, mean, out_dtype)), single[idx], what + " segment table")


def test_sage_table_is_clean_between_calls_and_in_a_cuda_graph():
    """a call of 2^18 + 777 rows, then one of 2^17 + 555 rows whose segments home in slots the first claimed, then the first
    again; then one call captured in a CUDA graph and replayed twice"""
    import euler_b200 as eb
    D, count = 64, 10
    _, g = _sage_graph(D)
    pool, _, _ = cc.sage_pool(count)
    want = _pool_reference(g, pool, count, D, True)
    for k, rows in enumerate((cc.SAGE_ROWS_BIG, cc.SAGE_ROWS_SMALL, cc.SAGE_ROWS_BIG)):
        idx = cc.sage_rows(count, rows, 10 + k)
        got = eb.sage_mean_aggregate(torch.from_numpy(pool[idx].reshape(-1)).cuda(), count, D)
        cases.eq(got.cpu().numpy(), want[idx], "call %d rows=%d" % (k, rows))
    idx = cc.sage_rows(count, cc.SAGE_ROWS, 20)
    d_ids = torch.from_numpy(pool[idx].reshape(-1)).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eb.sage_mean_aggregate(d_ids, count, D)
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = eb.sage_mean_aggregate(d_ids, count, D)
    torch.cuda.current_stream().wait_stream(s)
    for rep in range(2):
        out.fill_(float("nan"))
        cg.replay()
        torch.cuda.synchronize()
        cases.eq(out.cpu().numpy(), want[idx], "replay %d" % rep)


# ------------------------------------------------------------------------------------------------ edge table
def _attach_edges(gr, src, dst, typ, rs):
    """eu_graph_set_edges with a dense slot, a uint64 slot and a binary slot whose values name the edge's row"""
    from euler_b200 import _lib
    E = len(src)
    dense = np.stack([np.arange(E), -np.arange(E), np.arange(E) * 0.5], 1).astype(np.float32)
    ulen, blen = rs.randint(0, 4, size=E), rs.randint(0, 4, size=E)
    u_ptr = np.r_[0, np.cumsum(ulen)].astype(np.int64)
    u_val = (np.repeat(np.arange(E), ulen) * 10 + rs.randint(0, 10, size=int(u_ptr[-1]))).astype(np.uint64)
    b_ptr = np.r_[0, np.cumsum(blen)].astype(np.int64)
    b_val = rs.randint(0, 256, size=max(int(b_ptr[-1]), 1)).astype(np.uint8)
    keep = [np.ascontiguousarray(a) for a in (src.view(np.uint64), dst.view(np.uint64), typ, dense, np.asarray([3], np.int32),
                                              u_ptr, u_val, b_ptr, b_val)]
    d = _lib.EdgeDesc()
    d.n_edges = E
    d.src, d.dst, d.type = (a.ctypes.data for a in keep[:3])
    d.feat_dim, d.feat, d.n_feat_slots, d.feat_slot_dims = 3, keep[3].ctypes.data, 1, keep[4].ctypes.data
    d.n_u64_slots, d.u64_ptr, d.u64_val = 1, keep[5].ctypes.data, keep[6].ctypes.data
    d.n_bin_slots, d.bin_ptr, d.bin_val = 1, keep[7].ctypes.data, keep[8].ctypes.data
    _lib.check(_lib.load().eu_graph_set_edges(gr._h, C.byref(d)))
    return dense, (u_ptr, u_val), (b_ptr, b_val)


def test_edge_table_lookups():
    import euler_b200 as eb
    gr = graphs.cuda_graph(cc.collision_graph())
    src, dst, typ, absent = cc.edge_case()
    E = len(src)
    rs = np.random.RandomState(4)
    dense, (u_ptr, u_val), (b_ptr, b_val) = _attach_edges(gr, src, dst, typ, rs)
    eb.set_graph(gr)
    row = {}
    for r in range(E):
        row.setdefault((int(src[r]), int(dst[r]), int(typ[r])), r)   # the first row of a repeated triple is the edge
    present = np.stack([src, dst, typ.astype(np.int64)], 1)
    cl = present[1000:]
    q = np.concatenate([cl, absent, present[rs.randint(0, 1000, size=200)],
                        cl[:40] + [0, 0, 5], cl[40:80] * [1, 1, 0] + [0, 0, -1], cl[80:120] + [0, 0, 1 << 32],
                        cl[120:140] * [1, 1, 0] + [0, 0, INT32_MIN - 1]])
    rows = np.asarray([row.get((int(a), int(b), int(t)), -1) for a, b, t in q], np.int64)
    assert rows[len(cl) - 1] == 1000 and (rows[len(cl):len(cl) + len(absent)] < 0).all()
    assert (rows[-140:] < 0).all()
    d_q = torch.from_numpy(q).cuda()
    (got,) = eb.get_edge_dense_feature(d_q, ["feat0"], [4])
    cases.eq(got.cpu().numpy(), ref.dense_feature(dense, [3], rows, 0, 4), "edge dense feature")
    dv = -7
    ((_, vals, _),) = eb.get_edge_sparse_feature(d_q, ["u64_0"], [dv])
    want = np.concatenate([u_val[u_ptr[r]:u_ptr[r + 1]].astype(np.int64) if r >= 0 and u_ptr[r + 1] > u_ptr[r] else [dv]
                           for r in rows]).astype(np.int64)
    cases.eq(vals.cpu().numpy(), want, "edge sparse feature")
    (got,) = eb.get_edge_binary_feature(d_q, ["bin_0"])
    assert got == [bytes(b_val[b_ptr[r]:b_ptr[r + 1]]) if r >= 0 else b"" for r in rows], "edge binary feature"
