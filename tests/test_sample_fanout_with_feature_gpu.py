"""GPU: sample_fanout_with_feature -- sample_fanout's hops bit for bit, and the features of every hop's engine ids."""
import numpy as np
import pytest
import torch

import cases
import embedding_reference as er
import graphs
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu


def _dense_fetch(g, eng, dim):
    """get_dense_feature by id in numpy: the node's row, zeros for an absent id"""
    row = {int(x): r for r, x in enumerate(g["ids"])}
    out = np.zeros((len(eng), dim), np.float32)
    for i, x in enumerate(np.asarray(eng).astype(np.uint64)):
        r = row.get(int(x), -1)
        if r >= 0:
            out[i] = g["feat"][r, :dim]
    return out


def _bags_of(sp):
    (idx, vals, shape) = sp
    idx, vals = idx.cpu().numpy(), vals.cpu().numpy()
    return [list(vals[idx[:, 0] == i]) for i in range(shape[0])], idx, shape


@pytest.mark.parametrize("rng", ["minstd", "philox"])
def test_hops_equal_sample_fanout_and_features_follow_engine_ids(rng):
    import euler_b200
    g = er.slot_graph(21, 80, [lambda r, n: r.randint(0, 4, size=n), lambda r, n: r.randint(1, 3, size=n)],
                      [lambda r, k: r.randint(0, 500, size=k), lambda r, k: r.randint(0, 9, size=k)], node0=True, feat_dim=6)
    assert g["ids"][0] == 0                                     # node 0 exists
    euler_b200.set_graph(er.cuda_slot_graph(g), rng=rng, seed=77)
    seeds = g["ids"][np.random.RandomState(3).randint(0, 80, size=400)].astype(np.int64)
    seeds[:3] = [12345, 0, 7]                                    # an absent id, node 0 itself
    ctx = euler_b200.context()
    ctx.seed(77)
    nb, ws, ts, dense, sparse = euler_b200.sample_fanout_with_feature(seeds, [[0], [0]], [4, 3], -1, ["feat0"], [6],
                                                                      ["u64_0", "u64_1"], [500, 9])
    d1 = ctx.draws()
    ctx.seed(77)
    ids2, ws2, ts2 = euler_b200.sample_fanout(seeds, [[0], [0]], [4, 3], -1)
    assert ctx.draws() == d1
    B = len(seeds)
    assert [w.shape for w in ws] == [(B, 4), (B, 4, 3)] and [t.shape for t in ts] == [(B, 4), (B, 4, 3)]
    for l in range(3):
        assert torch.equal(nb[l], ids2[l])
    for l in range(2):
        assert torch.equal(ws[l].reshape(-1), ws2[l]) and torch.equal(ts[l].reshape(-1), ts2[l])
    if rng == "minstd":                                          # the oracle's own draws
        po.seed(77)
        o_ids, o_ws, o_ts = graphs.oracle_graph(g).op_sample_fanout(seeds, [[0], [0]], [4, 3])
        for l in range(2):
            cases.eq(nb[l + 1].cpu().numpy(), o_ids[l], "ids hop %d" % l)
            cases.eq(ws[l].reshape(-1).cpu().numpy(), o_ws[l], "weights hop %d" % l)
    # kept rows (first id not the default fill): engine ids = packed ids, so their features are a fetch by the returned ids;
    # the rows packed away are checked through the engine ids in test_engine_ids_of_rows_packed_away
    for l in range(3):
        ids_l = nb[l].cpu().numpy()
        if l > 0:
            cnt = [4, 3][l - 1]
            rows = ids_l.reshape(-1, cnt)
            kept = rows[:, 0] != -1
        for j, (sp, dflt) in enumerate(zip(sparse[l * 2:(l + 1) * 2], (500, 9))):
            got, idx, shape = _bags_of(sp)
            assert shape[0] == len(ids_l) and shape[1] == max(len(b) for b in got)
            if l == 0:
                assert got == er.bags(g["ids"], g["u64_ptr"], g["u64_val"], 2, ids_l, j, dflt)
                continue
            want = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], 2, ids_l, j, dflt)
            flat_kept = np.repeat(kept, cnt)
            assert [b for b, k in zip(got, flat_kept) if k] == [b for b, k in zip(want, flat_kept) if k]
        dv = dense[l].cpu().numpy()
        if l == 0:
            np.testing.assert_array_equal(dv, _dense_fetch(g, ids_l, 6))
        else:
            flat_kept = np.repeat(kept, cnt)
            np.testing.assert_array_equal(dv[flat_kept], _dense_fetch(g, ids_l[flat_kept], 6))


def test_engine_ids_of_rows_packed_away():
    """through the C entry point: the engine ids it writes, TF-packed, are the ids it returns, and the features are fetched by
    the engine ids (rows whose first draw is node 0 included)"""
    import ctypes as C
    import euler_b200
    from euler_b200 import _lib
    g = er.slot_graph(22, 60, [lambda r, n: r.randint(0, 3, size=n)], [lambda r, k: r.randint(0, 50, size=k)], node0=True, feat_dim=4)
    nbr, gp = g["nbr"], g["grp_ptr"]                              # make node 0 a frequent neighbor, so first draws of it occur
    nbr[np.random.RandomState(6).rand(len(nbr)) < 0.3] = 0
    for r in range(60):
        nbr[gp[r]:gp[r + 1]] = np.sort(nbr[gp[r]:gp[r + 1]])
    euler_b200.set_graph(er.cuda_slot_graph(g), rng="minstd", seed=5)
    seeds = torch.as_tensor(g["ids"].astype(np.int64), device="cuda")
    B, cnt = seeds.numel(), 3
    ids, eng = torch.empty(B * cnt, dtype=torch.int64, device="cuda"), torch.empty(B * cnt, dtype=torch.int64, device="cuda")
    w, t = torch.empty(B * cnt, device="cuda"), torch.empty(B * cnt, dtype=torch.int32, device="cuda")
    dense = [torch.empty((B, 4), device="cuda"), torch.empty((B * cnt, 4), device="cuda")]
    ptrs = [torch.empty(B + 1, dtype=torch.int64, device="cuda"), torch.empty(B * cnt + 1, dtype=torch.int64, device="cuda")]
    tot, mx = np.zeros(2, np.int64), np.zeros(2, np.int64)
    P = lambda xs: (C.c_void_p * len(xs))(*[x.data_ptr() for x in xs])   # noqa: E731
    et, cs = np.zeros(1, np.int32), np.asarray([cnt], np.int32)
    fd, dd, sf = np.zeros(1, np.int32), np.asarray([4], np.int32), np.zeros(1, np.int32)
    ctx = euler_b200.ops._ctx_on_stream()
    _lib.check(_lib.load().eu_sample_fanout_with_feature(ctx._h, seeds.data_ptr(), B, et.ctypes.data, 1, cs.ctypes.data, 1, -1,
                                                         P([ids]), P([w]), P([t]), P([eng]), 1, fd.ctypes.data, dd.ctypes.data,
                                                         P(dense), 1, sf.ctypes.data, P(ptrs), tot.ctypes.data, mx.ctypes.data))
    e = eng.cpu().numpy().reshape(B, cnt)
    packed, kept = er.tf_pack(e, -1)
    assert np.array_equal(ids.cpu().numpy().reshape(B, cnt), packed)
    assert (~kept & (e != 0).any(1)).any(), "no row drew node 0 first"
    np.testing.assert_array_equal(dense[1].cpu().numpy(), _dense_fetch(g, e.reshape(-1), 4))
    for k, (nodes, n) in enumerate(((seeds.cpu().numpy(), B), (e.reshape(-1), B * cnt))):
        bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], 1, nodes, 0, 50)
        assert tot[k] == sum(len(b) for b in bl) and mx[k] == max(len(b) for b in bl)
        assert np.array_equal(np.diff(ptrs[k].cpu().numpy()), [len(b) for b in bl])


def test_reference_case_on_the_tiny_fixture(tiny_dir):
    """neighbor_ops_test.py:203-222 (testSampleFanoutWithFeature): nodes [1, 2, 0, 3], [['0','1'],['0','1']], counts [3, 3],
    dense f3 / f4 of dims [2, 3], sparse f1 / f2 with default 0 -- the draws against the oracle, the features against the
    fixture's own values through get_dense_feature / get_sparse_feature"""
    import euler_b200
    gr = euler_b200.Graph.load(tiny_dir)
    euler_b200.set_graph(gr, rng="minstd", seed=1)
    nodes = np.asarray([1, 2, 0, 3], np.int64)
    euler_b200.seed(31)
    nb, ws, ts, dense, sparse = euler_b200.sample_fanout_with_feature(nodes, [['0', '1'], ['0', '1']], [3, 3], -1, ["f3", "f4"], [2, 3],
                                                                      ["f1", "f2"], [0, 0])
    assert len(nb) == 3 and len(dense) == 6 and len(sparse) == 6
    assert [w.shape for w in ws] == [(4, 3), (4, 3, 3)] and [t.shape for t in ts] == [(4, 3), (4, 3, 3)]
    po.seed(31)
    o_ids, o_ws, o_ts = graphs.oracle_graph(graphs.load_tiny_csr()).op_sample_fanout(nodes, [[0, 1], [0, 1]], [3, 3], -1)
    for l in range(2):
        cases.eq(nb[l + 1].cpu().numpy(), o_ids[l], "ids hop %d" % l)
        cases.eq(ws[l].reshape(-1).cpu().numpy(), o_ws[l], "weights hop %d" % l)
        cases.eq(ts[l].reshape(-1).cpu().numpy(), o_ts[l], "types hop %d" % l)
    # the tiny graph has no node 0 and its draws are never 0, so engine ids equal the packed ids wherever a row was kept;
    # rows without a result are filled and read the default / zero features
    for l in range(3):
        ids_l = nb[l]
        f3, f4 = euler_b200.get_dense_feature(ids_l, ["f3", "f4"], [2, 3])
        assert torch.equal(dense[2 * l], f3) and torch.equal(dense[2 * l + 1], f4)
        for j, nm in enumerate(["f1", "f2"]):
            (idx, vals, shape), = euler_b200.get_sparse_feature(ids_l, [nm], [0])
            si, sv, ss = sparse[2 * l + j]
            assert torch.equal(si, idx) and torch.equal(sv, vals) and tuple(ss) == tuple(shape)
