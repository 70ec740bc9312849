"""GPU: dense node features stored as bfloat16.  Every graph is built twice: with feat_dtype='bfloat16', and as an f32 graph
of the bf16 graph's own table widened to f32 (export()).  Every op that reads dense node features must give the same bits on
both; the stored table must be the round-to-nearest-even restatement of tests/bf16_reference.py."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import bf16_reference as br
import graphs

pytestmark = pytest.mark.gpu

SLOTS = (1, 3, 4, 16, 128, 200, 256)          # offsets 0, 1, 4, 8, 24, 152, 352: multiples of 4 and not
WIDTHS = (3, 64, 128, 200, 256, 516, 1024)     # one-slot graphs for the fused SAGE reduction's paths
N = 2000
ABSENT = 10 ** 9


def _features(rng, n, d, specials=True):
    f = (rng.standard_normal((n, d)) * 3).astype(np.float32)
    if specials:
        sp = br.special_values()
        mask = rng.rand(n, d) < 0.02
        f[mask] = sp[rng.randint(0, len(sp), size=int(mask.sum()))]
    return f


def _pair(build):
    """(the bf16 graph, the f32 graph of its exported table); build(feat_dtype, feat or None for the original features)"""
    gb = build("bfloat16", None)
    return gb, build("float32", gb.export()["feat"])


def _csr(g, slots, feat):
    import euler_b200

    def build(dt, f):
        return euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                         node_w=g["node_w"], cum_w=g["cum_w"], feat=feat if f is None else f,
                                         feat_slot_dims=list(slots), feat_dtype=dt)
    return build


@pytest.fixture(scope="module")
def env():
    rng = np.random.RandomState(11)
    g = graphs.random_graph(seed=11, n=N, T=1, avg_deg=6)
    feat = _features(rng, N, sum(SLOTS))
    single = {}
    for d in WIDTHS:
        f = _features(rng, N, d)
        single[d] = (f, _pair(_csr(g, (d,), f)))
    ties = (rng.randint(-4, 5, size=(N, 146)) / 4).astype(np.float32)     # quarters: many ties, all exact in bf16
    ties[rng.rand(*ties.shape) < 0.1] = np.float32(-0.0)
    ties[rng.rand(*ties.shape) < 0.01] = np.float32("nan")
    ties[::7] = np.float32(0.5)
    finite = _features(rng, N, 3 + 16 + 128, specials=False)
    finite[:, :3] = rng.randint(0, 2, size=(N, 3))                         # 0 / 1 labels
    return dict(g=g, feat=feat, multi=_pair(_csr(g, SLOTS, feat)), single=single, ties=_pair(_csr(g, (16, 130), ties)),
                train=_pair(_csr(g, (3, 16, 128), finite)))


def _use(graph, seed=1):
    import euler_b200
    euler_b200.set_graph(graph, rng="minstd", seed=seed)


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _both(pair, fn):
    """fn() on the bf16 graph, then on the f32 graph; the two results' bits must be equal"""
    outs = []
    for graph in pair:
        _use(graph)
        outs.append(fn())
    a, b = outs
    for x, y in zip(a if isinstance(a, (list, tuple)) else [a], b if isinstance(b, (list, tuple)) else [b]):
        if x is None:
            assert y is None
            continue
        assert x.dtype == y.dtype and x.shape == y.shape
        assert torch.equal(_bits(x), _bits(y))
    return a


def _ids(rng, M, absent=0.1):
    ids = rng.randint(1, N + 1, size=M).astype(np.int64)
    ids[rng.rand(M) < absent] = ABSENT
    ids[rng.rand(M) < absent / 2] = -1
    return ids


# ---------------------------------------------------------------------------- the stored table
def test_stored_table_is_the_device_rounding(env):
    gb, gf = env["multi"]
    assert (gb.feat_dtype, gf.feat_dtype) == ("bfloat16", "float32")
    got = gb.export()["feat"]
    want = br.rounded(env["feat"])
    nan = np.isnan(env["feat"])
    assert nan.any() and np.isinf(env["feat"]).any()
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan])
    assert np.array_equal(gf.export()["feat"].view(np.uint32), got.view(np.uint32))


def test_every_special_value_rounds_as_restated():
    import euler_b200
    sp = br.special_values()
    feat = np.tile(sp, (3, 1))
    g = graphs.random_graph(seed=2, n=3, T=1, avg_deg=1)
    gb = _csr(g, (len(sp),), feat)("bfloat16", None)
    got = gb.export()["feat"]
    nan = np.isnan(feat)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got.view(np.uint32)[~nan], br.rounded(feat).view(np.uint32)[~nan])
    _use(gb)
    out = euler_b200.get_dense_feature(g["ids"].astype(np.int64), [0], [len(sp)])[0].cpu().numpy()
    assert np.array_equal(out.view(np.uint32), got.view(np.uint32))


def test_rmat_table_is_the_rounded_f32_table():
    import euler_b200
    kw = dict(seed=3, feat_dim=36, feat_seed=9)
    gf = euler_b200.Graph.rmat(5000, 40000, **kw)
    gb = euler_b200.Graph.rmat(5000, 40000, feat_dtype="bfloat16", **kw)
    assert gb.feat_dtype == "bfloat16"
    ef, eb = gf.export(), gb.export()
    assert np.array_equal(eb["feat"].view(np.uint32), br.rounded(ef["feat"]).view(np.uint32))
    for k in ("ids", "grp_ptr", "nbr", "cum_w"):
        assert np.array_equal(ef[k], eb[k])
    hs = euler_b200.Graph.rmat_shard(5000, 40000, 1, 2, feat_dtype="bfloat16", **kw)
    es = hs.export()
    assert np.array_equal(es["feat"].view(np.uint32), eb["feat"][es["ids"].astype(np.int64) - 1].view(np.uint32))
    hh = euler_b200.Graph.rmat_hetero(5000, 40000, 2, 2, feat_dtype="bfloat16", **kw)
    assert hh.feat_dtype == "bfloat16"


def test_load_and_initialize_graph_round_on_the_device(tiny_dir):
    import euler_b200
    gf = euler_b200.Graph.load(tiny_dir)
    gb = euler_b200.Graph.load(tiny_dir, feat_dtype="bfloat16")
    ef, eb = gf.export(), gb.export()
    assert gb.feat_dtype == "bfloat16" and gf.feat_dim > 0
    assert np.array_equal(eb["feat"].view(np.uint32), br.rounded(ef["feat"]).view(np.uint32))
    ids = ef["ids"].astype(np.int64)
    g2 = euler_b200.Graph.from_csr(ef["ids"], ef["grp_ptr"], ef["nbr"], n_edge_types=ef["T"], node_type=ef["node_type"],
                                   node_w=ef["node_w"], cum_w=ef["cum_w"], grp_cum=ef["grp_cum"], feat=eb["feat"],
                                   feat_slot_dims=[gf.dense_feature_dim(s) for s in range(8) if gf.dense_feature_dim(s) >= 0])
    slots = [s for s in range(8) if gf.dense_feature_dim(s) >= 0]
    dims = [gf.dense_feature_dim(s) + 2 for s in slots]
    _both((gb, g2), lambda: euler_b200.get_dense_feature(ids, slots, dims))
    assert euler_b200.initialize_graph({"mode": "local", "data_path": tiny_dir, "feature_dtype": "bfloat16"})
    gi = euler_b200.get_graph()
    assert gi.feat_dtype == "bfloat16"
    assert np.array_equal(gi.export()["feat"].view(np.uint32), eb["feat"].view(np.uint32))
    _both((gi, g2), lambda: euler_b200.get_dense_feature(ids, slots, dims))


def test_hbm_bytes_drop_by_two_bytes_per_element(env):
    gb, gf = env["single"][256][1]
    assert gf.hbm_bytes - gb.hbm_bytes == 2 * N * 256


# ---------------------------------------------------------------------------- get_dense_feature
@pytest.mark.parametrize("aligned", [True, False])
def test_get_dense_feature_every_slot_width_and_alignment(env, aligned):
    from euler_b200 import ops
    rng = np.random.RandomState(3)
    nodes = torch.as_tensor(_ids(rng, 3001), device="cuda")
    M = nodes.numel()
    table = br.rounded(env["feat"])
    offs = np.concatenate([[0], np.cumsum(SLOTS)])
    for fid in list(range(len(SLOTS))) + [99, -1]:
        w = SLOTS[fid] if 0 <= fid < len(SLOTS) else 0
        for dim in sorted({1, 3, 4, 16, 128, 200, 256, w + 3, max(w - 1, 1), max(w, 1)}):
            def fetch():
                buf = torch.full((M * dim + 1,), 7.0, device="cuda")
                out = (buf[:-1] if aligned else buf[1:]).view(M, dim)
                ops._call("eu_get_dense_feature", nodes, M, fid, dim, out)
                return out
            got = _both(env["multi"], fetch).cpu().numpy()
            want = np.zeros((M, dim), np.float32)
            ids = nodes.cpu().numpy()
            ok = (ids >= 1) & (ids <= N)
            c = min(w, dim)
            if c:
                want[ok, :c] = table[ids[ok] - 1, offs[fid]:offs[fid] + c]
            nan = np.isnan(want)                 # the device's NaN need not be numpy's: compared as NaN-ness
            assert np.array_equal(np.isnan(got), nan), (fid, dim)
            assert np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan]), (fid, dim)


# ---------------------------------------------------------------------------- the fused SAGE reduction
def _segments(rng, rows, count, repeat):
    """rows segments of count ids: absent ids and -1 among them, some rows with no existing neighbour, and (repeat) most
    segments copies of a few hundred distinct ones, as a fanout's deep hop repeats them"""
    distinct = _ids(rng, (min(rows, 300) if repeat else rows) * count).reshape(-1, count)
    seg = distinct[rng.randint(0, len(distinct), size=rows)] if repeat else distinct
    seg[:5] = ABSENT
    return torch.as_tensor(seg.reshape(-1), device="cuda")


def _aggregate(ids, rows, count, dim, mean):
    from euler_b200 import ops
    out = torch.full((rows, dim), 7.0, device="cuda")
    ops._call("eu_sage_mean_aggregate" if mean else "eu_sage_add_aggregate", ids, rows, count, dim, out)
    return out


@pytest.mark.parametrize("count", [1, 10, 25])
@pytest.mark.parametrize("dim", WIDTHS)
def test_sage_mean_and_add_below_the_dedup_rows(env, dim, count):
    rng = np.random.RandomState(dim + count)
    ids = _segments(rng, 700, count, repeat=False)
    pair = env["single"][dim][1]
    for mean in (True, False):
        _both(pair, lambda: _aggregate(ids, 700, count, dim, mean))
        _both(pair, lambda: _aggregate(ids, 700, count, dim - 1 if dim > 1 else dim, mean))   # narrower: the generic path
    _both(env["multi"], lambda: _aggregate(ids, 700, count, sum(SLOTS), True))                 # several slots: generic


@pytest.mark.parametrize("count", [1, 10, 25])
@pytest.mark.parametrize("dim", [3, 128, 256])
def test_sage_mean_and_add_above_the_dedup_rows(env, dim, count):
    rows = (1 << 17) + 5
    ids = _segments(np.random.RandomState(count), rows, count, repeat=True)
    pair = env["single"][dim][1]
    for mean in (True, False):
        out = _both(pair, lambda: _aggregate(ids, rows, count, dim, mean))
        assert torch.equal(_bits(out[:5]), _bits(torch.zeros(5, dim)))      # rows with no neighbour: +0.0


# ---------------------------------------------------------------------------- ShallowEncoder's dense slots
def test_shallow_encode_and_pool_with_dense_slots(env):
    import euler_b200
    rng = np.random.RandomState(4)
    nodes = torch.as_tensor(_ids(rng, 1500), device="cuda")
    dense = [(0, 1), (1, 5), (2, 4), (3, 16), (5, 199), (6, 256), (99, 2)]
    _both(env["multi"], lambda: euler_b200.shallow_encode(nodes, None, dense, (), "concat"))
    for pool in ("sum", "mean"):
        _both(env["multi"], lambda: euler_b200.shallow_encode_pool(nodes, 10, None, dense, (), pool))
    in_table = torch.as_tensor(rng.randint(0, N + 2, size=1500), device="cuda")
    id_table = torch.randn(N + 2, 16, generator=torch.Generator().manual_seed(1)).cuda()
    _both(env["multi"], lambda: euler_b200.shallow_encode(in_table, id_table, [(3, 16), (1, 3), (6, 256)], (), "add"))


# ---------------------------------------------------------------------------- LGCEncoder's top-k
@pytest.mark.parametrize("k", [1, 3, 6, 16])
def test_neighbor_top_k_feature_with_ties_signed_zeros_and_nans(env, k):
    import euler_b200
    rng = np.random.RandomState(k)
    nodes = torch.as_tensor(_ids(rng, 400), device="cuda")
    nbrs = torch.as_tensor(_ids(rng, 400 * 20).reshape(400, 20), device="cuda")
    for slot, dim in ((0, 16), (1, 130), (1, 131), (0, 3)):
        _both(env["ties"], lambda: euler_b200.neighbor_top_k_feature(nodes, nbrs, slot, dim, k))


# ---------------------------------------------------------------------------- sample_fanout_with_feature
def test_sample_fanout_with_feature_dense_outputs(env):
    import euler_b200
    seeds = torch.as_tensor(_ids(np.random.RandomState(5), 300), device="cuda")

    def run():
        euler_b200.seed(9)
        nb, ws, ts, dense, sparse = euler_b200.sample_fanout_with_feature(seeds, [[0], [0]], [4, 3], -1, ["feat1", "feat5"],
                                                                          [3, 201], [], [])
        assert all(x.dtype == torch.float32 for x in dense)
        return list(dense) + list(nb)
    _both(env["multi"], run)


# ---------------------------------------------------------------------------- repeats and CUDA graphs
def test_bits_repeat_and_capture_replays_eager(env):
    import euler_b200
    gb = env["single"][256][1][0]
    _use(gb)
    rng = np.random.RandomState(6)
    nodes = torch.as_tensor(_ids(rng, 2048), device="cuda")
    ids = _segments(rng, 1024, 10, repeat=True)
    nbrs = nodes[:200 * 10].reshape(200, 10)

    def ops_():
        return [euler_b200.get_dense_feature(nodes, [0], [256])[0], euler_b200.sage_mean_aggregate(ids, 10, 256),
                euler_b200.neighbor_top_k_feature(nodes[:200], nbrs, 0, 256, 3),
                euler_b200.shallow_encode(nodes, None, [(0, 250)], (), "concat")]
    first, again = ops_(), ops_()
    for a, b in zip(first, again):
        assert torch.equal(_bits(a), _bits(b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops_()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            captured = ops_()
    torch.cuda.current_stream().wait_stream(s)
    for t in captured:
        t.fill_(7.0)
    cg.replay()
    torch.cuda.synchronize()
    for a, b in zip(captured, first):
        assert torch.equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------- the sharded paths refuse
def test_sharded_feature_paths_refuse_and_write_nothing(env):
    import euler_b200
    from euler_b200 import _lib
    from euler_b200.graph import Context
    from euler_b200.sharded import PeerShardedGraph
    lib = _lib.load()
    gb = env["single"][128][1][0]
    ctx = Context(gb)
    ctx.reserve(4096)
    sym, handle = C.c_void_p(), (C.c_char * 64)()
    assert lib.eu_sym_create(ctx._h, 0, 1, 1024, 16, 1024, 128, C.byref(sym), handle) == 0
    try:
        assert lib.eu_sym_connect(sym, bytes(handle.raw)) == 0
        ptrs = [C.c_void_p() for _ in range(5)]
        assert lib.eu_sym_outputs(sym, *[C.byref(p) for p in ptrs]) == 0
        view = PeerShardedGraph._view(types.SimpleNamespace(torch=torch, dev=torch.device("cuda", 0)), ptrs[4].value, 1024 * 128,
                                      torch.float32)
        view.fill_(5.0)
        ids = torch.arange(1, 101, device="cuda")
        out = torch.full((10, 128), 7.0, device="cuda")
        torch.cuda.synchronize()
        assert lib.eu_sym_get_dense_feature(sym, ids.data_ptr(), 100, 0, 128, 1) == 4      # EU_ERR_UNSUPPORTED
        assert b"f32 tables only" in lib.eu_last_error()
        assert lib.eu_sym_sage_mean(sym, ids.data_ptr(), 10, 10, 128, 1, out.data_ptr()) == 4
        torch.cuda.synchronize()
        assert bool((view == 5.0).all()) and bool((out == 7.0).all())
    finally:
        lib.eu_sym_destroy(sym)
        ctx.close()
    peer = types.SimpleNamespace(torch=torch, graph=gb, feature_graph=None)
    with pytest.raises(euler_b200.EulerError, match="float32 feature tables only"):
        PeerShardedGraph.get_dense_feature(peer, ids, 0, 128)
    with pytest.raises(euler_b200.EulerError, match="float32 feature tables only"):
        PeerShardedGraph.sage_mean(peer, ids, 10, 10, 128)


# ---------------------------------------------------------------------------- training steps
def _step(pair, make, seeds, seed):
    """one SGD step of make() on each graph of the pair, from the same initial parameters and draws: the forward's bits are
    equal, the updated parameters equal up to the order of torch's atomic gradient sums"""
    import euler_b200
    res = []
    for graph in pair:
        _use(graph)
        torch.manual_seed(0)
        model = make()
        opt = torch.optim.SGD(model.parameters(), lr=0.5)
        euler_b200.seed(seed)
        emb, loss, name, metric = model(seeds)
        opt.zero_grad()
        loss.backward()
        opt.step()
        res.append((emb.detach(), loss.detach(), [p.detach().clone() for p in model.parameters()]))
    (e0, l0, p0), (e1, l1, p1) = res
    assert torch.equal(_bits(e0), _bits(e1)) and torch.equal(_bits(l0.reshape(1)), _bits(l1.reshape(1)))
    for a, b in zip(p0, p1):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7)


def test_supervised_sage_encoder_step(env):
    from euler_b200.encoders import SageEncoder
    from euler_b200.supervised import SuperviseModel

    class Sage(SuperviseModel):
        def __init__(self):
            super().__init__("feat0", 3, dim=8, device="cuda")
            self.encoder = SageEncoder([[0], [0]], [5, 3], 8, feature_idx=["feat1", "feat2"], feature_dim=[16, 128], max_id=N,
                                       device="cuda")

        def embed(self, n_id):
            return self.encoder(n_id)
    _step(env["train"], Sage, torch.arange(1, 257, device="cuda"), 5)


def test_lgcn_step(env):
    from euler_b200.supervised import LGCN
    _step(env["train"], lambda: LGCN(16, [0], "feat0", 3, feature_idx="feat2", feature_dim=128, k=3, nb_num=10, out_dim=8,
                                     device="cuda"), torch.arange(1, 257, device="cuda"), 3)
