"""GPU: dense node features placed in mapped pinned host memory (feat_place='host'), with an HBM cache of the feat_cache_rows
rows of highest in-degree.  Every graph is built twice from the same arrays or seed: device-placed, and host-placed with
C = 0, 1, a partial cache (which splits one call's rows between both tiers) and C = n.  Every op that reads dense rows must
give the device graph's bits; the cached rows must be a numpy restatement of the in-degree ranking on export()'s CSR."""

import numpy as np
import pytest
import torch

import graphs
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

N = 2000
ABSENT = 10 ** 9
SLOTS = (1, 3, 4, 16, 128, 200, 256)
WIDTHS = (3, 128, 256, 384, 516)              # the fused mean's FULL 128 / 256, <= 512, > 512 and the scalar path
DTYPES = ("float32", "bfloat16")


def _caches(n):
    return (0, 1, n // 3, n)


def _csr_graph(seed, T=2, id_stride=1, absent_nbrs=True):
    g = graphs.random_graph(seed=seed, n=N, T=T, avg_deg=5, id_stride=id_stride, hub=300)
    g["nbr"] = g["nbr"].copy()
    g["nbr"][np.isin(g["nbr"], g["ids"][-20:])] = g["ids"][0]          # the last 20 rows: in-degree 0
    if absent_nbrs:                       # neighbour ids without a row: listed, never counted
        rng = np.random.RandomState(seed)
        g["nbr"][rng.rand(len(g["nbr"])) < 0.03] = ABSENT
    return g


def _build(g, slots, feat, dtype, place="device", cache=0):
    import euler_b200
    return euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                     node_w=g["node_w"], cum_w=g["cum_w"], grp_cum=g["grp_cum"], feat=feat,
                                     feat_slot_dims=list(slots), feat_dtype=dtype, feat_place=place, feat_cache_rows=cache)


def _placements(g, slots, feat, dtype):
    """[device graph, host graphs for every cache size]"""
    return [_build(g, slots, feat, dtype)] + [_build(g, slots, feat, dtype, "host", c) for c in _caches(N)]


def expected_slots(e, C):
    """the in-degree ranking restated on an exported CSR: rows by (in-degree descending, row ascending), the first C get
    slots 0 .. C-1"""
    ids = e["ids"].astype(np.uint64)
    row_of = {}
    for r, i in enumerate(ids):
        row_of[int(i)] = r                # a repeated id maps to its last row, as the id -> row table does
    n = len(ids)
    deg = np.zeros(n, np.int64)
    rows = np.array([row_of.get(int(x), -1) for x in e["nbr"]], np.int64)
    np.add.at(deg, rows[rows >= 0], 1)
    order = np.lexsort((np.arange(n), -deg))
    slots = np.full(n, -1, np.int32)
    slots[order[:C]] = np.arange(C, dtype=np.int32)
    return slots, deg


@pytest.fixture(scope="module")
def env():
    rng = np.random.RandomState(5)
    g = _csr_graph(5)
    out = dict(g=g)
    for dt in DTYPES:
        feat = (rng.standard_normal((N, sum(SLOTS))) * 3).astype(np.float32)
        out[("multi", dt)] = _placements(g, SLOTS, feat, dt)
        for w in WIDTHS:
            f = rng.uniform(-1, 1, size=(N, w)).astype(np.float32)
            out[(w, dt)] = _placements(g, (w,), f, dt)
    return out


def _use(graph, seed=1):
    import euler_b200
    euler_b200.set_graph(graph, rng="minstd", seed=seed)


def _bits(t):
    t = torch.as_tensor(t)
    return t.detach().contiguous().view(torch.int32).cpu()


def _same_everywhere(graphs_, fn):
    """fn() on every graph; every result's bits must equal the first (device-placed) graph's"""
    ref = None
    for k, graph in enumerate(graphs_):
        _use(graph)
        out = fn()
        out = list(out) if isinstance(out, (list, tuple)) else [out]
        if ref is None:
            ref = out
            continue
        assert len(out) == len(ref)
        for x, y in zip(ref, out):
            if x is None:
                assert y is None
                continue
            assert x.shape == y.shape and torch.equal(_bits(x), _bits(y)), (k, graph.feat_place, graph.feat_cache_rows)
    return ref


def _ids(rng, M, absent=0.1):
    ids = rng.randint(1, N + 1, size=M).astype(np.int64)
    ids[rng.rand(M) < absent] = ABSENT
    ids[rng.rand(M) < absent / 2] = -1
    return ids


# ---------------------------------------------------------------------------- the selection
@pytest.mark.parametrize("T,id_stride", [(1, 1), (2, 1), (3, 3)])
def test_cached_rows_are_the_in_degree_ranking(T, id_stride):
    g = _csr_graph(7 + T, T=T, id_stride=id_stride)
    feat = np.random.RandomState(1).standard_normal((N, 8)).astype(np.float32)
    e = None
    for C in _caches(N) + (N - 1,):
        gr = _build(g, (8,), feat, "float32", "host", C)
        assert (gr.feat_place, gr.feat_cache_rows) == ("host", C)
        e = gr.export() if e is None else e
        want, deg = expected_slots(e, C)
        assert np.array_equal(gr.feat_cache_slots(), want), C
    assert (deg == 0).any() and len(np.unique(deg)) < N // 4          # zero in-degree rows, and ties
    dev = _build(g, (8,), feat, "float32")
    assert np.array_equal(dev.feat_cache_slots(), np.full(N, -1, np.int32))


def test_rmat_selection_and_table(tiny_dir):
    import euler_b200
    kw = dict(seed=3, feat_dim=36, feat_seed=9)
    for dt in DTYPES:
        gd = euler_b200.Graph.rmat(5000, 40000, feat_dtype=dt, **kw)
        gh = euler_b200.Graph.rmat(5000, 40000, feat_dtype=dt, feat_place="host", feat_cache_rows=700, **kw)
        ed, eh = gd.export(), gh.export()
        for k in ("ids", "grp_ptr", "nbr", "cum_w", "feat"):
            assert np.array_equal(ed[k].view(np.uint8), eh[k].view(np.uint8)), k
        assert np.array_equal(gh.feat_cache_slots(), expected_slots(eh, 700)[0])
        hd = euler_b200.Graph.rmat_hetero(3000, 30000, 3, 2, feat_dtype=dt, **kw)
        hh = euler_b200.Graph.rmat_hetero(3000, 30000, 3, 2, feat_dtype=dt, feat_place="host", feat_cache_rows=1000, **kw)
        assert np.array_equal(hd.export()["feat"].view(np.uint32), hh.export()["feat"].view(np.uint32))
        assert np.array_equal(hh.feat_cache_slots(), expected_slots(hh.export(), 1000)[0])
    # the loaded fixture
    gl = euler_b200.Graph.load(tiny_dir, feat_place="host", feat_cache_rows=3)
    assert np.array_equal(gl.feat_cache_slots(), expected_slots(gl.export(), 3)[0])


# ---------------------------------------------------------------------------- exports and accounting
@pytest.mark.parametrize("dt", DTYPES)
def test_export_and_bytes(env, dt):
    gs = env[(256, dt)]
    want = gs[0].export()
    es = 2 if dt == "bfloat16" else 4
    for gr in gs[1:]:
        got = gr.export()
        for k in ("ids", "node_type", "node_w", "grp_ptr", "nbr", "cum_w", "grp_cum", "feat"):
            assert np.array_equal(want[k].view(np.uint8), got[k].view(np.uint8)), k
        assert gr.host_bytes == N * 256 * es
        table = -(-N * 256 * es // 256) * 256                 # the device table's allocation, 256-byte granular
        cache = -(-max(gr.feat_cache_rows, 1) * 256 * es // 256) * 256 if gr.feat_cache_rows else 0
        slot = -(-N * 4 // 256) * 256
        assert gs[0].hbm_bytes - gr.hbm_bytes == table - cache - slot, gr.feat_cache_rows
    assert gs[0].host_bytes == 0 and gs[0].feat_place == "device" and gs[0].feat_cache_rows == 0


# ---------------------------------------------------------------------------- get_dense_feature
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("aligned", [True, False])
def test_get_dense_feature(env, dt, aligned):
    from euler_b200 import ops
    nodes = torch.as_tensor(_ids(np.random.RandomState(3), 3001), device="cuda")
    M = nodes.numel()
    for fid in list(range(len(SLOTS))) + [99, -1]:
        w = SLOTS[fid] if 0 <= fid < len(SLOTS) else 0
        for dim in sorted({1, 3, 4, 16, 128, 256, w + 3, max(w, 1)}):
            def fetch():
                buf = torch.full((M * dim + 1,), 7.0, device="cuda")
                out = (buf[:-1] if aligned else buf[1:]).view(M, dim)
                ops._call("eu_get_dense_feature", nodes, M, fid, dim, out)
                return out
            _same_everywhere(env[("multi", dt)], fetch)


@pytest.mark.parametrize("dt", DTYPES)
def test_get_dense_feature_host_variant_and_names(env, dt):
    import euler_b200
    from euler_b200 import _lib
    from euler_b200.graph import Context
    ids = _ids(np.random.RandomState(4), 900)
    ref = None
    for gr in env[("multi", dt)]:
        ctx = Context(gr)
        out = np.zeros((900, 130), np.float32)
        _lib.check(_lib.load().eu_get_dense_feature_host(ctx._h, ids.ctypes.data, 900, 4, 130, out.ctypes.data))
        ctx.sync()
        ctx.close()
        _use(gr)
        named = euler_b200.get_dense_feature(ids, ["feat3", "feat5"], [16, 200])
        got = [out] + [x.cpu().numpy() for x in named]
        if ref is None:
            ref = got
        for a, b in zip(ref, got):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---------------------------------------------------------------------------- the fused SAGE reduction
def _segments(rng, rows, count, repeat):
    distinct = _ids(rng, (min(rows, 300) if repeat else rows) * count).reshape(-1, count)
    seg = distinct[rng.randint(0, len(distinct), size=rows)] if repeat else distinct
    seg[:5] = ABSENT
    return torch.as_tensor(seg.reshape(-1), device="cuda")


def _aggregate(ids, rows, count, dim, mean):
    from euler_b200 import ops
    out = torch.full((rows, dim), 7.0, device="cuda")
    ops._call("eu_sage_mean_aggregate" if mean else "eu_sage_add_aggregate", ids, rows, count, dim, out)
    return out


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("dim", WIDTHS)
def test_sage_mean_and_add_every_instantiation(env, dt, dim):
    rng = np.random.RandomState(dim)
    for count in (1, 10):
        ids = _segments(rng, 700, count, repeat=False)
        for mean in (True, False):
            _same_everywhere(env[(dim, dt)], lambda: _aggregate(ids, 700, count, dim, mean))
            _same_everywhere(env[(dim, dt)], lambda: _aggregate(ids, 700, count, dim - 1, mean))   # narrower: generic
    ids = _segments(rng, 700, 10, repeat=False)
    _same_everywhere(env[("multi", dt)], lambda: _aggregate(ids, 700, 10, sum(SLOTS), True))       # several slots


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("dim", [3, 128, 256])
def test_sage_mean_above_the_dedup_rows(env, dt, dim):
    rows = (1 << 17) + 5                   # kRepeatMinRows: the deduplicated path
    ids = _segments(np.random.RandomState(dim), rows, 10, repeat=True)
    for mean in (True, False):
        _same_everywhere(env[(dim, dt)], lambda: _aggregate(ids, rows, 10, dim, mean))


# ---------------------------------------------------------------------------- ShallowEncoder, LGCN's top-k, the fanout
@pytest.mark.parametrize("dt", DTYPES)
def test_shallow_encode_and_pool(env, dt):
    import euler_b200
    rng = np.random.RandomState(6)
    nodes = torch.as_tensor(_ids(rng, 1280), device="cuda")
    dense = [(0, 1), (1, 5), (2, 4), (3, 16), (5, 199), (6, 256), (99, 2)]
    gs = env[("multi", dt)]
    _same_everywhere(gs, lambda: euler_b200.shallow_encode(nodes, None, dense, (), "concat"))
    for count in (1, 10, 64):
        for pool in ("sum", "mean"):
            _same_everywhere(gs, lambda: euler_b200.shallow_encode_pool(nodes, count, None, dense, (), pool))
    in_table = torch.as_tensor(rng.randint(0, N + 2, size=1280), device="cuda")
    id_table = torch.randn(N + 2, 16, generator=torch.Generator().manual_seed(1)).cuda()
    _same_everywhere(gs, lambda: euler_b200.shallow_encode(in_table, id_table, [(3, 16), (1, 3), (6, 256)], (), "add"))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("k", [3, 6, 16])          # KMAX 4, 8, 16
def test_neighbor_top_k_feature(env, dt, k):
    import euler_b200
    rng = np.random.RandomState(k)
    nodes = torch.as_tensor(_ids(rng, 400), device="cuda")
    nbrs = torch.as_tensor(_ids(rng, 400 * 20).reshape(400, 20), device="cuda")
    for slot, dim in ((3, 16), (4, 130), (6, 256), (0, 3)):
        _same_everywhere(env[("multi", dt)], lambda: euler_b200.neighbor_top_k_feature(nodes, nbrs, slot, dim, k))


@pytest.mark.parametrize("dt", DTYPES)
def test_sample_fanout_with_feature(env, dt):
    import euler_b200
    seeds = torch.as_tensor(_ids(np.random.RandomState(8), 300), device="cuda")

    def run():
        euler_b200.seed(9)
        nb, ws, ts, dense, sparse = euler_b200.sample_fanout_with_feature(seeds, [[0, 1], [0, 1]], [4, 3], -1,
                                                                          ["feat1", "feat5"], [3, 201], [], [])
        return list(dense) + list(nb) + list(ws)
    _same_everywhere(env[("multi", dt)], run)


def test_gcn_encoder_infer(env):
    from euler_b200.encoders import GCNEncoder
    ids = torch.as_tensor(_ids(np.random.RandomState(9), 500), device="cuda")

    def run():
        torch.manual_seed(0)
        enc = GCNEncoder([[0], [0, 1]], 8, feature_idx=4, feature_dim=128, device="cuda")
        with torch.no_grad():
            return [enc.infer(ids), enc.infer(chunk_rows=777)]
    _same_everywhere(env[("multi", "float32")], run)


# ---------------------------------------------------------------------------- capture
def test_capture_replays_eager(env):
    import euler_b200
    gr = env[(256, "bfloat16")][3]                # the partial cache
    _use(gr)
    rng = np.random.RandomState(6)
    nodes = torch.as_tensor(_ids(rng, 2048), device="cuda")
    ids = _segments(rng, 1024, 10, repeat=True)
    nbrs = nodes[:200 * 10].reshape(200, 10)

    def ops_():
        return [euler_b200.get_dense_feature(nodes, [0], [256])[0], euler_b200.sage_mean_aggregate(ids, 10, 256),
                euler_b200.neighbor_top_k_feature(nodes[:200], nbrs, 0, 256, 3),
                euler_b200.shallow_encode(nodes, None, [(0, 250)], (), "concat")]
    first = ops_()
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


# ---------------------------------------------------------------------------- a whole training step
def test_supervised_sage_encoder_step():
    """one step over GetLabelFromFea and minimize: loss and every gradient bit-equal across placements"""
    from euler_b200.encoders import SageEncoder
    from euler_b200.supervised import SuperviseModel
    g = _csr_graph(12, T=1)
    rng = np.random.RandomState(12)
    feat = rng.uniform(-1, 1, size=(N, 3 + 16 + 128)).astype(np.float32)
    feat[:, :3] = rng.randint(0, 2, size=(N, 3))

    class Sage(SuperviseModel):
        def __init__(self):
            super().__init__("feat0", 3, dim=8, device="cuda")
            self.encoder = SageEncoder([[0], [0]], [5, 3], 8, feature_idx=["feat1", "feat2"], feature_dim=[16, 128], max_id=N,
                                       device="cuda")

        def embed(self, n_id):
            return self.encoder(n_id)
    seeds = torch.arange(1, 257, device="cuda")
    for dt in DTYPES:
        def step():
            import euler_b200
            torch.manual_seed(0)
            model = Sage()
            euler_b200.seed(5)
            emb, loss, name, metric = model(seeds)
            loss.backward()
            return [emb.detach(), loss.detach().reshape(1)] + [p.grad for p in model.parameters() if p.grad is not None]
        _same_everywhere([_build(g, (3, 16, 128), feat, dt)] +
                         [_build(g, (3, 16, 128), feat, dt, "host", c) for c in _caches(N)], step)


# ---------------------------------------------------------------------------- loading
def test_load_and_initialize_graph(tiny_dir):
    import euler_b200
    gd = euler_b200.Graph.load(tiny_dir)
    slots = [s for s in range(8) if gd.dense_feature_dim(s) >= 0]
    dims = [gd.dense_feature_dim(s) + 2 for s in slots]
    ids = gd.export()["ids"].astype(np.int64)
    ids = np.concatenate([ids, [ABSENT, -1]])
    n = gd.num_nodes
    gs = [gd] + [euler_b200.Graph.load(tiny_dir, feat_place="host", feat_cache_rows=c) for c in (0, 1, n // 2, n)]
    _same_everywhere(gs, lambda: euler_b200.get_dense_feature(ids, slots, dims))
    assert euler_b200.initialize_graph({"mode": "local", "data_path": tiny_dir, "feature_place": "host",
                                        "feature_cache_rows": str(n // 2)})
    gi = euler_b200.get_graph()
    assert (gi.feat_place, gi.feat_cache_rows) == ("host", n // 2)
    assert np.array_equal(gi.feat_cache_slots(), expected_slots(gi.export(), n // 2)[0])
    _same_everywhere([gd, gi], lambda: euler_b200.get_dense_feature(ids, slots, dims))


# ---------------------------------------------------------------------------- refusals and memory
def _rss():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
    return 0


def test_refusals_leave_nothing_and_create_close_holds_steady(env):
    import euler_b200
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(euler_b200.EulerError, match="outside"):
        euler_b200.Graph.rmat(5000, 40000, feat_dim=64, feat_place="host", feat_cache_rows=5001)
    with pytest.raises(euler_b200.EulerError, match="needs feat_place='host'"):
        euler_b200.Graph.rmat(5000, 40000, feat_dim=64, feat_cache_rows=1)
    assert torch.cuda.mem_get_info()[0] == free0
    # the sharded feature paths refuse a host-placed graph
    import types
    from euler_b200.sharded import PeerShardedGraph
    peer = types.SimpleNamespace(torch=torch, graph=env[(128, "float32")][2], feature_graph=None)
    ids = torch.arange(1, 101, device="cuda")
    with pytest.raises(euler_b200.EulerError, match="held in HBM only"):
        PeerShardedGraph.get_dense_feature(peer, ids, 0, 128)
    with pytest.raises(euler_b200.EulerError, match="held in HBM only"):
        PeerShardedGraph.sage_mean(peer, ids, 10, 10, 128)

    def cycle():
        g = euler_b200.Graph.rmat(20000, 100000, feat_dim=256, feat_place="host", feat_cache_rows=5000)   # 20 MB pinned
        assert g.host_bytes == 20000 * 256 * 4
        g.close()
    for _ in range(3):
        cycle()
    torch.cuda.synchronize()
    rss0, free1 = _rss(), torch.cuda.mem_get_info()[0]
    for _ in range(20):
        cycle()
    torch.cuda.synchronize()
    assert _rss() - rss0 < 40 << 20                     # 20 cycles of 20 MB tables: nothing kept
    assert abs(torch.cuda.mem_get_info()[0] - free1) < 64 << 20


# ---------------------------------------------------------------------------- a table and a cache past 2^31 elements
def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_host_table_and_cache_past_2_31_elements():
    import euler_b200
    n, d = 8_500_000, 256                      # 2.18e9 elements: 8.7 GB pinned, and an 8.45M-row cache of 8.65 GB
    table = n * d * 4
    if _mem_available() < 2 * table:
        pytest.skip("needs %.1f GB of MemAvailable (twice the pinned table) on a shared host; %.1f GB available"
                    % (2 * table / 1e9, _mem_available() / 1e9))
    if torch.cuda.mem_get_info()[0] < table + (8 << 30):
        pytest.skip("needs the cache plus 8 GB of free device memory")
    C = 8_450_000
    assert C * d > 1 << 31
    g = euler_b200.Graph.rmat(n, 4 * n, feat_dim=d, feat_place="host", feat_cache_rows=C)
    try:
        slots = g.feat_cache_slots()
        assert (slots >= 0).sum() == C
        rng = np.random.RandomState(1)
        cached, uncached = np.flatnonzero(slots >= 0), np.flatnonzero(slots < 0)
        rows = np.concatenate([cached[rng.randint(0, C, 3000)], np.flatnonzero(slots >= C - 500),
                               uncached[rng.randint(0, len(uncached), 1000)], [n - 1]])
        assert int(slots[rows].max()) * d > 1 << 31             # cache rows past 2^31 elements
        ids = (rows + 1).astype(np.int64)
        _use(g)
        got = euler_b200.get_dense_feature(ids, [0], [d])[0].cpu().numpy()
        want = po.rmat_feat_rows(ids, n, d, 7)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        seg = torch.as_tensor(np.stack([ids[:1000], ids[1000:2000], ids[2000:3000]], 1).reshape(-1), device="cuda")
        mean = euler_b200.sage_mean_aggregate(seg, 3, d).cpu().numpy()
        f = want[:3000].reshape(3, 1000, d).transpose(1, 0, 2)
        acc = np.zeros((1000, d), np.float32)
        for j in range(3):
            acc = (acc + f[:, j]).astype(np.float32)
        assert np.array_equal(mean.view(np.uint32), (acc / np.float32(3 + 1e-7)).astype(np.float32).view(np.uint32))
    finally:
        g.close()
