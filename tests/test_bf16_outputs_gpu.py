"""GPU: bfloat16 outputs of the graph-feature ops (out_dtype= / dense_dtype=, the eu_*_out_dtype entry points).  On f32 and
bf16 tables, device-placed and host-placed (cache 0 and n / 3 rows), every bf16 output must be, bit for bit, the f32 op's
output converted on the device (.to(torch.bfloat16)), and the round-to-nearest-even restatement of tests/bf16_reference.py
(NaN compared as NaN-ness: the device's canonical NaN need not be numpy's)."""
import ctypes as C

import numpy as np
import pytest
import torch

import bf16_reference as br
import graphs

pytestmark = pytest.mark.gpu

SLOTS = (1, 3, 4, 16, 128, 200, 256)          # offsets 0, 1, 4, 8, 24, 152, 352: multiples of 4 and not
WIDTHS = (3, 64, 128, 200, 256, 516, 1024)     # one-slot graphs: every k_sage_mean form and the generic one
COUNTS = (1, 2, 10, 15, 25, 64)
N = 2000
ABSENT = 10 ** 9
BF = torch.bfloat16
VARIANTS = [(dt, place, cache) for dt in ("float32", "bfloat16") for place, cache in (("device", 0), ("host", 0), ("host", N // 3))]
VIDS = ["%s-%s-%d" % v for v in VARIANTS]


def _features(rng, n, d, specials=True):
    f = (rng.standard_normal((n, d)) * 3).astype(np.float32)
    if specials:
        sp = br.special_values()
        mask = rng.rand(n, d) < 0.03
        f[mask] = sp[rng.randint(0, len(sp), size=int(mask.sum()))]
    return f


@pytest.fixture(scope="module")
def env():
    import euler_b200
    rng = np.random.RandomState(21)
    g = graphs.random_graph(seed=21, n=N, T=1, avg_deg=6)

    def build(slots, feat):
        return {v: euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                             node_w=g["node_w"], cum_w=g["cum_w"], feat=feat, feat_slot_dims=list(slots),
                                             feat_dtype=v[0], feat_place=v[1], feat_cache_rows=v[2]) for v in VARIANTS}
    ties = (rng.randint(-4, 5, size=(N, 146)) / 4).astype(np.float32)
    ties[rng.rand(*ties.shape) < 0.1] = np.float32(-0.0)
    ties[rng.rand(*ties.shape) < 0.02] = np.float32("nan")
    ties[:, 16:] += (rng.standard_normal((N, 130)) * 1e-3).astype(np.float32)   # values that round: ties of bf16, not of f32
    yield dict(g=g, multi=build(SLOTS, _features(rng, N, sum(SLOTS))),
               single={d: build((d,), _features(rng, N, d)) for d in WIDTHS}, ties=build((16, 130), ties))
    small = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(small), rng="minstd", seed=1)


def _use(graph, seed=1):
    import euler_b200
    euler_b200.set_graph(graph, rng="minstd", seed=seed)


def _h(t):
    """the int16 bits of a bf16 tensor, on the host"""
    return t.detach().contiguous().view(torch.int16).cpu()


def _check(f32, bf):
    """bf (bf16) is f32 rounded on the device, bit for bit, and the numpy restatement of that rounding (on at most 4096 rows
    of a large output: its first rows and rows spread over the rest)"""
    assert bf.dtype == BF and f32.dtype == torch.float32 and bf.shape == f32.shape
    assert torch.equal(bf.view(torch.int16), f32.to(BF).view(torch.int16))
    if f32.dim() > 1 and f32.shape[0] > 4096:
        r = torch.cat([torch.arange(2048), torch.linspace(2048, f32.shape[0] - 1, 2048).long()]).to(f32.device)
        f32, bf = f32[r], bf[r]
    x = f32.detach().cpu().numpy()
    got = _h(bf).numpy().view(np.uint16)
    want = br.round_bits(x).reshape(x.shape)
    nan = np.isnan(x)
    assert np.array_equal(np.isnan(br.widen(got)).reshape(x.shape), nan)
    assert np.array_equal(got[~nan], want[~nan])


def _ids(rng, M, absent=0.1):
    ids = rng.randint(1, N + 1, size=M).astype(np.int64)
    ids[rng.rand(M) < absent] = ABSENT
    ids[rng.rand(M) < absent / 2] = -1
    return torch.as_tensor(ids, device="cuda")


def _raw(name, shape, dtype, offset, *args):
    """the entry point `name` into a fresh output of dtype and shape that starts `offset` elements into its buffer"""
    from euler_b200 import ops
    n = int(np.prod(shape))
    buf = torch.full((n + offset,), 7.0, dtype=dtype, device="cuda")
    out = buf[offset:]
    ops._call(name, *args, out)
    return out.view(shape)


# ---------------------------------------------------------------------------- get_dense_feature
@pytest.mark.parametrize("variant", VARIANTS, ids=VIDS)
def test_dense_feature_is_the_rounded_f32_feature(env, variant):
    import euler_b200
    _use(env["multi"][variant])
    nodes = _ids(np.random.RandomState(1), 1537)
    for fid, width in enumerate(SLOTS):
        for dim in sorted({max(width - 1, 1), width, width + 5, 256}):   # below, at and past the slot width (zero pad)
            f32 = euler_b200.get_dense_feature(nodes, [fid], [dim])[0]
            _check(f32, euler_b200.get_dense_feature(nodes, [fid], [dim], out_dtype=BF)[0])
            for offset in (0, 1):   # offset by one element: the scalar path
                _check(f32, _raw("eu_get_dense_feature_out_dtype", (1537, dim), BF, offset, nodes, 1537, fid, dim, 1))
    f32 = euler_b200.get_dense_feature(nodes, [0, 3, 6, 42], [1, 16, 256, 8])    # an unknown slot reads zeros
    for a, b in zip(f32, euler_b200.get_dense_feature(nodes, [0, 3, 6, 42], [1, 16, 256, 8], out_dtype=BF)):
        _check(a, b)
    empty = euler_b200.get_dense_feature(nodes[:0], [6], [256], out_dtype=BF)[0]
    assert empty.shape == (0, 256) and empty.dtype == BF


@pytest.mark.parametrize("place,cache", [("device", 0), ("host", 0), ("host", N // 3)])
def test_bf16_table_returns_its_stored_bits(env, place, cache):
    import euler_b200
    graph = env["multi"][("bfloat16", place, cache)]
    _use(graph)
    stored = (graph.export()["feat"].view(np.uint32) >> 16).astype(np.uint16)
    nodes = torch.as_tensor(env["g"]["ids"].astype(np.int64), device="cuda")   # every row, in row order
    got = euler_b200.get_dense_feature(nodes, [0, 1, 2, 3, 4, 5, 6], SLOTS, out_dtype=BF)
    assert np.array_equal(np.concatenate([_h(x).numpy().view(np.uint16) for x in got], 1), stored)


# ---------------------------------------------------------------------------- the fused SAGE mean and sum
def _aggregate(name, ids, rows, count, dim, dtype, offset=0):
    code = 1 if dtype == BF else 0
    return _raw(name, (rows, dim), dtype, offset, ids, rows, count, dim, code)


def _fanout_hop(count, B=8192, first=16):
    """the deep hop of a real fanout: B seeds drawn `first` times, then `count` neighbours of each of those rows (B * first
    >= 2^17 rows, with the sampler's repeated segments)"""
    import euler_b200
    seeds = _ids(np.random.RandomState(count), B, absent=0.02)
    euler_b200.seed(count)
    nb, _, _ = euler_b200.sample_fanout(seeds, [[0], [0]], [first, count])
    return nb[2].reshape(-1), B * first


@pytest.mark.parametrize("dim", WIDTHS)
@pytest.mark.parametrize("variant", VARIANTS, ids=VIDS)
def test_sage_mean_and_add_are_the_rounded_f32_results(env, variant, dim):
    import euler_b200
    _use(env["single"][dim][variant])
    rng = np.random.RandomState(dim)
    for count in COUNTS:
        small = _ids(rng, 700 * count)
        small[:5 * count] = ABSENT                            # rows without a neighbour: +0.0
        hop, big = _fanout_hop(count)
        assert big >= 1 << 17
        for ids, rows in ((small, 700), (hop, big)):
            for name in ("eu_sage_mean_aggregate_out_dtype", "eu_sage_add_aggregate_out_dtype"):
                f32 = _aggregate(name, ids, rows, count, dim, torch.float32)
                bf = _aggregate(name, ids, rows, count, dim, BF)
                _check(f32, bf)
                if rows == 700 or count in (2, 25):              # outputs offset by one element, both dtypes
                    assert torch.equal(_aggregate(name, ids, rows, count, dim, torch.float32, 1).view(torch.int32), f32.view(torch.int32))
                    assert torch.equal(_h(_aggregate(name, ids, rows, count, dim, BF, 1)), _h(bf))
        assert not _h(_aggregate("eu_sage_mean_aggregate_out_dtype", small, 700, count, dim, BF)[:5]).any()
    assert torch.equal(_h(euler_b200.sage_mean_aggregate(hop, COUNTS[-1], dim, out_dtype=BF)),
                       _h(euler_b200.sage_mean_aggregate(hop, COUNTS[-1], dim).to(BF)))


def test_sage_mean_on_several_slots_takes_the_generic_path(env):
    import euler_b200
    for variant in VARIANTS:
        _use(env["multi"][variant])
        ids = _ids(np.random.RandomState(2), 900 * 10)
        for dim in (sum(SLOTS), 100):
            _check(euler_b200.sage_mean_aggregate(ids, 10, dim), euler_b200.sage_mean_aggregate(ids, 10, dim, out_dtype=BF))


# ---------------------------------------------------------------------------- the host-buffer twins
@pytest.mark.parametrize("variant", VARIANTS, ids=VIDS)
def test_host_twins_into_pageable_and_pinned_buffers(env, variant):
    import euler_b200
    from euler_b200 import _lib
    _use(env["single"][256][variant])
    lib, h = _lib.load(), euler_b200.context()._h
    nodes = _ids(np.random.RandomState(3), 3000)
    hn = np.ascontiguousarray(nodes.cpu().numpy())
    dev_feat = euler_b200.get_dense_feature(nodes, [0], [256], out_dtype=BF)[0]
    dev_mean = euler_b200.sage_mean_aggregate(nodes, 10, 256, out_dtype=BF)
    for pinned in (False, True):
        feat = torch.full((3000, 256), 7.0, dtype=BF, pin_memory=pinned)
        mean = torch.full((300, 256), 7.0, dtype=BF, pin_memory=pinned)
        _lib.check(lib.eu_get_dense_feature_host_out_dtype(h, hn.ctypes.data, 3000, 0, 256, 1, feat.data_ptr()))
        _lib.check(lib.eu_sage_mean_aggregate_host_out_dtype(h, hn.ctypes.data, 300, 10, 256, 1, mean.data_ptr()))
        assert torch.equal(feat.view(torch.int16), _h(dev_feat)) and torch.equal(mean.view(torch.int16), _h(dev_mean))


# ---------------------------------------------------------------------------- LGCEncoder's top-k
@pytest.mark.parametrize("k", [1, 3, 8, 16])
def test_neighbor_top_k_feature_with_ties_signed_zeros_and_nans(env, k):
    import euler_b200
    rng = np.random.RandomState(k)
    nodes = _ids(rng, 400)
    nbrs = _ids(rng, 400 * 20).reshape(400, 20)
    for variant in VARIANTS:
        _use(env["ties"][variant])
        for slot, dim in ((0, 16), (1, 130), (1, 131), (0, 3)):
            f32 = euler_b200.neighbor_top_k_feature(nodes, nbrs, slot, dim, k)
            _check(f32, euler_b200.neighbor_top_k_feature(nodes, nbrs, slot, dim, k, out_dtype=BF))
        if variant[0] == "bfloat16":   # a bf16 table's values come back as stored
            got = euler_b200.neighbor_top_k_feature(nodes, nbrs, 1, 130, k, out_dtype=BF)
            f32 = euler_b200.neighbor_top_k_feature(nodes, nbrs, 1, 130, k)   # the stored bits, widened: the upper halves
            assert torch.equal(_h(got), (f32.view(torch.int32) >> 16).to(torch.int16).cpu())


# ---------------------------------------------------------------------------- sample_fanout_with_feature
@pytest.mark.parametrize("variant", VARIANTS, ids=VIDS)
def test_sample_fanout_with_feature_bf16_dense(env, variant):
    import euler_b200
    _use(env["multi"][variant])
    seeds = _ids(np.random.RandomState(5), 300)

    def run(dtype):
        euler_b200.seed(9)
        out = euler_b200.sample_fanout_with_feature(seeds, [[0], [0]], [4, 3], -1, ["feat1", "feat6", 5], [3, 256, 201], [], [],
                                                    dense_dtype=dtype)
        nxt = euler_b200.sample_neighbor(seeds, [0], 5)   # a following draw continues the same engine
        return out, nxt
    (nb, ws, ts, dense, sparse), nxt = run(torch.float32)
    (nb2, ws2, ts2, dense2, sparse2), nxt2 = run(BF)
    for a, b in zip(nb + ws + ts + list(nxt), nb2 + ws2 + ts2 + list(nxt2)):
        assert a.dtype == b.dtype and torch.equal(a, b)
    assert len(dense) == len(dense2) == 9 and not sparse and not sparse2
    for a, b in zip(dense, dense2):
        _check(a, b)


# ---------------------------------------------------------------------------- repeats, CUDA graphs, no host sync
def _all_ops(nodes, ids, nbrs):
    import euler_b200
    return [euler_b200.get_dense_feature(nodes, [0], [256], out_dtype=BF)[0], euler_b200.sage_mean_aggregate(ids, 10, 256, out_dtype=BF),
            euler_b200.neighbor_top_k_feature(nodes[:200], nbrs, 0, 256, 3, out_dtype=BF)]


def test_bits_repeat_and_capture_replays_eager(env):
    _use(env["single"][256][("bfloat16", "host", N // 3)])
    nodes = _ids(np.random.RandomState(6), 2048)
    hop, _ = _fanout_hop(10)
    ids = hop[:(1 << 17) * 10]
    nbrs = nodes[:2000].reshape(200, 10)
    first, again = _all_ops(nodes, ids, nbrs), _all_ops(nodes, ids, nbrs)
    for a, b in zip(first, again):
        assert torch.equal(_h(a), _h(b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _all_ops(nodes, ids, nbrs)
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            captured = _all_ops(nodes, ids, nbrs)
    torch.cuda.current_stream().wait_stream(s)
    for x in captured:
        x.fill_(0)
    cg.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, captured):
        assert torch.equal(_h(a), _h(b))


def test_device_twins_do_not_wait_for_the_stream(env):
    """each device twin returns while a long kernel queued before it is still running"""
    import euler_b200
    _use(env["single"][256][("float32", "device", 0)])
    nodes = _ids(np.random.RandomState(7), 2048)
    hop, _ = _fanout_hop(10)
    nbrs = nodes[:2000].reshape(200, 10)
    def calls():
        _all_ops(nodes, hop, nbrs)
        euler_b200.sample_fanout_with_feature(nodes, [[0]], [3], -1, [0], [256], [], [], dense_dtype=BF)
    calls()   # scratch and allocator blocks sized before the timed calls
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(2_000_000_000)
    done.record()
    calls()
    assert not done.query()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------- refusals
def test_unknown_out_dtype_writes_nothing(env):
    import euler_b200
    from euler_b200 import _lib
    _use(env["single"][256][("float32", "device", 0)])
    lib, ctx = _lib.load(), euler_b200.context()
    h = ctx._h
    nodes = _ids(np.random.RandomState(8), 300)
    hn = np.ascontiguousarray(nodes.cpu().numpy())
    out = torch.full((300, 3, 256), 7.0, device="cuda")
    host = np.full((300, 256), 7.0, np.float32)
    before = ctx.draws()
    for bad in (2, -1, 99):
        calls = {
            "eu_get_dense_feature_out_dtype": lambda: lib.eu_get_dense_feature_out_dtype(h, nodes.data_ptr(), 300, 0, 256, bad, out.data_ptr()),
            "eu_get_dense_feature_host_out_dtype": lambda: lib.eu_get_dense_feature_host_out_dtype(h, hn.ctypes.data, 300, 0, 256, bad,
                                                                                                  host.ctypes.data),
            "eu_sage_mean_aggregate_out_dtype": lambda: lib.eu_sage_mean_aggregate_out_dtype(h, nodes.data_ptr(), 30, 10, 256, bad,
                                                                                            out.data_ptr()),
            "eu_sage_mean_aggregate_host_out_dtype": lambda: lib.eu_sage_mean_aggregate_host_out_dtype(h, hn.ctypes.data, 30, 10, 256, bad,
                                                                                                      host.ctypes.data),
            "eu_sage_add_aggregate_out_dtype": lambda: lib.eu_sage_add_aggregate_out_dtype(h, nodes.data_ptr(), 30, 10, 256, bad,
                                                                                          out.data_ptr()),
            "eu_neighbor_top_k_feature_out_dtype": lambda: lib.eu_neighbor_top_k_feature_out_dtype(
                h, nodes.data_ptr(), 30, nodes.data_ptr(), 10, 0, 256, 2, bad, out.data_ptr()),
            "eu_sample_fanout_with_feature_out_dtype": lambda: _fanout_with_feature_raw(lib, h, nodes, bad, out),
        }
        for name, call in calls.items():
            assert call() == 1, name
            assert lib.eu_last_error().decode() == "%s: unknown output dtype %d (EU_FEAT_F32 or EU_FEAT_BF16)" % (name, bad)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()) and bool((host == 7.0).all())
    assert ctx.draws() == before


def _fanout_with_feature_raw(lib, h, nodes, dtype, out):
    ids, w, t, eng = (torch.full((900,), 5, dtype=d, device="cuda") for d in (torch.int64, torch.float32, torch.int32, torch.int64))
    P = C.c_void_p * 1
    rc = lib.eu_sample_fanout_with_feature_out_dtype(
        h, nodes.data_ptr(), 300, np.zeros(1, np.int32).ctypes.data, 1, np.full(1, 3, np.int32).ctypes.data, 1, -1,
        P(ids.data_ptr()), P(w.data_ptr()), P(t.data_ptr()), P(eng.data_ptr()), 1, np.zeros(1, np.int32).ctypes.data,
        np.full(1, 256, np.int32).ctypes.data, dtype, (C.c_void_p * 2)(out.data_ptr(), out.data_ptr()), 0, None, None, None, None)
    torch.cuda.synchronize()
    assert bool((ids == 5).all()) and bool((w == 5).all()) and bool((t == 5).all()) and bool((eng == 5).all())
    return rc


# ---------------------------------------------------------------------------- bf16 outputs past 2^31 elements
T31 = 1 << 31


@pytest.fixture(scope="module")
def wide():
    import euler_b200
    free, _ = torch.cuda.mem_get_info()
    if free < (12 << 30):
        pytest.skip("needs 12 GB of free device memory")
    g = euler_b200.Graph.rmat(200_000, 1_000_000, feat_dim=256)
    euler_b200.set_graph(g, rng="minstd", seed=1)
    yield euler_b200
    small = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(small), rng="minstd", seed=1)
    del g
    torch.cuda.empty_cache()


def _sampled_rows(rows, k=3000):
    """row 0, the rows either side of element 2^31 at width 256, the last row and k random rows past 2^31"""
    rng = np.random.RandomState(rows % 1000)
    first = T31 // 256
    return torch.as_tensor(np.concatenate([[0, first - 1, first, rows - 1], rng.randint(first, rows, size=k)]), device="cuda")


def test_dense_feature_bf16_output_past_2_31(wide):
    M = T31 // 256 + 40_000
    nodes = torch.randint(0, 200_010, (M,), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    out = wide.get_dense_feature(nodes, [0], [256], out_dtype=BF)[0]
    assert out.numel() > T31
    r = _sampled_rows(M)
    _check(wide.get_dense_feature(nodes[r], [0], [256])[0], out[r])
    del out


def test_sage_mean_bf16_output_past_2_31(wide):
    rows, count = T31 // 256 + 40_000, 2
    ids = torch.randint(0, 200_010, (rows * count,), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    ids[count * 10:count * 600] = ids[count * 9:count * 10].repeat(590)    # one segment repeated 591 times
    out = wide.sage_mean_aggregate(ids, count, 256, out_dtype=BF)
    assert out.numel() > T31
    r = _sampled_rows(rows)
    r = torch.cat([r, torch.arange(9, 600, device="cuda")])
    seg = ids.view(rows, count)[r].reshape(-1)
    _check(wide.sage_mean_aggregate(seg, count, 256), out[r])
    del out
