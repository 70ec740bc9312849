"""The host-buffer C ABI (the 16 eu_*_host entry points) against the device entry points on the same inputs.

Every entry point runs with page-locked caller buffers (torch pin_memory, DMA'd in place) and with pageable ones (numpy,
staged through the ctx's pinned buffer); both must equal the device entry point bit for bit, RNG ops under the same engine
seeds.  Also checked: the ragged entry points' cap contract, every entry point with empty inputs, and calls that grow the
ctx's staging buffers, between calls and between the two phases of a ragged call."""
import ctypes as C

import numpy as np
import pytest
import torch

import cases
import graphs

pytestmark = pytest.mark.gpu
MODES = ("pinned", "pageable")
P2 = C.c_void_p * 2
SENTINEL = {np.dtype(np.int64): -7, np.dtype(np.float32): -7.5, np.dtype(np.int32): -7, np.dtype(np.uint8): 0xA5}


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def env():
    """a 2-edge-type, 3-node-type graph with a hub, a 24-wide dense feature, two uint64 slots and one binary slot per node
    (some of them empty); nodes to query include absent ids and 0"""
    import euler_b200
    from euler_b200 import _lib
    g = graphs.random_graph(seed=91, n=6000, T=2, avg_deg=8, n_node_types=3, feat_dim=24, hub=700, zero_w_frac=0.05)
    n = len(g["ids"])
    rs = np.random.RandomState(92)
    u64_len = rs.randint(1, 6, size=2 * n) * (rs.rand(2 * n) > 0.3)
    u64_ptr = np.concatenate([[0], np.cumsum(u64_len)]).astype(np.int64)
    u64_val = rs.randint(1, 2 ** 62, size=int(u64_ptr[-1]), dtype=np.int64).astype(np.uint64)
    bin_len = rs.randint(0, 14, size=n)
    bin_ptr = np.concatenate([[0], np.cumsum(bin_len)]).astype(np.int64)
    bin_val = rs.randint(0, 256, size=int(bin_ptr[-1])).astype(np.uint8)
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=2, cum_w=g["cum_w"], grp_cum=g["grp_cum"],
                                   node_type=g["node_type"], node_w=g["node_w"], n_node_types=3, feat=g["feat"],
                                   u64_ptr=u64_ptr, u64_val=u64_val, n_u64_slots=2, bin_ptr=bin_ptr, bin_val=bin_val, n_bin_slots=1)
    nodes = g["ids"][rs.randint(0, n, size=900)].astype(np.int64)
    nodes[::11] = 10 ** 15
    nodes[5::13] = 0
    hub = int(np.argmax(np.diff(g["grp_ptr"]))) // 2
    nodes[1] = g["ids"][hub]
    return dict(g=g, gr=gr, lib=_lib.load(), nodes=nodes)


def host(mode, a):
    """a copy of `a` in page-locked or in pageable host memory"""
    a = np.ascontiguousarray(a)
    if mode == "pageable" or a.size == 0:   # an empty buffer is never copied
        return a.copy()
    t = torch.from_numpy(a.copy()).pin_memory()
    assert t.is_pinned()
    return t.numpy()   # shares (and keeps alive) the pinned storage


def host_out(mode, n, dtype):
    return host(mode, np.full(n, SENTINEL[np.dtype(dtype)], dtype))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def dev_out(n, dtype):
    return torch.empty(n, dtype=getattr(torch, np.dtype(dtype).name), device="cuda")


def call(fn, ctx, *args):
    """fn(ctx, *args) with arrays and tensors passed as pointers; they stay referenced for the whole call"""
    from euler_b200 import _lib
    conv = [a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    _lib.check(fn(ctx._h, *conv))


def contexts(env, seed=7, engines=1):
    """a host-side and a device-side ctx with the same engines"""
    import euler_b200
    out = []
    for _ in range(2):
        c = euler_b200.Context(env["gr"], "minstd", seed)
        if engines > 1:
            c.set_engines(engines, [seed + b for b in range(engines)])
        out.append(c)
    return out


def fetched(ctx, pairs):
    """(host result, device tensor, label) -> (host result, device result on the host, label), after the device ctx's work"""
    ctx.sync()
    return [(h, d.cpu().numpy(), label) for h, d, label in pairs]


# ------------------------------------------------------------------ one function per entry point: [(host, device, label)]
def fanout(env, mode, nodes, nb=1):
    lib = env["lib"]
    B = len(nodes) // nb
    et = np.asarray([[0, 1], [1, 0]], np.int32)
    cs = np.asarray([4, 3], np.int32)
    hc, dc = contexts(env, engines=nb)
    sizes = [nb * B * 4, nb * B * 12]
    dts = (np.int64, np.float32, np.int32)
    h = [[host_out(mode, k, dt) for k in sizes] for dt in dts]
    d = [[dev_out(k, dt) for k in sizes] for dt in dts]
    hn = host(mode, nodes[:nb * B])
    ptrs = [P2(*[x.ctypes.data for x in arrs]) for arrs in h]
    if nb == 1:
        call(lib.eu_sample_fanout_host, hc, hn, B, et, 2, cs, 2, -1, *ptrs)
    else:
        call(lib.eu_sample_fanout_batched_host, hc, hn, nb, B, et, 2, cs, 2, -1, *ptrs)
    call(lib.eu_sample_fanout_batched, dc, dev(nodes[:nb * B]), nb, B, et, 2, cs, 2, -1, *[P2(*[x.data_ptr() for x in arrs]) for arrs in d])
    return fetched(dc, [(h[k][l], d[k][l], "fanout nb=%d out %d hop %d" % (nb, k, l)) for k in range(3) for l in range(2)])


def fanout_batched(env, mode, nodes):
    return fanout(env, mode, nodes, nb=2)


def sample_neighbor(env, mode, nodes):
    lib, B, et = env["lib"], len(nodes), np.asarray([0, 1], np.int32)
    hc, dc = contexts(env)
    h = [host_out(mode, 5 * B, dt) for dt in (np.int64, np.float32, np.int32)]
    d = [dev_out(5 * B, dt) for dt in (np.int64, np.float32, np.int32)]
    call(lib.eu_sample_neighbor_host, hc, host(mode, nodes), B, et, 2, 5, -3, *h)
    call(lib.eu_sample_neighbor, dc, dev(nodes), B, et, 2, 5, -3, *d)
    return fetched(dc, [(x, y, "sample_neighbor %d" % k) for k, (x, y) in enumerate(zip(h, d))])


def sample_neighbor_raw(env, mode, nodes):
    lib, B, et = env["lib"], len(nodes), np.asarray([1, 0], np.int32)
    hc, dc = contexts(env)
    h = [host_out(mode, 4 * B, dt) for dt in (np.int64, np.float32, np.int32)]
    d = [dev_out(4 * B, dt) for dt in (np.int64, np.float32, np.int32)]
    call(lib.eu_sample_neighbor_raw_host, hc, host(mode, nodes), B, et, 2, 4, *h)
    call(lib.eu_sample_neighbor_raw, dc, dev(nodes), B, et, 2, 4, *d)
    return fetched(dc, [(x, y, "sample_neighbor_raw %d" % k) for k, (x, y) in enumerate(zip(h, d))])


def sample_node(env, mode, nodes):
    lib, count, types = env["lib"], len(nodes), np.asarray([-1], np.int32)
    hc, dc = contexts(env)
    h, d = host_out(mode, count, np.int64), dev_out(count, np.int64)
    call(lib.eu_sample_node_host, hc, count, types, 1, h)
    call(lib.eu_sample_node, dc, count, types, 1, d)
    return fetched(dc, [(h, d, "sample_node")])


def random_walk(env, mode, nodes):
    lib, B, L = env["lib"], len(nodes), 4
    et = np.asarray([[0, 1]] * L, np.int32)
    hc, dc = contexts(env)
    h, d = host_out(mode, B * (L + 1), np.int64), dev_out(B * (L + 1), np.int64)
    call(lib.eu_random_walk_host, hc, host(mode, nodes), B, et, 2, L, C.c_float(0.5), C.c_float(2.0), -1, h)
    call(lib.eu_random_walk, dc, dev(nodes), B, et, 2, L, C.c_float(0.5), C.c_float(2.0), -1, d)
    return fetched(dc, [(h, d, "random_walk")])


def dense_feature(env, mode, nodes):
    lib, M = env["lib"], len(nodes)
    hc, dc = contexts(env)
    h, d = host_out(mode, M * 24, np.float32), dev_out(M * 24, np.float32)
    call(lib.eu_get_dense_feature_host, hc, host(mode, nodes), M, 0, 24, h)
    call(lib.eu_get_dense_feature, dc, dev(nodes), M, 0, 24, d)
    return fetched(dc, [(h, d, "dense_feature")])


def sage_mean(env, mode, nodes):
    lib, rows = env["lib"], len(nodes) // 3
    hc, dc = contexts(env)
    h, d = host_out(mode, rows * 24, np.float32), dev_out(rows * 24, np.float32)
    call(lib.eu_sage_mean_aggregate_host, hc, host(mode, nodes[:3 * rows]), rows, 3, 24, h)
    call(lib.eu_sage_mean_aggregate, dc, dev(nodes[:3 * rows]), rows, 3, 24, d)
    return fetched(dc, [(h, d, "sage_mean")])


def mp_inputs(nodes, D=8):
    """N = len(nodes) / 3 rows of D floats to gather, E = len(nodes) rows to scatter and sorted i32 indices into the N rows
    (the scatters' deterministic path)"""
    rs = np.random.RandomState(len(nodes))
    E, N = len(nodes), len(nodes) // 3
    idx = np.sort(rs.randint(0, max(N, 1), size=E)).astype(np.int32)
    return rs.randn(N, D).astype(np.float32), rs.randn(E, D).astype(np.float32), idx, N, D


def gather(env, mode, nodes):
    lib = env["lib"]
    params, _, idx, N, D = mp_inputs(nodes)
    E = len(idx)
    hc, dc = contexts(env)
    h, d = host_out(mode, E * D, np.float32), dev_out(E * D, np.float32)
    call(lib.eu_gather_host, hc, host(mode, params), N, D, host(mode, idx), E, h)
    call(lib.eu_gather, dc, dev(params), N, D, dev(idx), E, d)
    return fetched(dc, [(h, d, "gather")])


def scatter(env, mode, nodes, name):
    lib = env["lib"]
    _, x, idx, N, D = mp_inputs(nodes)
    E = len(idx)
    hc, dc = contexts(env)
    h, d = host_out(mode, N * D, np.float32), dev_out(N * D, np.float32)
    call(getattr(lib, "eu_%s_host" % name), hc, host(mode, x), D, host(mode, idx), E, N, h)
    call(getattr(lib, "eu_%s" % name), dc, dev(x), D, dev(idx), E, N, d)
    return fetched(dc, [(h, d, name)])


def scatter_add(env, mode, nodes):
    return scatter(env, mode, nodes, "scatter_add")


def scatter_max(env, mode, nodes):
    return scatter(env, mode, nodes, "scatter_max")


def node_type(env, mode, nodes):
    lib, B = env["lib"], len(nodes)
    hc, dc = contexts(env)
    h, d = host_out(mode, B, np.int32), dev_out(B, np.int32)
    call(lib.eu_get_node_type_host, hc, host(mode, nodes), B, h)
    call(lib.eu_get_node_type, dc, dev(nodes), B, d)
    return fetched(dc, [(h, d, "node_type")])


def node_weight(env, mode, nodes):
    """no device entry point: the graph's node_w of each node's row, 0.0 for absent ids, computed with torch on the device"""
    g, lib, B = env["g"], env["lib"], len(nodes)
    hc, _ = contexts(env)
    h = host_out(mode, B, np.float32)
    call(lib.eu_get_node_weight_host, hc, host(mode, nodes), B, h)
    ids = dev(g["ids"].astype(np.int64))   # sorted: row = searchsorted
    q = dev(nodes)
    row = torch.searchsorted(ids, q).clamp_(max=len(ids) - 1)
    d = torch.where(ids[row] == q, dev(g["node_w"])[row], torch.zeros((), device="cuda"))
    return [(h, d.cpu().numpy(), "node_weight")]


# ragged: spec = (host fn, device fn, [value dtypes], extra args between M and cap)
RAGGED = {
    "full_neighbor": ("eu_get_full_neighbor_host", "eu_get_full_neighbor", (np.int64, np.float32, np.int32),
                      lambda: (np.asarray([1, 0, 1], np.int32), 3)),
    "sparse_feature": ("eu_get_sparse_feature_host", "eu_get_sparse_feature", (np.int64,), lambda: (1, 77)),
    "binary_feature": ("eu_get_binary_feature_host", "eu_get_binary_feature", (np.uint8,), lambda: (0,)),
}


def ragged_device(env, which, nodes):
    """the device entry point's out_ptr and values (cap = total)"""
    _, dfn, dts, extra = RAGGED[which]
    lib, M = env["lib"], len(nodes)
    _, dc = contexts(env)
    dn, ptr = dev(nodes), dev_out(M + 1, np.int64)
    mid = extra()
    call(getattr(lib, dfn), dc, dn, M, *mid, 0, ptr, *[None] * len(dts))
    dc.sync()
    total = int(ptr[-1].item())
    vals = [dev_out(total, dt) for dt in dts]
    call(getattr(lib, dfn), dc, dn, M, *mid, total, ptr, *vals)
    dc.sync()
    return ptr.cpu().numpy(), [v.cpu().numpy() for v in vals]


def ragged_host(env, which, mode, nodes, cap, ctx=None):
    """the host entry point with sentinel-filled outputs of `cap` entries: (out_ptr, total, values)"""
    hfn, _, dts, extra = RAGGED[which]
    lib, M = env["lib"], len(nodes)
    ctx = ctx or contexts(env)[0]
    ptr = host_out(mode, M + 1, np.int64)
    vals = [host_out(mode, cap, dt) for dt in dts]
    total = C.c_int64(-1)
    call(getattr(lib, hfn), ctx, host(mode, nodes), M, *extra(), cap, ptr, *[v if cap else None for v in vals], C.byref(total))
    return ptr, total.value, vals


def ragged(which):
    def run(env, mode, nodes):
        w_ptr, w_vals = ragged_device(env, which, nodes)
        total = int(w_ptr[-1])
        ptr, t0, _ = ragged_host(env, which, mode, nodes, 0)
        ptr2, t1, vals = ragged_host(env, which, mode, nodes, total)
        assert t0 == t1 == total
        return [(ptr, w_ptr, which + " ptr (cap 0)"), (ptr2, w_ptr, which + " ptr")] + \
               [(v, w, "%s values %d" % (which, k)) for k, (v, w) in enumerate(zip(vals, w_vals))]
    return run


OPS = {"sample_fanout_batched": fanout_batched, "sample_fanout": fanout, "sample_neighbor": sample_neighbor,
       "sample_neighbor_raw": sample_neighbor_raw, "sample_node": sample_node, "random_walk": random_walk,
       "get_dense_feature": dense_feature, "sage_mean_aggregate": sage_mean, "gather": gather, "scatter_add": scatter_add,
       "scatter_max": scatter_max, "get_node_type": node_type, "get_node_weight": node_weight,
       "get_full_neighbor": ragged("full_neighbor"), "get_sparse_feature": ragged("sparse_feature"),
       "get_binary_feature": ragged("binary_feature")}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("op", sorted(OPS))
def test_host_entry_point_equals_device_entry_point(env, op, mode):
    for got, want, label in OPS[op](env, mode, env["nodes"]):
        cases.eq(np.asarray(got).reshape(-1), np.asarray(want).reshape(-1), "%s (%s)" % (label, mode))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("which", sorted(RAGGED))
def test_ragged_cap_contract(env, which, mode):
    """cap = 0: out_ptr and total only; cap = total: every value; 0 < cap < total: exactly the first cap values"""
    nodes = env["nodes"]
    w_ptr, w_vals = ragged_device(env, which, nodes)
    total = int(w_ptr[-1])
    assert total > 3
    ptr, t, vals = ragged_host(env, which, mode, nodes, 0)
    assert t == total
    cases.eq(ptr, w_ptr, "cap 0: out_ptr")
    for cap in (total, total // 3):
        ptr, t, vals = ragged_host(env, which, mode, nodes, cap)
        assert t == total
        cases.eq(ptr, w_ptr, "cap %d: out_ptr" % cap)
        for v, w in zip(vals, w_vals):
            cases.eq(v, w[:cap], "cap %d of %d: values" % (cap, total))
    # a buffer longer than cap: nothing past the first cap entries is written
    hfn, _, dts, extra = RAGGED[which]
    cap = total // 3
    ctx = contexts(env)[0]
    ptr = host_out(mode, len(nodes) + 1, np.int64)
    vals = [host_out(mode, total, dt) for dt in dts]
    t = C.c_int64(-1)
    call(getattr(env["lib"], hfn), ctx, host(mode, nodes), len(nodes), *extra(), cap, ptr, *vals, C.byref(t))
    for v, w in zip(vals, w_vals):
        cases.eq(v[:cap], w[:cap], "first cap values")
        assert (v[cap:] == SENTINEL[v.dtype]).all(), "%s wrote past cap" % which


def test_empty_calls_succeed(env):
    """B / M / E / count = 0 on a fresh ctx: every entry point returns EU_OK; the ragged ones give out_ptr = [0], total 0"""
    for op in sorted(OPS):
        if op.startswith(("get_full", "get_sparse", "get_binary")):
            continue
        for got, want, label in OPS[op](env, "pageable", env["nodes"][:0]):
            assert np.asarray(got).size == 0 and np.asarray(want).size == 0, label
    for which in sorted(RAGGED):
        for cap in (0, 5):
            ptr, t, vals = ragged_host(env, which, "pageable", env["nodes"][:0], cap)
            assert t == 0 and ptr.tolist() == [0], which
            assert all((v == SENTINEL[v.dtype]).all() for v in vals), which


@pytest.mark.parametrize("mode", MODES)
def test_growing_calls_on_one_ctx(env, mode):
    """calls larger than any before them on the same ctx (the staging buffers grow mid-sequence, and within a ragged call
    between its two phases), interleaved so that the stage holds another op's data, equal the device entry points"""
    nodes = env["nodes"]
    ctx = contexts(env)[0]
    for M in (1, 40, 300, len(nodes)):
        sub = nodes[:M]
        # a fresh-ctx reference for the device side, the shared ctx for the host side
        for which in sorted(RAGGED):
            w_ptr, w_vals = ragged_device(env, which, sub)
            ptr, t, vals = ragged_host(env, which, mode, sub, int(w_ptr[-1]), ctx=ctx)
            assert t == int(w_ptr[-1])
            cases.eq(ptr, w_ptr, "%s M=%d out_ptr" % (which, M))
            for v, w in zip(vals, w_vals):
                cases.eq(v, w, "%s M=%d values" % (which, M))
        h = host_out(mode, M * 24, np.float32)
        call(env["lib"].eu_get_dense_feature_host, ctx, host(mode, sub), M, 0, 24, h)
        for got, want, label in dense_feature(env, mode, sub):
            cases.eq(h, want, "shared ctx: %s M=%d" % (label, M))
