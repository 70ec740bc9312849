"""GPU: the neighbour mean over a CSR adjacency (ops.adjacency_mean, eu_adjacency_mean and its backward) against a float32
restatement of its documented order and against float64; GCNEncoder with the fused aggregators against the float64
composition on the graph's get_multi_hop_neighbor hops; one GeniePath training step."""
import copy

import numpy as np
import pytest
import torch

import embedding_reference as er

pytestmark = pytest.mark.gpu

N_NODES = 600
SLOT_DIMS = (5, 12, 3)          # the dense slots feat0, feat1, feat2
K = 256                         # kSegChunk


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = er.slot_graph(7, N_NODES, [lambda rng, n: rng.randint(0, 4, size=n)], [lambda rng, k: rng.randint(0, 40, size=k)],
                      feat_dim=sum(SLOT_DIMS))
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=list(SLOT_DIMS),
                                   u64_ptr=g["u64_ptr"], u64_val=g["u64_val"], n_u64_slots=g["S"])
    return dict(g=g, gr=gr)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)


def _adjacency(m, lens, seed=0):
    """indptr / cols (numpy i64) of rows with the given entry counts over m columns; every row's first two entries share a
    column (a multi-edge)"""
    rng = np.random.RandomState(seed)
    lens = np.asarray(lens, np.int64)
    cols = rng.randint(0, max(m, 1), size=int(lens.sum())).astype(np.int64)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    for i in range(len(lens)):
        if lens[i] >= 2:
            cols[indptr[i] + 1] = cols[indptr[i]]
    return indptr, cols


LENS = [0, 1, 256, 257, 3 * 256 + 40, 5, 0, 2, 13, 255, 512, 1]


def _restated(x, indptr, cols):
    """the documented order in float32: chunks of 256 from each row's first entry, each from +0 left to right, the chunk
    sums in chunk order from +0, one rounded division by max(fl(deg), 1e-7)"""
    x = x.astype(np.float32)
    n = len(indptr) - 1
    out = np.zeros((n, x.shape[1]), np.float32)
    for i in range(n):
        b, e = int(indptr[i]), int(indptr[i + 1])
        sums = []
        for c0 in range(b, e, K):
            acc = np.zeros(x.shape[1], np.float32)
            for k in range(c0, min(c0 + K, e)):
                acc = acc + x[cols[k]]
            sums.append(acc)
        if len(sums) == 1:
            s = sums[0]
        else:
            s = np.zeros(x.shape[1], np.float32)
            for p in sums:
                s = s + p
        out[i] = s / np.maximum(np.float32(e - b), np.float32(1e-7))
    return out


def _x(m, D, off=0, seed=1):
    """the same seeded rows, their data pointer `off` floats past a 16-byte boundary"""
    t = torch.empty(m * D + off, device="cuda")
    t[off:] = torch.randn(m * D, generator=torch.Generator().manual_seed(seed)).cuda()
    return t[off:].view(m, D)


def _raw(sym, *args):
    from euler_b200 import _lib, ops
    return getattr(_lib.load(), sym)(ops._ctx_on_stream()._h, *args)


def _ptr(t, off_bytes=0):
    return None if t is None else t.data_ptr() + off_bytes


@pytest.mark.parametrize("D", (1, 3, 4, 16, 128, 200))
def test_forward_bit_exact(env, D):
    import euler_b200
    m = 300
    indptr, cols = _adjacency(m, LENS, seed=D)
    want = _restated(_x(m, D).cpu().numpy(), indptr, cols)
    ip, cl = torch.as_tensor(indptr, device="cuda"), torch.as_tensor(cols, device="cuda")
    for off in (0, 1):                                        # x 16-byte aligned, and 4 bytes past
        x = _x(m, D, off)
        got = euler_b200.adjacency_mean(x, (ip, cl, None))
        assert got.shape == (len(LENS), D)
        assert got.cpu().numpy().tobytes() == want.tobytes(), (D, off)
        buf = torch.empty(len(LENS) * D + 1, device="cuda")   # out 4 bytes past a 16-byte boundary
        assert _raw("eu_adjacency_mean", _ptr(x), m, _ptr(ip), _ptr(cl), len(LENS), len(cols), D, _ptr(buf, 4)) == 0
        assert buf[1:].cpu().numpy().tobytes() == want.tobytes(), (D, off)
    assert not want[0].any() and not want[6].any()           # rows without entries


def test_forward_within_1e6_of_float64_and_empty_shapes(env):
    import euler_b200
    m, D = 500, 64
    indptr, cols = _adjacency(m, LENS * 3, seed=9)
    x = _x(m, D)
    got = euler_b200.adjacency_mean(x, (torch.as_tensor(indptr, device="cuda"), torch.as_tensor(cols, device="cuda")))
    xd = x.double().cpu().numpy()
    want = np.stack([xd[cols[indptr[i]:indptr[i + 1]]].sum(0) / max(indptr[i + 1] - indptr[i], 1e-7) for i in range(len(indptr) - 1)])
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-6, atol=1e-6)
    empty = torch.zeros(0, dtype=torch.int64, device="cuda")
    assert euler_b200.adjacency_mean(x, (torch.zeros(1, dtype=torch.int64, device="cuda"), empty)).shape == (0, D)   # n = 0
    out = euler_b200.adjacency_mean(torch.zeros(0, D, device="cuda"), (torch.zeros(4, dtype=torch.int64, device="cuda"), empty))
    assert out.shape == (3, D) and not out.any()                                                                    # m = 0


def test_forward_captures_in_a_cuda_graph(env):
    import euler_b200
    m, D = 400, 32
    indptr, cols = _adjacency(m, LENS, seed=4)
    adj = (torch.as_tensor(indptr, device="cuda"), torch.as_tensor(cols, device="cuda"))
    x = _x(m, D)
    eager = euler_b200.adjacency_mean(x, adj)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        euler_b200.adjacency_mean(x, adj)
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = euler_b200.adjacency_mean(x, adj)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    cg.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == eager.cpu().numpy().tobytes()


def test_raw_abi_statuses(env):
    INVALID, UNSUPPORTED = 1, 4
    m, D = 10, 4
    indptr, cols = _adjacency(m, [2, 0, 3], seed=1)
    x, ip, cl = _x(m, D), torch.as_tensor(indptr, device="cuda"), torch.as_tensor(cols, device="cuda")
    out = torch.empty(3 * D, device="cuda")
    f = "eu_adjacency_mean"
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), 3, 5, D, _ptr(out)) == 0
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), 3, 5, 0, _ptr(out)) == INVALID          # D < 1
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), -1, 5, D, _ptr(out)) == INVALID         # negative sizes
    assert _raw(f, _ptr(x), -2, _ptr(ip), _ptr(cl), 3, 5, D, _ptr(out)) == INVALID
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), 3, -5, D, _ptr(out)) == INVALID
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), 3, 5, D, None) == INVALID               # NULL pointers that are needed
    assert _raw(f, None, m, _ptr(ip), _ptr(cl), 3, 5, D, _ptr(out)) == INVALID
    assert _raw(f, _ptr(x), m, _ptr(ip), None, 3, 5, D, _ptr(out)) == INVALID
    assert _raw(f, _ptr(x), 0, _ptr(ip), _ptr(cl), 3, 5, D, _ptr(out)) == INVALID          # entries without columns
    assert _raw(f, None, 0, None, None, 0, 0, D, None) == 0                                # nothing to do
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), 1 << 31, 5, D, _ptr(out)) == UNSUPPORTED
    assert _raw(f, _ptr(x), 1 << 31, _ptr(ip), _ptr(cl), 3, 5, D, _ptr(out)) == UNSUPPORTED
    assert _raw(f, _ptr(x), m, _ptr(ip), _ptr(cl), 3, (1 << 31) - 2, D, _ptr(out)) == UNSUPPORTED   # chunks reach 2^31
    b = "eu_adjacency_mean_backward"
    g, gx = torch.ones(3, D, device="cuda"), torch.empty(m, D, device="cuda")
    assert _raw(b, _ptr(g), _ptr(ip), _ptr(cl), 3, 5, m, D, _ptr(gx)) == 0
    assert _raw(b, _ptr(g), _ptr(ip), _ptr(cl), 3, 5, m, D, None) == INVALID
    assert _raw(b, None, _ptr(ip), _ptr(cl), 3, 5, m, D, _ptr(gx)) == INVALID
    assert _raw(b, _ptr(g), _ptr(ip), _ptr(cl), 3, 5, m, -1, _ptr(gx)) == INVALID
    assert _raw(b, _ptr(g), _ptr(ip), _ptr(cl), 3, 5, 1 << 31, D, _ptr(gx)) == UNSUPPORTED


def _grad(x, adj, grad_out):
    import euler_b200
    leaf = x.detach().clone().requires_grad_(True)
    euler_b200.adjacency_mean(leaf, adj).backward(grad_out)
    return leaf.grad


@pytest.mark.parametrize("D", (3, 128))
def test_backward_f64_run_to_run_and_untouched_columns(env, D):
    m = 900
    lens = LENS * 2
    indptr, cols = _adjacency(m, lens, seed=D)
    cols[cols == 7] = 8                                         # column 7 has no entries
    cols[indptr[4]:indptr[5]] = 11                              # column 11 gets more than 3 chunks of entries
    adj = (torch.as_tensor(indptr, device="cuda"), torch.as_tensor(cols, device="cuda"))
    x = _x(m, D)
    go = torch.randn(len(lens), D, generator=torch.Generator().manual_seed(5)).cuda()
    g1, g2 = _grad(x, adj, go), _grad(x, adj, go)
    assert g1.cpu().numpy().tobytes() == g2.cpu().numpy().tobytes()
    gd = go.double().cpu().numpy()
    want = np.zeros((m, D))
    for i in range(len(lens)):
        deg = indptr[i + 1] - indptr[i]
        for k in range(indptr[i], indptr[i + 1]):
            want[cols[k]] += gd[i] / deg
    np.testing.assert_allclose(g1.cpu().numpy(), want, rtol=1e-5, atol=1e-5)
    assert not g1[7].any() and not want[7].any()
    untouched = np.setdiff1d(np.arange(m), cols)
    assert len(untouched) and not g1[torch.as_tensor(untouched, device="cuda")].any()


def test_backward_exact_on_integer_gradients(env):
    """gs = grad_out / deg is an integer when grad_out is deg times one: every sum is exact, through a column of more than
    three chunks of entries"""
    m, D = 50, 8
    lens = [1, 3, 0, 800, 4, 300, 2]
    indptr, cols = _adjacency(m, lens, seed=2)
    cols[indptr[3]:indptr[3] + 700] = 5                         # column 5: 700 entries of row 3 and more
    cols[indptr[5]:indptr[6]] = 5
    adj = (torch.as_tensor(indptr, device="cuda"), torch.as_tensor(cols, device="cuda"))
    rng = np.random.RandomState(3)
    q = rng.randint(-4, 5, size=(len(lens), D)).astype(np.float64)
    go = torch.as_tensor(q * np.maximum(np.diff(indptr), 1)[:, None], dtype=torch.float32, device="cuda")
    want = np.zeros((m, D))
    for i in range(len(lens)):
        for k in range(indptr[i], indptr[i + 1]):
            want[cols[k]] += q[i]
    got = _grad(_x(m, D), adj, go).cpu().numpy()
    assert (np.sum(cols == 5)) > 3 * K
    np.testing.assert_array_equal(got, want.astype(np.float32))


# ---------------------------------------------------------------------------- encoders
def _encoder(cls, aggregator, layers, use_residual, fused, **kw):
    torch.manual_seed(0)
    return cls([[0]] * layers, 8, aggregator, feature_idx=["feat0", "feat1"], feature_dim=[5, 12], max_id=N_NODES + 1,
               use_id=True, sparse_feature_idx=["u64_0"], sparse_feature_max_id=[40], embedding_dim=[6, 3],
               use_residual=use_residual, head_num=2, fused=fused, device="cuda", **kw)


def _f64_copy(model):
    """a float64 copy of model with every fused flag off"""
    ref = copy.deepcopy(model).double()
    for mod in ref.modules():
        if hasattr(mod, "fused"):
            mod.fused = False
    return ref


def _f64_features(monkeypatch):
    """get_dense_feature hands out float64 rows from here on (the float64 copy's composition reads them)"""
    from euler_b200 import ops
    real = ops.get_dense_feature
    monkeypatch.setattr(ops, "get_dense_feature", lambda *a, **k: [t.double() for t in real(*a, **k)])


def _close(a, b, what):
    a, b = a.double(), b.double()
    assert (a - b).abs().max() <= 1e-5 * max(b.abs().max(), 1e-3), what


@pytest.mark.parametrize("use_residual", (False, True))
@pytest.mark.parametrize("layers", (1, 2))
@pytest.mark.parametrize("aggregator", ("gcn", "mean", "attention"))
def test_gcn_encoder_fused_matches_the_f64_composition(env, monkeypatch, aggregator, layers, use_residual):
    from euler_b200.encoders import GCNEncoder
    seeds = torch.as_tensor(env["g"]["ids"][:96].astype(np.int64).reshape(32, 3), device="cuda")
    enc = _encoder(GCNEncoder, aggregator, layers, use_residual, True)
    ref = _f64_copy(enc)
    out = enc(seeds)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).cuda()
    (out * w).sum().backward()
    _f64_features(monkeypatch)
    want = ref(seeds)
    (want * w.double()).sum().backward()
    assert out.shape == (32, 3, 8) and out.dtype == torch.float32 and want.dtype == torch.float64
    _close(out, want, "forward")
    got, exp = dict(enc.named_parameters()), dict(ref.named_parameters())
    assert got.keys() == exp.keys()
    for n, p in got.items():
        assert p.grad is not None, n
        _close(p.grad, exp[n].grad, n)


def test_adjacency_mean_is_the_aggregators_mean_on_real_hops(env):
    """adjacency_mean over get_multi_hop_neighbor's hop 1 against its float32 restatement, bit for bit"""
    import euler_b200
    nodes, adjs = euler_b200.get_multi_hop_neighbor(env["g"]["ids"][:200].astype(np.int64), [[0], [0]])
    indptr, cols, _ = adjs[1]
    x = _x(nodes[2].numel(), 16)
    got = euler_b200.adjacency_mean(x, adjs[1])
    assert got.shape == (nodes[1].numel(), 16) and cols.numel() > 0
    assert got.cpu().numpy().tobytes() == _restated(x.cpu().numpy(), indptr.cpu().numpy(), cols.cpu().numpy()).tobytes()


def test_geniepath_step_fused_against_f64(env, monkeypatch):
    from euler_b200.supervised import GeniePath
    seeds = torch.as_tensor(env["g"]["ids"][:64].astype(np.int64), device="cuda")
    torch.manual_seed(0)
    model = GeniePath(8, [[0], [0]], "feat2", 3, max_id=N_NODES + 1, feature_idx=["feat0", "feat1"], feature_dim=[5, 12],
                      use_id=True, head_num=2, device="cuda")
    ref = _f64_copy(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.5)
    emb, loss, name, metric = model(seeds)
    opt.zero_grad()
    loss.backward()
    _f64_features(monkeypatch)
    emb64, loss64, _, _ = ref(seeds)
    loss64.backward()
    assert emb.shape == (64, 8) and name == "f1" and 0 <= float(metric) <= 1
    _close(emb, emb64, "embedding")
    assert abs(float(loss) - float(loss64)) <= 1e-5 * abs(float(loss64))
    for (n, p), (_, q) in zip(model.named_parameters(), ref.named_parameters()):
        if q.grad is None:                                   # outputs[:, 0, :]: the aggregators never reach the loss
            assert p.grad is None, n
            continue
        _close(p.grad, q.grad, n)
    before = [p.detach().clone() for p in model.parameters()]
    opt.step()
    assert any(not torch.equal(a, b) for a, b in zip(before, model.parameters()))
