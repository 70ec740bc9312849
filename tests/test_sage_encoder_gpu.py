"""GPU: ShallowEncoder's rows pooled per fanout segment (ops.shallow_encode_pool, eu_shallow_encode_pool and its backward
passes) against a fixed-order restatement over shallow_encode's rows and against float64; SageEncoder / ShuffleSageEncoder
with the pooled deepest hop against the literal composition; one supervised and one DGI training step."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import embedding_reference as er

pytestmark = pytest.mark.gpu

N_NODES, N_ROWS, N_ID = 600, 1000, 1000   # graph ids 1 .. 600; slot tables of N_ROWS rows; id table of N_ID rows
SLOT_DIMS = (5, 12, 3)                     # the dense slots feat0, feat1, feat2
ABSENT = (0, 650, 999)                     # ids the graph does not hold, all inside the id table; 999 is the default_node
COUNTS = (1, 2, 5, 10, 25, 64)
M = 3200                                   # divisible by every count
DENSE = [("feat0", 8), ("feat1", 7), ("feat2", 3), (99, 2)]   # padded, clipped, as stored, an unknown slot


def _lens_mixed(rng, n):   # 0 (default), 1, ordinary, and a few bags of more than 256 values
    k = rng.choice([0, 1, 2, 3, 5, 9], size=n, p=[0.3, 0.2, 0.2, 0.15, 0.1, 0.05])
    k[rng.choice(n, size=3, replace=False)] = [257, 300, 700]
    return k


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = er.slot_graph(5, N_NODES, [_lens_mixed, lambda rng, n: rng.randint(1, 4, size=n)],
                      [lambda rng, k: rng.randint(0, N_ROWS - 1, size=k), lambda rng, k: rng.randint(0, 50, size=k)],
                      feat_dim=sum(SLOT_DIMS))
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=list(SLOT_DIMS),
                                   u64_ptr=g["u64_ptr"], u64_val=g["u64_val"], n_u64_slots=g["S"])
    rng = np.random.RandomState(2)
    nodes = g["ids"][rng.randint(0, N_NODES, size=M)].astype(np.int64)
    nodes[rng.choice(M, size=300, replace=False)] = rng.choice(ABSENT, size=300)   # absent nodes and default_node rows
    nodes[64:128] = 999                                                            # whole segments of the default node
    nodes[:N_NODES] = g["ids"]                                                     # every node, the long bags included
    return dict(g=g, gr=gr, nodes=nodes)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)


def _table(n_rows, dim, seed=3, offset=0):
    """a table whose data pointer is `offset` floats past a 16-byte boundary"""
    t = torch.randn(n_rows * dim + offset, generator=torch.Generator().manual_seed(seed)).cuda()
    return t[offset:].view(n_rows, dim)


def _inputs(dim, off=0, combiners=("sum", "mean")):
    id_table = _table(N_ID, dim, seed=1, offset=off)
    sparse = [("u64_0", _table(N_ROWS, dim, seed=2, offset=off), N_ROWS - 1, combiners[0]),
              ("u64_1", _table(60, dim, seed=3, offset=off), 55, combiners[1]),
              ("no_such_slot", _table(20, dim, seed=4), 7, "sum")]
    return id_table, sparse


def _check_forward(nodes, count, id_table, dense, sparse, what):
    import euler_b200
    rows = euler_b200.shallow_encode(nodes, id_table, dense, sparse, "concat")
    for pool in ("sum", "mean"):
        out = euler_b200.shallow_encode_pool(nodes, count, id_table, dense, sparse, pool)
        want = er.pool_f32(rows, count, pool)
        assert out.shape == want.shape and out.dtype == torch.float32
        assert out.cpu().numpy().tobytes() == want.tobytes(), (what, count, pool)
    mean = rows.view(-1, count, rows.shape[1]).mean(1)
    mag = rows.abs().view(-1, count, rows.shape[1]).mean(1)
    assert ((out - mean).abs() <= 1e-6 * mag + 1e-7).all(), (what, count)


@pytest.mark.parametrize("dim", (1, 3, 4, 16, 128))
def test_pool_forward_bit_exact(env, dim):
    nodes = env["nodes"]
    for off in (0, 1):   # aligned and unaligned tables (and, for dim 1 and 3, unaligned slot columns in the output)
        id_table, sparse = _inputs(dim, off)
        for count in COUNTS:
            for dense in (DENSE, DENSE[:1], []):
                _check_forward(nodes, count, id_table, dense, sparse, (dim, off, len(dense)))


@pytest.mark.parametrize("dim", (4, 5))
def test_pool_forward_every_subset_of_inputs(env, dim):
    nodes = env["nodes"]
    id_table, sparse = _inputs(dim, combiners=("sqrtn", "mean"))
    for use_id, use_dense, use_sparse in itertools.product((False, True), repeat=3):
        if not (use_id or use_dense or use_sparse):
            continue
        for count in (1, 10, 64):
            _check_forward(nodes, count, id_table if use_id else None, DENSE if use_dense else [], sparse if use_sparse else [],
                           (use_id, use_dense, use_sparse))


def test_pool_count_one_is_the_row_and_empty_batch(env):
    import euler_b200
    nodes = env["nodes"]
    id_table, sparse = _inputs(16)
    rows = euler_b200.shallow_encode(nodes, id_table, DENSE, sparse, "concat")
    for pool in ("sum", "mean"):
        assert torch.equal(euler_b200.shallow_encode_pool(nodes, 1, id_table, DENSE, sparse, pool), rows)
        assert euler_b200.shallow_encode_pool([], 10, id_table, DENSE, sparse, pool).shape == (0, 16 + 20 + 48)
    out = euler_b200.shallow_encode_pool([999] * 20, 10, None, DENSE, [sparse[0]], "mean")   # default_node rows: rows like any other
    assert not out[:, :20].any()
    torch.testing.assert_close(out[:, 20:], sparse[0][1][N_ROWS - 1].expand(2, 16), rtol=1e-6, atol=0)


def _raw(sym, p, *args):
    from euler_b200 import _lib, ops
    return getattr(_lib.load(), sym)(ops._ctx_on_stream()._h, C.byref(p), *args)


def test_raw_abi_unaligned_output_and_statuses(env):
    """the C entry point with an out pointer 4 bytes past a 16-byte boundary gives the same bits; the refusals' statuses"""
    import euler_b200
    from euler_b200 import _lib
    nodes = torch.as_tensor(env["nodes"], device="cuda")
    id_table, sparse = _inputs(16)
    dense = DENSE[:2]
    p = er.shallow_problem(nodes, id_table, dense, sparse)
    W = 16 + 15 + 3 * 16
    buf = torch.empty(M // 10 * W + 1, device="cuda")
    assert _raw("eu_shallow_encode_pool", p, 10, 1, buf.data_ptr() + 4) == 0
    want = euler_b200.shallow_encode_pool(nodes, 10, id_table, dense, sparse, "mean")
    assert buf[1:].cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
    out = torch.empty(M * W, device="cuda")
    INVALID, UNSUPPORTED = 1, 4
    assert _raw("eu_shallow_encode_pool", p, 0, 1, out.data_ptr()) == INVALID
    assert _raw("eu_shallow_encode_pool", p, -3, 1, out.data_ptr()) == INVALID
    assert _raw("eu_shallow_encode_pool", p, 3, 1, out.data_ptr()) == INVALID          # 3200 % 3 != 0
    assert _raw("eu_shallow_encode_pool", p, 10, 2, out.data_ptr()) == INVALID         # no such pool
    assert _raw("eu_shallow_encode_pool", p, 10, 1, None) == INVALID
    assert _raw("eu_shallow_encode_pool", p, 640, 1, out.data_ptr()) == UNSUPPORTED    # beyond EU_SHALLOW_POOL_MAX_COUNT
    assert _lib.SHALLOW_POOL_MAX_COUNT == 512
    p_add = er.shallow_problem(nodes, id_table, [], sparse, comb=1)
    assert _raw("eu_shallow_encode_pool", p_add, 10, 1, out.data_ptr()) == UNSUPPORTED
    grads = (C.c_void_p * 4)(*[torch.empty_like(t).data_ptr() for t in [id_table] + [s[1] for s in sparse]])
    assert _raw("eu_shallow_encode_pool_backward", p, 3, 1, out.data_ptr(), grads) == INVALID
    assert _raw("eu_shallow_encode_pool_backward", p_add, 10, 1, out.data_ptr(), grads) == UNSUPPORTED


def test_bad_inputs_raise(env):
    import euler_b200
    nodes = env["nodes"]
    id_table, sparse = _inputs(4)
    with pytest.raises(euler_b200.EulerError, match="id table"):
        euler_b200.shallow_encode_pool(nodes, 10, id_table[:600], [], sparse)   # ids 650 and 999 lie outside
    with pytest.raises(euler_b200.EulerError, match="id table"):
        euler_b200.shallow_encode_pool([-1, 5], 2, id_table, [], [])
    with pytest.raises(euler_b200.EulerError, match="outside the table"):
        euler_b200.shallow_encode_pool(nodes, 10, None, [], [("u64_0", _table(500, 4), 0)])   # slot 0 holds values up to 998
    for dv in (60, -1):
        with pytest.raises(euler_b200.EulerError, match="default_value"):
            euler_b200.shallow_encode_pool(nodes, 10, None, [], [("u64_1", _table(60, 4), dv)])
    with pytest.raises(euler_b200.EulerError, match="pool"):
        euler_b200.shallow_encode_pool(nodes, 10, id_table, [], [], pool="max")
    for count in (0, -1, 3, 640):
        with pytest.raises(euler_b200.EulerError, match="count|segments"):
            euler_b200.shallow_encode_pool(nodes, count, id_table, [], sparse)


def test_forward_captures_in_a_cuda_graph(env):
    import euler_b200
    nodes = torch.as_tensor(env["nodes"], device="cuda")
    id_table, sparse = _inputs(16)
    eager = euler_b200.shallow_encode_pool(nodes, 10, id_table, DENSE, sparse, "mean")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        euler_b200.shallow_encode_pool(nodes, 10, id_table, DENSE, sparse, "mean")
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = euler_b200.shallow_encode_pool(nodes, 10, id_table, DENSE, sparse, "mean")
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    cg.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == eager.cpu().numpy().tobytes()


# ---------------------------------------------------------------------------- gradients
def _leaves(id_table, sparse):
    leaves = [id_table.detach().clone().requires_grad_(True)] + [t.detach().clone().requires_grad_(True) for _, t, _, _ in sparse]
    return leaves, [(n, leaf, dv, c) for (n, _, dv, c), leaf in zip(sparse, leaves[1:])]


def _pool_grads(nodes, count, pool, id_table, sparse, grad, sparse_grad=False):
    import euler_b200
    leaves, sp = _leaves(id_table, sparse)
    out = euler_b200.shallow_encode_pool(nodes, count, leaves[0], DENSE, sp, pool, sparse_grad=sparse_grad)
    return torch.autograd.grad(out, leaves, grad)


def _composed_grads(nodes, count, pool, id_table, sparse, grad):
    import euler_b200
    leaves, sp = _leaves(id_table, sparse)
    rows = euler_b200.shallow_encode(nodes, leaves[0], DENSE, sp, "concat").view(-1, count, grad.shape[1])
    return torch.autograd.grad(rows.mean(1) if pool == "mean" else rows.sum(1), leaves, grad)


def _want_grads(env, nodes, count, pool, id_table, sparse, grad):
    """float64 gradients of every table, and the sums of the terms' magnitudes"""
    import euler_b200
    g = env["g"]
    gn = np.repeat(grad.cpu().double().numpy(), count, axis=0) / (count if pool == "mean" else 1)
    dims = [id_table.shape[1]] + [t.shape[1] for _, t, _, _ in sparse]
    cols, c0 = [], 0
    for j, d in enumerate(dims):
        cols.append(slice(c0, c0 + d))
        c0 += d + (20 if j == 0 else 0)   # the dense columns follow the id columns
    w, m = np.zeros((N_ID, dims[0])), np.zeros((N_ID, dims[0]))
    np.add.at(w, nodes, gn[:, cols[0]])
    np.add.at(m, nodes, np.abs(gn[:, cols[0]]))
    want, mag = [w], [m]
    for k, (n, t, dv, c) in enumerate(sparse):
        bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, euler_b200.get_graph().sparse_feature_id(n), dv)
        want.append(er.grad_f64(gn[:, cols[k + 1]], bl, t.shape[0], c))
        mag.append(er.grad_f64(np.abs(gn[:, cols[k + 1]]), bl, t.shape[0], c))
    return want, mag


@pytest.mark.parametrize("pool", ("sum", "mean"))
@pytest.mark.parametrize("dim,count", [(3, 5), (16, 10), (128, 2), (16, 64)])
def test_gradients_f64_composition_run_to_run_untouched_and_sparse(env, dim, count, pool):
    nodes = env["nodes"]
    id_table, sparse = _inputs(dim, combiners=("mean", "sqrtn"))
    grad = torch.randn(M // count, 4 * dim + 20, generator=torch.Generator().manual_seed(9)).cuda()
    g1 = _pool_grads(nodes, count, pool, id_table, sparse, grad)
    g2 = _pool_grads(nodes, count, pool, id_table, sparse, grad)
    gs = _pool_grads(nodes, count, pool, id_table, sparse, grad, sparse_grad=True)
    gc = _composed_grads(nodes, count, pool, id_table, sparse, grad)
    want, mag = _want_grads(env, nodes, count, pool, id_table, sparse, grad)
    for t in range(len(g1)):
        assert torch.equal(g1[t], g2[t]), t
        got = g1[t].cpu().numpy()
        err = np.abs(got - want[t])
        assert (err <= 1e-5 * mag[t] + 1e-7).all(), (t, float((err / (mag[t] + 1e-30)).max()))
        assert (np.abs(got - gc[t].cpu().numpy()) <= 1e-5 * mag[t] + 1e-7).all(), t
        assert not got[mag[t].sum(1) == 0].any()   # rows no entry names are exactly zero
        s = gs[t]
        assert s.is_sparse and s.is_coalesced()
        assert np.array_equal(s.indices()[0].cpu().numpy(), np.flatnonzero(mag[t].sum(1) > 0))
        assert torch.equal(s.to_dense(), g1[t])


def test_node_repeated_many_times_is_exact(env):
    """one node in 20 480 positions, segments of 10, an integer gradient: every entry counted exactly, over many chunks"""
    import euler_b200
    node = int(env["g"]["ids"][7])
    nodes = np.full(20480, node, np.int64)
    id_t = torch.zeros(N_ID, 8, device="cuda", requires_grad=True)
    t = torch.zeros(60, 8, device="cuda", requires_grad=True)
    out = euler_b200.shallow_encode_pool(nodes, 10, id_t, [], [("u64_1", t, 55)], "sum")
    out.backward(torch.full_like(out, 3.0))
    assert id_t.grad[node, 0].item() == 3.0 * 20480 and id_t.grad.sum().item() == 3.0 * 20480 * 8
    bag = er.bags(env["g"]["ids"], env["g"]["u64_ptr"], env["g"]["u64_val"], env["g"]["S"], nodes[:1], 1, 55)[0]
    want = np.zeros(60)
    np.add.at(want, bag, 3.0 * 20480)
    assert np.array_equal(t.grad[:, 0].cpu().numpy(), want)


def _outside_torch():
    free, total = torch.cuda.mem_get_info()
    return total - free - torch.cuda.memory_reserved()


def test_forward_and_backward_never_hold_the_row_matrix(env):
    """M = 1.28M nodes at W = 16 + 128 columns: the [M, W] matrix is 737 MB, and the composition holds it twice (the rows
    and their gradient); forward + backward of the pooled op stay under half of one, torch's allocator peak and the growth of
    the library's scratch together"""
    import euler_b200
    rng = np.random.RandomState(3)
    count, Mbig = 10, 1_280_000
    nodes = torch.as_tensor(env["g"]["ids"][rng.randint(0, N_NODES, size=Mbig)].astype(np.int64), device="cuda")
    t = torch.zeros(60, 16, device="cuda", requires_grad=True)
    dense = [("feat1", 128)]
    matrix = Mbig * (16 + 128) * 4
    euler_b200.shallow_encode_pool(nodes[:100], count, None, dense, [("u64_1", t, 55)], "mean").sum().backward()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base, outside = torch.cuda.memory_allocated(), _outside_torch()
    torch.cuda.reset_peak_memory_stats()
    out = euler_b200.shallow_encode_pool(nodes, count, None, dense, [("u64_1", t, 55)], "mean")
    out.backward(torch.ones_like(out))
    torch.cuda.synchronize()
    used = torch.cuda.max_memory_allocated() - base + max(0, _outside_torch() - outside)
    assert used < matrix / 2, (used, matrix)


# ---------------------------------------------------------------------------- SageEncoder
METAPATH = {1: [[0]], 2: [[0], [0]]}
FANOUTS = {1: [10], 2: [3, 5]}


def _encoder(cls, aggregator, layers, concat, fused, sparse_grad=False, **kw):
    torch.manual_seed(0)
    return cls(METAPATH[layers], FANOUTS[layers], 6, aggregator=aggregator, concat=concat, feature_idx=["feat0", "feat1"],
               feature_dim=[8, 7], max_id=N_ID - 2, use_id=True, sparse_feature_idx=["u64_0", "u64_1"],
               sparse_feature_max_id=[N_ROWS - 2, 58], embedding_dim=[8, 8, 4], fused=fused, sparse_grad=sparse_grad, device="cuda", **kw)


def _count_pool_calls(monkeypatch):
    from euler_b200 import ops
    calls = []
    real = ops.shallow_encode_pool

    def wrapper(*a, **k):
        calls.append(a[1])
        return real(*a, **k)
    monkeypatch.setattr(ops, "shallow_encode_pool", wrapper)
    return calls


@pytest.mark.parametrize("concat", (False, True))
@pytest.mark.parametrize("layers", (1, 2))
@pytest.mark.parametrize("aggregator", ("mean", "gcn", "meanpool", "maxpool"))
def test_sage_encoder_fused_matches_the_composition(env, monkeypatch, aggregator, layers, concat):
    import euler_b200
    from euler_b200.encoders import SageEncoder
    calls = _count_pool_calls(monkeypatch)
    seeds = torch.as_tensor(env["g"]["ids"][:96].astype(np.int64).reshape(32, 3), device="cuda")
    res = {}
    for fused in (True, False):
        enc = _encoder(SageEncoder, aggregator, layers, concat, fused)
        assert enc.dims == [35] + [6] * layers
        euler_b200.seed(11)
        out = enc(seeds)
        assert out.shape == (32, 3, 6)
        out.square().sum().backward()
        res[fused] = (out.detach(), {n: p.grad.clone() for n, p in enc.named_parameters()})
        if fused:
            assert calls == ([FANOUTS[layers][-1]] if aggregator in ("mean", "gcn") else [])   # the pool aggregators compose
    assert len(calls) <= 1                                                                     # fused=False never pools
    torch.testing.assert_close(res[True][0], res[False][0], rtol=1e-5, atol=1e-6)
    assert res[True][1].keys() == res[False][1].keys()
    for n, a in res[True][1].items():
        b = res[False][1][n]
        assert (a - b).abs().max() <= 1e-5 * b.abs().max() + 1e-9, n


def test_shared_add_encoder_takes_the_composition(env, monkeypatch):
    import euler_b200
    from euler_b200.encoders import SageEncoder, ShallowEncoder
    calls = _count_pool_calls(monkeypatch)
    seeds = torch.as_tensor(env["g"]["ids"][:32].astype(np.int64), device="cuda")
    for kw in (dict(combiner="add", dim=8), dict(combiner="concat", dim=8)):
        torch.manual_seed(0)
        shared = ShallowEncoder(feature_idx=["feat0"], feature_dim=[8], max_id=N_ID - 2, sparse_feature_idx=["u64_1"],
                                sparse_feature_max_id=[58], embedding_dim=8, device="cuda", **kw)
        enc = SageEncoder(METAPATH[2], FANOUTS[2], 6, max_id=N_ID - 2, shared_node_encoder=shared, device="cuda")
        assert enc.dims == [8, 6, 6] and enc(seeds).shape == (32, 6)
    assert calls == []


def _f64(t):
    return t.detach().double().cpu().numpy()


def _encode_f64(enc, env, nodes):
    """ShallowEncoder's 'concat' row in float64 from the encoder's parameters and the graph's arrays"""
    g, sh = env["g"], enc._node_encoder
    nodes = np.asarray(nodes)
    parts = [_f64(sh.embedding.embeddings)[nodes]]
    row = {int(i): r for r, i in enumerate(g["ids"])}
    off = np.concatenate([[0], np.cumsum(SLOT_DIMS)])
    for name, d in zip(sh.feature_idx, sh.feature_dim):
        s = int(name[4:])
        f = np.zeros((len(nodes), d))
        k = min(d, SLOT_DIMS[s])
        for i, n in enumerate(nodes):
            if int(n) in row:
                f[i, :k] = g["feat"][row[int(n)], off[s]:off[s] + k]
        parts.append(f)
    for s, (m, e) in enumerate(zip(sh.sparse_feature_max_id, sh.sparse_embeddings)):
        bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, s, m + 1)
        parts.append(er.lookup_f64(_f64(e.embeddings), bl, "sum"))
    return np.concatenate(parts, 1)


def _sage_f64(enc, env, samples):
    """SageEncoder.call's loop with the mean aggregator in float64"""
    hidden = [_encode_f64(enc, env, s.cpu().numpy()) for s in samples]
    L = enc.num_layers
    for layer in range(L):
        a = enc.aggregators[layer]
        nxt = []
        for hop in range(L - layer):
            neigh = hidden[hop + 1].reshape(-1, enc.fanouts[hop], enc.dims[layer]).mean(1)
            act = (lambda v: np.maximum(v, 0)) if layer < L - 1 else (lambda v: v)   # Dense's own activation, per term
            nxt.append(act(hidden[hop] @ _f64(a.self_layer.kernel)) + act(neigh @ _f64(a.neigh_layer.kernel)))
        hidden = nxt
    return hidden[0]


def test_supervised_step_fused_composed_and_f64(env):
    """SuperviseModel over SageEncoder, one SGD step: loss and updated tables, fused vs fused=False vs float64"""
    import euler_b200
    from euler_b200.encoders import SageEncoder
    from euler_b200.supervised import SuperviseModel

    class SupervisedGraphSage(SuperviseModel):
        def __init__(self, fused, sparse_grad):
            super().__init__("feat2", 3, dim=6, device="cuda")
            self.encoder = _encoder(SageEncoder, "mean", 2, False, fused, sparse_grad)

        def embed(self, n_id):
            return self.encoder(n_id)

    seeds = torch.as_tensor(env["g"]["ids"][:64].astype(np.int64), device="cuda")

    def step(fused, sparse_grad=False):
        torch.manual_seed(0)
        model = SupervisedGraphSage(fused, sparse_grad)
        euler_b200.seed(5)
        samples = model.encoder.sample(seeds)
        logit = _sage_f64(model.encoder, env, samples) @ _f64(model.out_fc.weight).T
        label = _f64(euler_b200.get_dense_feature(seeds, ["feat2"], [3])[0])
        loss64 = np.mean(np.maximum(logit, 0) - logit * label + np.log1p(np.exp(-np.abs(logit))))
        euler_b200.seed(5)
        opt = torch.optim.SGD(model.parameters(), lr=0.5)
        emb, loss, name, metric = model(seeds)
        assert emb.shape == (64, 6) and name == "f1" and 0 <= float(metric) <= 1
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss.detach(), loss64, [p.detach().clone() for p in model.parameters()]

    loss_c, loss64, p_c = step(False)
    assert abs(float(loss_c) - loss64) <= 1e-5 * abs(loss64)
    for sparse_grad in (False, True):
        loss_f, _, p_f = step(True, sparse_grad)
        assert abs(float(loss_f) - loss64) <= 1e-5 * abs(loss64)
        for a, b in zip(p_f, p_c):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def test_dgi_step_fused_composed_and_f64(env):
    """one DGI step with a fixed generator: loss and updated tables, fused vs fused=False; the loss against float64"""
    import euler_b200
    from euler_b200.unsupervised import DGI
    seeds = torch.as_tensor(env["g"]["ids"][:64].astype(np.int64), device="cuda")

    def step(fused):
        torch.manual_seed(0)
        model = DGI(0, [0], N_ID - 2, METAPATH[2], FANOUTS[2], 6, feature_idx=["feat0", "feat1"], feature_dim=[8, 7], use_id=True,
                    sparse_feature_idx=["u64_0", "u64_1"], sparse_feature_max_id=[N_ROWS - 2, 58], embedding_dim=[8, 8, 4],
                    fused=fused, device="cuda")
        enc = model._target_encoder
        euler_b200.seed(5)
        samples = enc.sample(seeds.unsqueeze(-1))
        shuffled = enc.shuffle_samples(samples, torch.Generator().manual_seed(3))
        h, h_neg = _sage_f64(enc, env, samples), _sage_f64(enc, env, shuffled)
        read = 1 / (1 + np.exp(-h.mean(0)))
        k = _f64(model.kernel.kernel)
        lg, nlg = (h @ k) @ read, (h_neg @ k) @ read
        xent = lambda x, z: np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))   # noqa: E731
        loss64 = np.concatenate([xent(lg, 1), xent(nlg, 0)]).mean()
        euler_b200.seed(5)
        opt = torch.optim.SGD(model.parameters(), lr=0.5)
        emb, loss, name, metric = model(seeds, torch.Generator().manual_seed(3))
        assert emb.shape == (64, 6) and name == "mrr" and 0 < float(metric) <= 1
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss.detach(), loss64, [p.detach().clone() for p in model.parameters()]

    loss_c, loss64, p_c = step(False)
    loss_f, _, p_f = step(True)
    assert abs(float(loss_c) - loss64) <= 1e-5 * abs(loss64) and abs(float(loss_f) - loss64) <= 1e-5 * abs(loss64)
    for a, b in zip(p_f, p_c):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
