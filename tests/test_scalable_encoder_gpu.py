"""GPU: the embedding-store ops (ops.store_exchange / store_accumulate, eu_store_exchange / eu_store_accumulate) bit for bit
against restatements of their documented meaning and order, their refusals and CUDA-graph replay; ScalableSageEncoder /
ScalableGCNEncoder's fused steps against the float64 composition, and run to run."""
import numpy as np
import pytest
import torch

import graphs

pytestmark = pytest.mark.gpu

N_NODES = 400   # graph ids 1 .. 400: the encoders' max_id, so their stores have 402 rows


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = graphs.random_graph(seed=5, n=N_NODES, T=1, avg_deg=6, feat_dim=8, hub=150)
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=1, node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=[8])
    return dict(g=g, gr=gr)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)


def _table(n_rows, dim, seed, offset=0):
    """a random table whose data pointer is `offset` floats past a 16-byte boundary"""
    t = torch.randn(n_rows * dim + offset, generator=torch.Generator().manual_seed(seed)).cuda()
    return t[offset:].view(n_rows, dim)


def _bits(t):
    return t.detach().cpu().numpy().view(np.int32)


def _ids(n_rows, M, seed):
    """ids with repeats: random ones, one id 50 times through the list, and a run of one id"""
    rng = np.random.RandomState(seed)
    ids = rng.randint(0, n_rows, size=M)
    if M >= 200:
        ids[rng.choice(M, size=50, replace=False)] = 7
        ids[100:140] = n_rows - 1
    return torch.as_tensor(ids, dtype=torch.int64, device="cuda")


# ---------------------------------------------------------------------------- exchange
def _exchange_want(S, G, ids, rows):
    S, G = S.copy(), G.copy()
    taken = G[ids].copy()
    for i, v in enumerate(ids):
        S[v] = rows[i]              # the last occurrence wins
    G[ids] = 0
    return S, G, taken


@pytest.mark.parametrize("offset", (0, 1))
@pytest.mark.parametrize("dim", (1, 3, 4, 16, 128, 200))
def test_exchange_bits(env, dim, offset):
    import euler_b200
    n_rows, M = 500, 3000
    store, grad_store = _table(n_rows, dim, 1, offset), _table(n_rows, dim, 2, offset)
    rows, ids = _table(M, dim, 3, offset), _ids(n_rows, M, 4)
    want = _exchange_want(store.cpu().numpy(), grad_store.cpu().numpy(), ids.cpu().numpy(), rows.cpu().numpy())
    taken = euler_b200.store_exchange(store, grad_store, ids, rows)
    for got, w in zip((store, grad_store, taken), want):
        assert np.array_equal(_bits(got), w.view(np.int32))   # untouched rows included
    empty = torch.zeros(0, dtype=torch.int64, device="cuda")
    before = store.clone(), grad_store.clone()
    assert euler_b200.store_exchange(store, grad_store, empty, rows[:0]).shape == (0, dim)
    assert torch.equal(store, before[0]) and torch.equal(grad_store, before[1])


def test_exchange_and_accumulate_refuse_bad_ids_untouched(env):
    import euler_b200
    store, grad_store, rows = _table(50, 8, 1), _table(50, 8, 2), _table(4, 8, 3)
    before = store.clone(), grad_store.clone()
    for bad in (-1, 50):
        ids = torch.as_tensor([3, bad, 3, 9], device="cuda")
        with pytest.raises(euler_b200.EulerError, match="outside"):
            euler_b200.store_exchange(store, grad_store, ids, rows)
        with pytest.raises(euler_b200.EulerError, match="outside"):
            euler_b200.store_accumulate(grad_store, ids, rows)
        assert torch.equal(store, before[0]) and torch.equal(grad_store, before[1])
    with pytest.raises(euler_b200.EulerError, match="count"):
        euler_b200.store_accumulate(grad_store, torch.arange(4, device="cuda"), rows[:1], count=3)
    with pytest.raises(euler_b200.EulerError, match="float32"):
        euler_b200.store_exchange(store.double(), grad_store, torch.arange(4, device="cuda"), rows)
    with pytest.raises(euler_b200.EulerError, match="contiguous"):
        euler_b200.store_accumulate(grad_store.t(), torch.arange(4, device="cuda"), rows)


def _replays(call, tables, args):
    """call(*tables, *args) eagerly and as a CUDA-graph replay from the same starting tables: (eager, replayed) outputs"""
    start = [t.clone() for t in tables]
    eager_out = call(*tables, *args)
    eager = [t.clone() for t in tables] + ([eager_out.clone()] if eager_out is not None else [])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(*tables, *args)                        # sizes the scratch outside the capture
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = call(*tables, *args)
    torch.cuda.current_stream().wait_stream(s)
    for t, s0 in zip(tables, start):
        t.copy_(s0)
    cg.replay()
    torch.cuda.synchronize()
    return eager, [t.clone() for t in tables] + ([out] if out is not None else [])


def test_exchange_and_accumulate_capture(env):
    import euler_b200
    ids = _ids(300, 2000, 5)
    eager, replayed = _replays(euler_b200.store_exchange, [_table(300, 16, 1), _table(300, 16, 2)], (ids, _table(2000, 16, 3)))
    assert all(torch.equal(a, b) for a, b in zip(eager, replayed))
    eager, replayed = _replays(euler_b200.store_accumulate, [_table(300, 16, 2)], (ids, _table(200, 16, 3), 10, "mean"))
    assert all(torch.equal(a, b) for a, b in zip(eager, replayed))


# ---------------------------------------------------------------------------- accumulate
def _accumulate_f32(old, ids, grad, count, pool):
    """the documented order in float32: each id's entries in input order, chunks of 256 from +0, the chunk sums in chunk
    order from +0, then one add to the stored row"""
    out = old.copy()
    entries = {}
    for e, v in enumerate(ids):
        entries.setdefault(v, []).append(e)
    c = np.float32(count)
    for v, es in entries.items():
        sums = []
        for k in range(0, len(es), 256):
            acc = np.zeros(old.shape[1], np.float32)
            for e in es[k:k + 256]:
                x = grad[e // count]
                acc = acc + (x / c if pool == "mean" else x)
            sums.append(acc)
        total = sums[0]
        if len(sums) > 1:
            total = np.zeros(old.shape[1], np.float32)
            for s in sums:
                total = total + s
        out[v] = old[v] + total
    return out


@pytest.mark.parametrize("pool", ("sum", "mean"))
@pytest.mark.parametrize("count", (1, 2, 10, 25))
@pytest.mark.parametrize("dim,offset", [(16, 0), (3, 0), (128, 1)])
def test_accumulate_bits(env, count, pool, dim, offset):
    import euler_b200
    n_rows, R = 600, 240
    ids = _ids(n_rows, R * count, 6)
    grad, old = _table(R, dim, 7, offset), _table(n_rows, dim, 8, offset)
    grad_store = old.clone()
    euler_b200.store_accumulate(grad_store, ids, grad, count, pool)
    again = old.clone()
    euler_b200.store_accumulate(again, ids, grad, count, pool)
    assert torch.equal(grad_store, again)                                   # run to run
    want = _accumulate_f32(old.cpu().numpy(), ids.cpu().numpy(), grad.cpu().numpy(), count, pool)
    assert np.array_equal(_bits(grad_store), want.view(np.int32))          # untouched rows included
    # the gradient of shallow_encode_pool over the store, as its sparse backward gives it, added once
    leaf = old.clone().requires_grad_()
    g, = torch.autograd.grad(euler_b200.shallow_encode_pool(ids, count, id_table=leaf, pool=pool, sparse_grad=True), leaf, grad)
    via = old.clone()
    via[g.indices()[0]] = old[g.indices()[0]] + g.values()
    assert torch.equal(grad_store, via)


def test_accumulate_one_id_many_times_is_exact(env):
    import euler_b200
    ids = torch.full((20480,), 11, dtype=torch.int64, device="cuda")
    grad = torch.randint(-4, 5, (2048, 8), generator=torch.Generator().manual_seed(3)).float().cuda()
    grad_store = torch.ones(40, 8, device="cuda")
    euler_b200.store_accumulate(grad_store, ids, grad, 10, "sum")
    want = torch.ones(40, 8, device="cuda")
    want[11] += 10 * grad.double().sum(0).float()
    assert torch.equal(grad_store, want)


# ---------------------------------------------------------------------------- encoders
def _seeds(step):
    rng = np.random.RandomState(20 + step)
    s = rng.randint(1, N_NODES + 1, size=96)
    s[:8] = s[8:16]                                                 # repeated seeds
    return torch.as_tensor(s, dtype=torch.int64, device="cuda")


def _make(cls, fused, **kw):
    torch.manual_seed(0)
    return cls([0], **kw, feature_idx=["feat0"], feature_dim=[8], max_id=N_NODES, use_id=True, embedding_dim=8,
               store_learning_rate=0.01, store_init_maxval=0.5, fused=fused, device="cuda",
               generator=torch.Generator(device="cuda").manual_seed(1))


def _run(enc, double=False):
    """three training steps; returns every table and parameter"""
    import euler_b200
    if double:
        enc = enc.double()
    torch.manual_seed(4)
    head = (torch.randn(enc.dims[-1], 1) * 0.5).cuda().to(torch.float64 if double else torch.float32).requires_grad_()
    opt = torch.optim.SGD(list(enc.parameters()) + [head], lr=0.05)
    for step in range(3):
        euler_b200.seed(100 + step)
        out = enc(_seeds(step), training=True)
        enc.train_step(torch.tanh(out @ head).square().mean(), opt)
    return enc.stores + enc.gradient_stores + [p.detach() for p in enc.parameters()] + [head.detach()]


CASES = [("ScalableSageEncoder", dict(fanout=5, num_layers=2, dim=8, aggregator="mean")),
         ("ScalableSageEncoder", dict(fanout=5, num_layers=3, dim=8, aggregator="gcn")),
         ("ScalableSageEncoder", dict(fanout=4, num_layers=2, dim=8, aggregator="meanpool")),
         ("ScalableGCNEncoder", dict(num_layers=2, dim=8, aggregator="gcn")),
         ("ScalableGCNEncoder", dict(num_layers=3, dim=8, aggregator="attention", head_num=2))]


@pytest.mark.parametrize("name,kw", CASES)
def test_encoder_steps_fused_against_f64_and_run_to_run(env, name, kw):
    from euler_b200 import encoders
    cls = getattr(encoders, name)
    fused = _run(_make(cls, True, **kw))
    again = _run(_make(cls, True, **kw))
    assert all(torch.equal(a, b) for a, b in zip(fused, again))
    want = _run(_make(cls, False, **kw), double=True)
    assert len(fused) == len(want)
    assert any((g != 0).any() for g in fused[kw["num_layers"] - 1:2 * (kw["num_layers"] - 1)])   # gradients reached the stores
    for k, (a, b) in enumerate(zip(fused, want)):
        torch.testing.assert_close(a.double(), b, rtol=1e-5, atol=1e-5, msg=lambda m: "tensor %d: %s" % (k, m))


def test_sage_store_layers_take_the_pooled_op(env, monkeypatch):
    import euler_b200
    from euler_b200 import encoders, ops
    calls = []
    real = ops.shallow_encode_pool
    monkeypatch.setattr(ops, "shallow_encode_pool", lambda *a, **k: calls.append(a[1]) or real(*a, **k))
    enc = _make(encoders.ScalableSageEncoder, True, fanout=5, num_layers=3, dim=8, aggregator="mean")
    euler_b200.seed(3)
    enc(_seeds(0), training=True)
    assert calls == [5, 5, 5]        # hop 1's node rows, then stores 0 and 1
    assert enc.store_loss.requires_grad
