"""GPU: the fused skip-gram step (ops.skipgram_xent_loss: eu_skipgram_loss and its backward passes) against the numpy
restatements of skipgram_reference, against the torch composition, and through whole DeepWalk and LINE steps."""
import copy

import numpy as np
import pytest
import torch

import skipgram_reference as sr

pytestmark = pytest.mark.gpu

DIMS = (1, 3, 4, 16, 32, 64, 128, 200)
PK = ((1, 0), (1, 1), (1, 5), (3, 5), (3, 20))


@pytest.fixture(scope="module")
def graph():
    import euler_b200
    g = euler_b200.Graph.rmat(4096, 40000, seed=11)
    euler_b200.set_graph(g, rng="minstd", seed=1)
    return g


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("P,K", PK)
def test_forward_logits_ranks_bit_exact(graph, dim, P, K):
    rng = np.random.RandomState(dim * 31 + P * 7 + K)
    n_rows, B = 300, 257
    src, pos, negs = sr.pair_ids(rng, B, P, K, n_rows)
    ctx = sr.context_ids(pos, negs)
    for off in (0, 1):
        target, context = sr.device_table(n_rows, dim, rng, off), sr.device_table(n_rows, dim, rng, 3 - off)
        logits, rank, loss = sr.device_forward(src, pos, negs, target, context)
        tn, cn = target.cpu().numpy(), context.cpu().numpy()
        x = logits.cpu().numpy()
        head = sr.logits_f32(tn, cn, src[:24], ctx[:24])          # the fixed order, literally, on the first rows
        assert x[:24].tobytes() == head.tobytes(), (dim, P, K, off)
        assert x.tobytes() == sr.forward64(tn, cn, src, ctx, P)[0].astype(np.float32).tobytes()   # dyadic: every order is exact
        assert np.array_equal(rank.cpu().numpy(), sr.rank_top_k_literal(x[:, :P], x[:, P:]))
        ref = sr.loss64(sr.forward64(tn, cn, src, ctx, P)[0], P)
        assert abs(float(loss) - ref) <= 1e-6 * abs(ref)


@pytest.mark.parametrize("name", ["mrr", "hit1", "hit3", "hit10", "mr"])
def test_metrics_exact_with_ties(graph, name):
    import euler_b200
    rng = np.random.RandomState(4)
    n_rows, dim, P, K = 50, 4, 2, 20
    target = sr.device_table(n_rows, dim, rng)
    target[:, 1:] = 0
    target[:, 0] = torch.tensor(rng.randint(-2, 3, size=n_rows), dtype=torch.float32)   # logits in a handful of values
    src, pos, negs = sr.pair_ids(rng, 999, P, K, n_rows)
    loss, met = euler_b200.skipgram_xent_loss(src, pos, negs, target, target, metric=name)
    x = sr.device_forward(src, pos, negs, target, target)[0].cpu().numpy()
    rank = sr.rank_top_k_literal(x[:, :P], x[:, P:])
    assert len(np.unique(x)) <= 25 and (rank > 0).sum() > 100
    want = sr.metric(rank, name)
    assert (int(met) == want) if name == 'mr' else abs(float(met) - float(want)) <= 1e-6 * float(want)


def test_out_of_range_ids_raise(graph):
    import euler_b200
    rng = np.random.RandomState(1)
    t = sr.device_table(100, 8, rng)
    src, pos, negs = sr.pair_ids(rng, 64, 1, 5, 100)
    for which, bad in (("src", -1), ("pos", 100), ("negs", 1 << 40)):
        s, p, n = src.copy(), pos.copy(), negs.copy()
        {"src": s, "pos": p, "negs": n}[which].flat[17] = bad
        with pytest.raises(euler_b200.EulerError, match="outside"):
            euler_b200.skipgram_xent_loss(s, p, n, t, t)
    loss, _ = euler_b200.skipgram_xent_loss(src, pos, negs, t, t)   # the ctx is fine afterwards
    assert np.isfinite(float(loss))


def test_empty_batch(graph):
    import euler_b200
    t = torch.randn(10, 8, device="cuda", requires_grad=True)
    c = torch.randn(10, 8, device="cuda", requires_grad=True)
    e = np.zeros((0, 1), np.int64)
    loss, met = euler_b200.skipgram_xent_loss(e[:, 0], e, np.zeros((0, 5), np.int64), t, c)
    assert np.isnan(float(loss.detach())) and np.isnan(float(met))
    loss.backward()
    assert float(t.grad.abs().sum()) == 0 and float(c.grad.abs().sum()) == 0


@pytest.mark.parametrize("dim", (1, 3, 16, 128, 200))
@pytest.mark.parametrize("P,K", ((1, 5), (3, 20), (1, 0)))
def test_gradients_match_float64(graph, dim, P, K):
    rng = np.random.RandomState(dim + 10 * K + P)
    n_rows, B = 500, 3000
    src, pos, negs = sr.pair_ids(rng, B, P, K, n_rows)
    if K:
        negs[:, 0] = 7                                 # a hub negative over many chunks
    ctx = sr.context_ids(pos, negs)
    for off in (0, 1):
        target, context = sr.device_table(n_rows, dim, rng, off, dyadic=False), sr.device_table(n_rows, dim, rng, off, dyadic=False)
        _, gt, gc = sr.device_grads(src, pos, negs, target, context)
        wt, wc = sr.grads64(target.cpu().numpy(), context.cpu().numpy(), src, ctx, P)
        for got, want in ((gt, wt), (gc, wc)):
            got = got.cpu().numpy()
            assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max() + 1e-12, (dim, P, K, off)
            untouched = np.abs(want).sum(1) == 0
            assert (got[untouched] == 0).all()


def _integer_setup(rng, dim, B, K, hub_reps):
    """tables and ids whose coefficients are exactly +-1 for g = B (P + K): positives' logits -128 - ..., negatives' +128 + ...
    (sigmoid rounds to 0 and 1), integer rows: every gradient is an integer, computed exactly"""
    n_rows = 400
    tv = rng.randint(-1, 2, size=(n_rows, dim)).astype(np.float32)
    tv[:, 0] = 8
    cv = rng.randint(-1, 2, size=(n_rows, dim)).astype(np.float32)
    cv[:200, 0] = -16                                   # rows [0, 200): positives
    cv[200:, 0] = 16                                    # rows [200, 400): negatives
    src = rng.randint(0, n_rows, size=B)
    pos = rng.randint(0, 200, size=(B, 1))
    negs = rng.randint(200, n_rows, size=(B, K))
    negs.flat[rng.choice(B * K, size=hub_reps, replace=False)] = 333
    return torch.tensor(tv).cuda(), torch.tensor(cv).cuda(), src, pos, negs


@pytest.mark.parametrize("dim", (4, 16, 5))
def test_integer_gradients_exact_through_many_chunks(graph, dim):
    rng = np.random.RandomState(dim)
    B, K = 2000, 5
    target, context, src, pos, negs = _integer_setup(rng, dim, B, K, hub_reps=1500)
    ctx = sr.context_ids(pos, negs)
    N = B * (1 + K)
    _, gt, gc = sr.device_grads(src, pos, negs, target, context, g=float(N))
    wt, wc = sr.grads64(target.cpu().numpy(), context.cpu().numpy(), src, ctx, 1, g=N)
    wt, wc = np.round(wt), np.round(wc)               # the f64 coefficients are +-1 up to e^-128
    assert np.array_equal(gt.cpu().numpy(), wt) and np.array_equal(gc.cpu().numpy(), wc)
    assert np.abs(wc[333]).max() > 1000                  # the hub's row sums > 5 chunks of entries


def test_gradients_bit_identical_run_to_run(graph):
    rng = np.random.RandomState(9)
    src, pos, negs = sr.pair_ids(rng, 20000, 1, 5, 3000)
    negs[:, 2] = 42
    target, context = sr.device_table(3000, 64, rng, dyadic=False), sr.device_table(3000, 64, rng, dyadic=False)
    for shared in (False, True):
        for sparse in (False, True):
            a = sr.device_grads(src, pos, negs, target, context, shared, sparse)
            b = sr.device_grads(src, pos, negs, target, context, shared, sparse)
            assert float(a[0].detach()) == float(b[0].detach())
            for x, y in zip(a[1:], b[1:]):
                if x is None:
                    continue
                x, y = (x.to_dense(), y.to_dense()) if x.is_sparse else (x, y)
                assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()


def test_shared_table_is_the_sum_of_both_gradients(graph):
    rng = np.random.RandomState(12)
    src, pos, negs = sr.pair_ids(rng, 5000, 3, 5, 700)
    negs[:, 1] = 5
    t = sr.device_table(700, 32, rng)
    _, g_sh, _ = sr.device_grads(src, pos, negs, t, t, shared=True)
    _, gt, gc = sr.device_grads(src, pos, negs, t, t.clone())
    want = (gt.double() + gc.double())
    assert torch.allclose(g_sh.double(), want, rtol=1e-6, atol=1e-6 * float(want.abs().max()))
    wt, wc = sr.grads64(t.cpu().numpy(), t.cpu().numpy(), src, sr.context_ids(pos, negs), 3)
    assert np.abs(g_sh.cpu().numpy() - (wt + wc)).max() <= 1e-5 * np.abs(wt + wc).max()


@pytest.mark.parametrize("shared", (False, True))
@pytest.mark.parametrize("dim", (3, 64))
def test_sparse_gradient_is_the_coalesced_dense_one(graph, shared, dim):
    rng = np.random.RandomState(dim + shared)
    src, pos, negs = sr.pair_ids(rng, 4000, 1, 5, 100000)
    negs[:, 0] = 99
    target, context = sr.device_table(100000, dim, rng, dyadic=False), sr.device_table(100000, dim, rng, dyadic=False)
    _, dt, dc = sr.device_grads(src, pos, negs, target, context, shared)
    _, st, sc = sr.device_grads(src, pos, negs, target, context, shared, sparse=True)
    for d, s in ((dt, st), (dc, sc)):
        if d is None:
            assert s is None
            continue
        assert s.is_sparse
        rows = s._indices()[0].cpu().numpy()   # raw: accumulation into .grad may clear the coalesced flag
        assert (np.diff(rows) > 0).all()                  # coalesced: distinct rows, ascending
        touched = np.nonzero(d.abs().sum(1).cpu().numpy())[0]
        assert set(touched) <= set(rows)
        assert d[torch.as_tensor(rows, device="cuda")].cpu().numpy().tobytes() == s._values().cpu().numpy().tobytes()
        assert s.to_dense().cpu().numpy().tobytes() == d.cpu().numpy().tobytes()


# ------------------------------------------------------------------------------------ whole steps
def _step64(tables, src, pos, negs, shared, lr):
    tb, cb = tables
    ctx = sr.context_ids(pos, negs)
    x, loss = sr.forward64(tb, cb, src, ctx, 1)
    gt, gc = sr.grads64(tb, cb, src, ctx, 1)
    if shared:
        return loss, (tb - lr * (gt + gc),)
    return loss, (tb - lr * gt, cb - lr * gc)


def _run_step(model, inputs, seed, lr):
    import euler_b200
    euler_b200.seed(seed)
    emb, loss, name, metric = model(inputs)
    model.zero_grad()
    loss.backward()
    with torch.no_grad():
        for p in model.parameters():
            p.add_(p.grad, alpha=-lr)
    return emb, loss, metric


@pytest.mark.parametrize("kind", ("deepwalk", "node2vec", "line1", "line2"))
@pytest.mark.parametrize("sparse", (False, True))
def test_whole_step_matches_float64_and_the_composition(graph, kind, sparse):
    import euler_b200
    from euler_b200 import unsupervised as un
    max_id, dim, lr = 4096, 32, 0.5
    torch.manual_seed(3)
    if kind in ("deepwalk", "node2vec"):
        pq = (1, 1) if kind == "deepwalk" else (0.5, 2)
        cls = un.DeepWalk if kind == "deepwalk" else un.Node2Vec
        model = cls(0, [0], max_id, dim, walk_len=5, walk_p=pq[0], walk_q=pq[1], num_negs=5, sparse_grad=sparse, device="cuda")
    else:
        model = un.Line(0, [0], max_id, dim, num_negs=5, order=int(kind[-1]), sparse_grad=sparse, device="cuda")
    shared = model.context_encoder is model.target_encoder
    composed = copy.deepcopy(model)
    composed.fused = False
    if shared:
        composed.context_encoder = composed.target_encoder
    inputs = torch.as_tensor(np.random.RandomState(5).randint(1, max_id + 1, size=256), dtype=torch.int64).cuda()
    before = [p.detach().double().cpu().numpy() for p in model.parameters()]
    euler_b200.seed(77)
    src, pos, negs = model.to_sample(inputs)
    B = src.shape[0]
    assert (src.shape, pos.shape, negs.shape) == model.sample_shapes(inputs.numel())
    assert int(pos.max()) <= max_id + 1 and int(negs.max()) <= max_id + 1
    loss64, after64 = _step64(before if not shared else (before[0], before[0]), src.cpu().numpy().reshape(-1),
                              pos.cpu().numpy(), negs.cpu().numpy(), shared, lr)
    emb, loss, metric = _run_step(model, inputs, 77, lr)
    _, loss_c, metric_c = _run_step(composed, inputs, 77, lr)
    assert emb.shape == (inputs.numel(), dim)
    assert abs(float(loss.detach()) - loss64) <= 1e-6 * loss64
    assert abs(float(loss.detach()) - float(loss_c.detach())) <= 1e-5 * loss64
    assert abs(float(metric) - float(metric_c)) <= 2.0 / B   # a near-tie may order differently under matmul's sums
    for got, got_c, want in zip(model.parameters(), composed.parameters(), after64):
        assert np.abs(got.detach().double().cpu().numpy() - want).max() <= 1e-5
        assert torch.allclose(got, got_c, rtol=0, atol=1e-5)
    assert B > 0
