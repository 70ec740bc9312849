"""GPU: the fused sparse-feature embedding (eu_sparse_embedding_lookup and its backward) against the numpy restatements of
embedding_lookup_sparse, against the composition get_sparse_feature + embedding_bag, and through SparseEmbedding."""
import numpy as np
import pytest
import torch

import embedding_reference as er

pytestmark = pytest.mark.gpu

DIMS = (1, 3, 4, 16, 64, 128, 200)


def _lens_mixed(rng, n):   # 0 (default), 1, ordinary, and a few bags of more than 256 values
    k = rng.choice([0, 1, 2, 3, 5, 9], size=n, p=[0.3, 0.2, 0.2, 0.15, 0.1, 0.05])
    k[rng.choice(n, size=3, replace=False)] = [257, 300, 700]
    return k


@pytest.fixture(scope="module")
def env():
    import euler_b200
    n_rows = 1000
    g = er.slot_graph(5, 600, [_lens_mixed, lambda rng, n: rng.randint(1, 4, size=n)],
                      [lambda rng, k: rng.randint(0, n_rows - 1, size=k), lambda rng, k: rng.randint(0, 50, size=k)])
    gr = er.cuda_slot_graph(g)
    euler_b200.set_graph(gr, rng="minstd", seed=1)
    rng = np.random.RandomState(2)
    nodes = np.concatenate([g["ids"][rng.randint(0, 600, size=700)], [0, 123456, 999999], g["ids"][:5], g["ids"][:5]]).astype(np.int64)
    return dict(g=g, gr=gr, nodes=nodes, n_rows=n_rows)


def _bags(env, nodes, fid, default):
    g = env["g"]
    return er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, fid, default)


def _table(n_rows, dim, seed=3, offset=0):
    """a table whose data pointer is `offset` floats past a 16-byte boundary"""
    t = torch.randn(n_rows * dim + offset, generator=torch.Generator().manual_seed(seed)).cuda()
    return t[offset:].view(n_rows, dim)


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_forward_bit_exact(env, dim, combiner):
    import euler_b200
    n_rows, nodes = env["n_rows"], env["nodes"]
    bl = _bags(env, nodes, 0, n_rows - 1)
    for off in (0, 1):   # aligned and unaligned table
        table = _table(n_rows, dim, offset=off)
        want = er.lookup_f32(table.cpu().numpy(), bl, combiner)
        out = euler_b200.sparse_feature_embedding(nodes, "u64_0", table, n_rows - 1, combiner)
        assert out.cpu().numpy().tobytes() == want.tobytes(), (dim, combiner, off)


@pytest.mark.parametrize("dim", (4, 16, 128))
def test_forward_unaligned_out_and_raw_abi(env, dim):
    """the C entry point with an out pointer 4 bytes past a 16-byte boundary: the same bits"""
    import euler_b200
    from euler_b200 import _lib
    n_rows, nodes = env["n_rows"], env["nodes"]
    table = _table(n_rows, dim)
    nd = torch.as_tensor(nodes, device="cuda")
    buf = torch.empty(len(nodes) * dim + 1, device="cuda")
    ctx = euler_b200.ops._ctx_on_stream()
    _lib.check(_lib.load().eu_sparse_embedding_lookup(ctx._h, nd.data_ptr(), len(nodes), 1, 7, table.data_ptr(), n_rows, dim, 1,
                                                      buf.data_ptr() + 4))
    want = er.lookup_f32(table.cpu().numpy(), _bags(env, nodes, 1, 7), "mean")
    assert buf[1:].cpu().numpy().tobytes() == want.tobytes()


def test_negative_zero_rows_and_empty_batch(env):
    import euler_b200
    n_rows = env["n_rows"]
    table = torch.zeros((n_rows, 8), device="cuda")
    table[n_rows - 1] = -0.0
    out = euler_b200.sparse_feature_embedding([999999], "u64_0", table, n_rows - 1)   # absent id: the default row
    assert torch.signbit(out).all()
    assert euler_b200.sparse_feature_embedding([], "u64_0", table, 0).shape == (0, 8)


def test_unknown_slot_gives_the_default_row(env):
    import euler_b200
    n_rows = env["n_rows"]
    table = _table(n_rows, 16)
    out = euler_b200.sparse_feature_embedding(env["nodes"][:50], "no_such_slot", table, 17, "sqrtn")
    assert torch.equal(out, table[17].expand(50, 16))


@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_matches_embedding_bag_composition(env, combiner):
    import euler_b200
    n_rows, nodes = env["n_rows"], env["nodes"]
    table = _table(n_rows, 64)
    (idx, vals, shape), = euler_b200.get_sparse_feature(nodes, ["u64_0"], [n_rows - 1])
    offsets = torch.searchsorted(idx[:, 0].contiguous(), torch.arange(len(nodes), device="cuda"))
    want = torch.nn.functional.embedding_bag(vals, table, offsets, mode="sum" if combiner == "sqrtn" else combiner)
    if combiner == "sqrtn":
        cnt = torch.bincount(idx[:, 0], minlength=len(nodes)).float()
        want = want / cnt.sqrt()[:, None]
    out = euler_b200.sparse_feature_embedding(nodes, "u64_0", table, n_rows - 1, combiner)
    torch.testing.assert_close(out, want, rtol=1e-6, atol=1e-5)


def test_out_of_range_values_raise(env):
    import euler_b200
    table = _table(500, 4)   # slot 0 holds values up to 998
    with pytest.raises(euler_b200.EulerError, match="outside the table"):
        euler_b200.sparse_feature_embedding(env["nodes"], "u64_0", table, 0)
    with pytest.raises(euler_b200.EulerError, match="default_value"):
        euler_b200.sparse_feature_embedding(env["nodes"], "u64_1", table, 500)
    with pytest.raises(euler_b200.EulerError, match="default_value"):
        euler_b200.sparse_feature_embedding(env["nodes"], "u64_1", table, -1)


def test_forward_captures_in_a_cuda_graph(env):
    import euler_b200
    n_rows, nodes = env["n_rows"], torch.as_tensor(env["nodes"], device="cuda")
    table = _table(n_rows, 64)
    eager = euler_b200.sparse_feature_embedding(nodes, "u64_0", table, n_rows - 1, "mean")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        euler_b200.sparse_feature_embedding(nodes, "u64_0", table, n_rows - 1, "mean")
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = euler_b200.sparse_feature_embedding(nodes, "u64_0", table, n_rows - 1, "mean")
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def _close_to_f64(got, grad, bl, n_rows, combiner):
    """|got - f64| <= 1e-5 * (the sum of the terms' magnitudes) per element: a long sum may cancel, its rounding may not"""
    want = er.grad_f64(grad.cpu().numpy(), bl, n_rows, combiner)
    mag = er.grad_f64(np.abs(grad.cpu().numpy()), bl, n_rows, combiner)
    err = np.abs(got.cpu().numpy() - want)
    assert (err <= 1e-5 * mag + 1e-7).all(), float((err / (mag + 1e-30)).max())


def _backward(nodes, fid, table, default, combiner, grad):
    import euler_b200
    t = table.detach().clone().requires_grad_(True)
    euler_b200.sparse_feature_embedding(nodes, fid, t, default, combiner).backward(grad)
    return t.grad


@pytest.mark.parametrize("dim", (3, 16, 64, 200))
@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_backward_against_f64_and_run_to_run(env, dim, combiner):
    n_rows, nodes = env["n_rows"], env["nodes"]
    table = _table(n_rows, dim)
    grad = torch.randn(len(nodes), dim, generator=torch.Generator().manual_seed(9)).cuda()
    g1 = _backward(nodes, "u64_0", table, n_rows - 1, combiner, grad)
    g2 = _backward(nodes, "u64_0", table, n_rows - 1, combiner, grad)
    assert torch.equal(g1, g2)
    bl = _bags(env, nodes, 0, n_rows - 1)
    _close_to_f64(g1, grad, bl, n_rows, combiner)
    touched = np.zeros(n_rows, bool)
    touched[[v for b in bl for v in b]] = True
    assert not g1[torch.as_tensor(~touched, device="cuda")].any()   # rows no entry names stay exactly zero


def test_backward_hot_values_span_many_chunks():
    """the default of a graph with 30 % empty slots, and one id present in 10^5+ bags: both segments cover many 256-entry
    chunks"""
    import euler_b200
    n, n_rows, hot = 250000, 5000, 42

    def lens(rng, k):
        x = rng.randint(1, 4, size=k)
        x[rng.rand(k) < 0.3] = 0
        return x

    def vals(rng, k):
        v = rng.randint(0, n_rows - 1, size=k)
        v[rng.rand(k) < 0.6] = hot
        return v
    g = er.slot_graph(11, n, [lens], [vals])
    euler_b200.set_graph(er.cuda_slot_graph(g), rng="minstd", seed=1)
    nodes = g["ids"].astype(np.int64)
    bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], 1, nodes, 0, n_rows - 1)
    assert sum(1 for b in bl if hot in b) > 100000 and sum(1 for b in bl if b == [n_rows - 1]) > 0.25 * n
    table = _table(n_rows, 16)
    counts = np.zeros(n_rows)
    for b in bl:
        np.add.at(counts, b, 1)
    ones = _backward(nodes, "u64_0", table, n_rows - 1, "sum", torch.ones(n, 16, device="cuda"))
    assert np.array_equal(ones[:, 0].cpu().numpy(), counts)   # integer sums below 2^24 are exact: every chunk is counted once
    grad = torch.randn(n, 16, generator=torch.Generator().manual_seed(4)).cuda()
    for combiner in ("sum", "mean"):
        g1 = _backward(nodes, "u64_0", table, n_rows - 1, combiner, grad)
        assert torch.equal(g1, _backward(nodes, "u64_0", table, n_rows - 1, combiner, grad))
        _close_to_f64(g1, grad, bl, n_rows, combiner)


@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_sparse_embedding_module_paths_agree(env, combiner):
    """SparseEmbedding: the fused lookup and the literal path over get_sparse_feature, forward and gradient"""
    import euler_b200
    from euler_b200.encoders import SparseEmbedding
    n_rows, nodes = env["n_rows"], env["nodes"]
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)
    emb = SparseEmbedding(n_rows - 1, 32, combiner=combiner, device="cuda")
    assert emb.embeddings.shape == (n_rows, 32) and emb.embeddings.abs().max() <= 0.0004
    with torch.no_grad():
        emb.embeddings.copy_(_table(n_rows, 32))
    grad = torch.randn(len(nodes), 32, generator=torch.Generator().manual_seed(5)).cuda()
    fused = emb.lookup(nodes, "u64_0", n_rows - 1)
    fused.backward(grad)
    g_fused = emb.embeddings.grad.clone()
    emb.embeddings.grad = None
    literal = emb(euler_b200.get_sparse_feature(nodes, ["u64_0"], [n_rows - 1])[0])
    literal.backward(grad)
    # two float32 summation orders (the literal path accumulates with atomics) over bags of up to 700 rows: they agree to
    # 1e-5 of the sum of the terms' magnitudes
    bl = _bags(env, nodes, 0, n_rows - 1)
    mag = torch.as_tensor(er.lookup_f64(np.abs(emb.embeddings.detach().cpu().numpy()), bl, combiner), device="cuda").float()
    assert ((fused - literal).abs() <= 1e-5 * mag + 1e-7).all()
    gmag = torch.as_tensor(er.grad_f64(np.abs(grad.cpu().numpy()), bl, n_rows, combiner), device="cuda").float()
    assert ((g_fused - emb.embeddings.grad).abs() <= 1e-5 * gmag + 1e-7).all()


def test_two_hop_sage_input_step_forward_and_backward(env):
    """SageEncoderNew's input step (encoders.py:590-626 with mean aggregators): sample_fanout, one embedding per hop and slot,
    then per layer mean(neighbors) concatenated with self -- against a float64 restatement, forward and gradient"""
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)
    n_rows, g = env["n_rows"], env["g"]
    seeds = g["ids"][:64].astype(np.int64)
    ids, _, _ = euler_b200.sample_fanout(seeds, [[0], [0]], [3, 2], default_node=0)
    table = _table(n_rows, 8).requires_grad_(True)
    hops = [euler_b200.sparse_feature_embedding(h, "u64_0", table, n_rows - 1, "sum") for h in ids]

    def layer(h):   # mean aggregator over each hop's neighbors, concatenated with self
        out = []
        for i in range(len(h) - 1):
            nb = h[i + 1].reshape(h[i].shape[0], -1, h[i].shape[1]).mean(1)
            out.append(torch.cat([h[i], nb], 1))
        return out
    x = layer(layer(hops))[0]
    gx = torch.randn_like(x)
    x.backward(gx)
    t64 = torch.as_tensor(table.detach().cpu().numpy(), dtype=torch.float64).requires_grad_(True)
    hops64 = []
    for h in ids:
        bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], h.cpu().numpy(), 0, n_rows - 1)
        hops64.append(torch.stack([t64[b].sum(0) for b in bl]))
    x64 = layer(layer(hops64))[0]
    x64.backward(torch.as_tensor(gx.cpu().numpy(), dtype=torch.float64))
    np.testing.assert_allclose(x.detach().cpu().numpy(), x64.detach().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(table.grad.cpu().numpy(), t64.grad.numpy(), rtol=1e-5, atol=1e-5)


def test_tiny_fixture_slots():
    """the tiny Euler 2.0 fixture's own sparse slots: the fused sum equals the float32 restatement over get_sparse_feature"""
    import os
    import euler_b200
    import graphs
    gr = euler_b200.Graph.load(os.path.join(graphs.GOLDEN, "tiny_euler"))
    euler_b200.set_graph(gr, rng="minstd", seed=1)
    nodes = np.asarray([1, 2, 0, 3, 4, 5, 6, 77], np.int64)
    for name in ("f1", "f2"):
        (idx, vals, _), = euler_b200.get_sparse_feature(nodes, [name], [0])
        idx, vals = idx.cpu().numpy(), vals.cpu().numpy()
        n_rows = int(vals.max()) + 1
        table = _table(n_rows, 5)
        bl = [list(vals[idx[:, 0] == i]) for i in range(len(nodes))]
        want = er.lookup_f32(table.cpu().numpy(), bl, "sum")
        out = euler_b200.sparse_feature_embedding(nodes, name, table, 0)
        assert out.cpu().numpy().tobytes() == want.tobytes(), name
