"""GPU: ShallowEncoder's fused input row (ops.shallow_encode, eu_shallow_encode and its backward passes) against the
composition of the single ops it replaces -- F.embedding, get_dense_feature, sparse_feature_embedding -- and against float64;
the sparse COO gradients of shallow_encode and sparse_feature_embedding; and ShallowEncoder in a two-hop training step."""
import numpy as np
import pytest
import torch

import embedding_reference as er

pytestmark = pytest.mark.gpu

N_NODES, N_ROWS, N_ID = 600, 1000, 1000   # graph ids 1 .. 600; slot tables of N_ROWS rows; id table of N_ID rows
SLOT_DIMS = (5, 12, 3)                     # the dense slots feat0, feat1, feat2 (feat0 ends at an unaligned column)
ABSENT = (0, 650, 999)                     # ids the graph does not hold, all inside the id table


def _lens_mixed(rng, n):   # 0 (default), 1, ordinary, and a few bags of more than 256 values
    k = rng.choice([0, 1, 2, 3, 5, 9], size=n, p=[0.3, 0.2, 0.2, 0.15, 0.1, 0.05])
    k[rng.choice(n, size=3, replace=False)] = [257, 300, 700]
    return k


def _graph(g):
    import euler_b200
    return euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                     node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=list(SLOT_DIMS),
                                     u64_ptr=g["u64_ptr"], u64_val=g["u64_val"], n_u64_slots=g["S"])


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = er.slot_graph(5, N_NODES, [_lens_mixed, lambda rng, n: rng.randint(1, 4, size=n)],
                      [lambda rng, k: rng.randint(0, N_ROWS - 1, size=k), lambda rng, k: rng.randint(0, 50, size=k)],
                      feat_dim=sum(SLOT_DIMS))
    gr = _graph(g)
    rng = np.random.RandomState(2)
    nodes = np.concatenate([g["ids"][rng.randint(0, N_NODES, size=700)], ABSENT, g["ids"][:5], g["ids"][:5]]).astype(np.int64)
    return dict(g=g, gr=gr, nodes=nodes)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)


def _table(n_rows, dim, seed=3, offset=0):
    """a table whose data pointer is `offset` floats past a 16-byte boundary"""
    t = torch.randn(n_rows * dim + offset, generator=torch.Generator().manual_seed(seed)).cuda()
    return t[offset:].view(n_rows, dim)


# the dense requests: feat0 padded (stored 5, asked 8), feat1 clipped (stored 12, asked 7), feat2 as stored, an unknown slot
DENSE = [("feat0", 8), ("feat1", 7), ("feat2", 3), (99, 2)]


def _inputs(dim, off=0, combiners=("sum", "mean")):
    id_table = _table(N_ID, dim, seed=1, offset=off)
    sparse = [("u64_0", _table(N_ROWS, dim, seed=2, offset=off), N_ROWS - 1, combiners[0]),
              ("u64_1", _table(60, dim, seed=3, offset=off), 55, combiners[1]),
              ("no_such_slot", _table(20, dim, seed=4), 7, "sum")]
    return id_table, sparse


@pytest.mark.parametrize("dim", (1, 3, 4, 16, 128))
def test_concat_forward_bit_exact(env, dim):
    import euler_b200
    nodes = env["nodes"]
    for off in (0, 1):   # aligned and unaligned tables (and, for dim 1 and 3, unaligned slot columns in the output)
        id_table, sparse = _inputs(dim, off)
        for dense in (DENSE, DENSE[:1], []):
            out = euler_b200.shallow_encode(nodes, id_table, dense, sparse, "concat")
            idp, dp, sp = er.composed_parts(nodes, id_table, dense, sparse)
            want = torch.cat(idp + dp + sp, 1)
            assert out.shape == want.shape and out.cpu().numpy().tobytes() == want.cpu().numpy().tobytes(), (dim, off, len(dense))
        out = euler_b200.shallow_encode(nodes, None, DENSE[:2], sparse[1:], "concat")   # no id table
        idp, dp, sp = er.composed_parts(nodes, None, DENSE[:2], sparse[1:])
        assert out.cpu().numpy().tobytes() == torch.cat(dp + sp, 1).cpu().numpy().tobytes()


def test_raw_abi_unaligned_output(env):
    """the C entry point with an out pointer 4 bytes past a 16-byte boundary: the same bits"""
    import ctypes as C
    import euler_b200
    from euler_b200 import _lib, ops
    nodes = torch.as_tensor(env["nodes"], device="cuda")
    id_table, sparse = _inputs(16)
    res = [(euler_b200.get_graph().sparse_feature_id(n), t, dv, ops._COMBINERS[c]) for n, t, dv, c in sparse]
    dense = [(0, 8), (1, 7)]
    p = ops._shallow_problem(nodes, id_table, dense, res, 0)
    W = 16 + 15 + 3 * 16
    buf = torch.empty(nodes.numel() * W + 1, device="cuda")
    _lib.check(_lib.load().eu_shallow_encode(ops._ctx_on_stream()._h, C.byref(p), buf.data_ptr() + 4, None))
    want = euler_b200.shallow_encode(nodes, id_table, [("feat0", 8), ("feat1", 7)], sparse, "concat")
    assert buf[1:].cpu().numpy().tobytes() == want.cpu().numpy().tobytes()


def test_empty_batch_and_absent_nodes(env):
    import euler_b200
    id_table, sparse = _inputs(4)
    assert euler_b200.shallow_encode([], id_table, DENSE, sparse, "concat").shape == (0, 4 + 20 + 12)
    emb, feats = euler_b200.shallow_encode(np.zeros((0,), np.int64), id_table, DENSE, sparse[:1], "add")
    assert emb.shape == (0, 4) and feats.shape == (0, 20)
    out = euler_b200.shallow_encode(list(ABSENT), None, DENSE, [sparse[0]], "concat")   # absent: zero features, the default row
    assert not out[:, :20].any()
    assert torch.equal(out[:, 20:], sparse[0][1][N_ROWS - 1].expand(3, 4))


@pytest.mark.parametrize("dim", (3, 16, 128))
def test_add_forward_bit_exact_and_close_to_f64(env, dim):
    import euler_b200
    nodes = env["nodes"]
    for off in (0, 1):
        id_table, sparse = _inputs(dim, off)
        emb, feats = euler_b200.shallow_encode(nodes, id_table, DENSE, sparse, "add")
        idp, dp, sp = er.composed_parts(nodes, id_table, DENSE, sparse)
        want = idp[0]
        for x in sp:
            want = want + x    # the documented order: id + sparse_0 + sparse_1 + ..
        assert emb.cpu().numpy().tobytes() == want.cpu().numpy().tobytes(), (dim, off)
        assert feats.cpu().numpy().tobytes() == torch.cat(dp, 1).cpu().numpy().tobytes()
        g = env["g"]
        parts = [id_table.cpu().double().numpy()[nodes]]
        mag = np.abs(parts[0])
        for n, t, dv, c in sparse:
            fid = euler_b200.get_graph().sparse_feature_id(n)
            bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, fid, dv)
            parts.append(er.lookup_f64(t.cpu().numpy(), bl, c))
            mag = mag + er.lookup_f64(np.abs(t.cpu().numpy()), bl, c)
        err = np.abs(emb.cpu().numpy() - sum(parts))
        assert (err <= 1e-6 * mag + 1e-7).all(), float((err / (mag + 1e-30)).max())
    emb, feats = euler_b200.shallow_encode(nodes, None, [], sparse[:1], "add")   # one term: its bits
    assert feats is None and torch.equal(emb, er.composed_parts(nodes, None, [], sparse[:1])[2][0])


def test_bad_inputs_raise(env):
    import euler_b200
    nodes = env["nodes"]
    id_table, sparse = _inputs(4)
    with pytest.raises(euler_b200.EulerError, match="id table"):
        euler_b200.shallow_encode(nodes, id_table[:600], [], sparse, "concat")   # ids 650 and 999 lie outside
    with pytest.raises(euler_b200.EulerError, match="id table"):
        euler_b200.shallow_encode([-1], id_table, [], [], "concat")
    with pytest.raises(euler_b200.EulerError, match="outside the table"):
        euler_b200.shallow_encode(nodes, None, [], [("u64_0", _table(500, 4), 0)], "concat")   # slot 0 holds values up to 998
    for dv in (60, -1):
        with pytest.raises(euler_b200.EulerError, match="default_value"):
            euler_b200.shallow_encode(nodes, None, [], [("u64_1", _table(60, 4), dv)], "concat")
    with pytest.raises(euler_b200.EulerError, match="one dim"):
        euler_b200.shallow_encode(nodes, id_table, [], [("u64_1", _table(60, 8), 0)], "add")
    with pytest.raises(euler_b200.EulerError, match="combiner"):
        euler_b200.shallow_encode(nodes, id_table, [], [], "max")
    with pytest.raises(euler_b200.EulerError, match="columns"):
        euler_b200.shallow_encode(nodes, None, [("feat0", 20000)], [], "concat")


def test_forward_captures_in_a_cuda_graph(env):
    import euler_b200
    nodes = torch.as_tensor(env["nodes"], device="cuda")
    id_table, sparse = _inputs(16)
    eager = euler_b200.shallow_encode(nodes, id_table, DENSE, sparse, "concat")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        euler_b200.shallow_encode(nodes, id_table, DENSE, sparse, "concat")
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = euler_b200.shallow_encode(nodes, id_table, DENSE, sparse, "concat")
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    cg.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == eager.cpu().numpy().tobytes()


def _grads(nodes, id_table, sparse, combiner, grad, sparse_grad=False):
    import euler_b200
    leaves = [id_table.detach().clone().requires_grad_(True)] + [t.detach().clone().requires_grad_(True) for _, t, _, _ in sparse]
    sp = [(n, leaf, dv, c) for (n, _, dv, c), leaf in zip(sparse, leaves[1:])]
    res = euler_b200.shallow_encode(nodes, leaves[0], DENSE, sp, combiner, sparse_grad=sparse_grad)
    return torch.autograd.grad(res if combiner == "concat" else res[0], leaves, grad)   # the op's own gradients


def _want_grads(env, nodes, id_table, sparse, combiner, grad):
    """float64 gradients of every table, and the sums of the terms' magnitudes"""
    import euler_b200
    g = env["g"]
    gn = grad.cpu().double().numpy()
    dims = [id_table.shape[1]] + [t.shape[1] for _, t, _, _ in sparse]
    cols, c0 = [], 0
    for j, d in enumerate(dims):
        if combiner == "concat":
            cols.append(slice(c0, c0 + d))
            c0 += d + (20 if j == 0 else 0)   # the dense columns follow the id columns
        else:
            cols.append(slice(0, d))
    want, mag = [], []
    w = np.zeros((N_ID, dims[0]))
    m = np.zeros((N_ID, dims[0]))
    np.add.at(w, nodes, gn[:, cols[0]])
    np.add.at(m, nodes, np.abs(gn[:, cols[0]]))
    want.append(w)
    mag.append(m)
    for k, (n, t, dv, c) in enumerate(sparse):
        fid = euler_b200.get_graph().sparse_feature_id(n)
        bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, fid, dv)
        want.append(er.grad_f64(gn[:, cols[k + 1]], bl, t.shape[0], c))
        mag.append(er.grad_f64(np.abs(gn[:, cols[k + 1]]), bl, t.shape[0], c))
    return want, mag


@pytest.mark.parametrize("combiner", ("concat", "add"))
@pytest.mark.parametrize("dim", (3, 16, 128))
def test_gradients_f64_run_to_run_untouched_and_sparse(env, combiner, dim):
    nodes = env["nodes"]
    id_table, sparse = _inputs(dim, combiners=("mean", "sqrtn"))
    W = 3 * dim + dim + 20 if combiner == "concat" else dim
    grad = torch.randn(len(nodes), W, generator=torch.Generator().manual_seed(9)).cuda()
    g1 = _grads(nodes, id_table, sparse, combiner, grad)
    g2 = _grads(nodes, id_table, sparse, combiner, grad)
    gs = _grads(nodes, id_table, sparse, combiner, grad, sparse_grad=True)
    want, mag = _want_grads(env, nodes, id_table, sparse, combiner, grad)
    for t in range(len(g1)):
        assert torch.equal(g1[t], g2[t]), t
        got = g1[t].cpu().numpy()
        err = np.abs(got - want[t])
        assert (err <= 1e-5 * mag[t] + 1e-7).all(), (t, float((err / (mag[t] + 1e-30)).max()))
        assert not got[mag[t].sum(1) == 0].any()   # rows no entry names are exactly zero
        touched = np.flatnonzero(mag[t].sum(1) > 0)
        s = gs[t]
        assert s.is_sparse and s.is_coalesced()
        assert np.array_equal(s.indices()[0].cpu().numpy(), touched)
        assert torch.equal(s.values(), g1[t][s.indices()[0]])
        assert torch.equal(s.to_dense(), g1[t])


def test_default_row_hit_by_many_entries_is_exact():
    """20 000 nodes, most with an empty slot: the default row gathers > 10 000 entries over many 256-entry chunks, and an
    integer gradient counts every entry exactly"""
    import euler_b200
    n = 20000

    def lens(rng, k):
        x = rng.randint(1, 4, size=k)
        x[rng.rand(k) < 0.7] = 0
        return x
    g = er.slot_graph(11, n, [lens], [lambda rng, k: rng.randint(0, 99, size=k)], feat_dim=0)
    euler_b200.set_graph(er.cuda_slot_graph(g), rng="minstd", seed=1)
    nodes = g["ids"].astype(np.int64)
    bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], 1, nodes, 0, 99)
    counts = np.zeros(100)
    for b in bl:
        np.add.at(counts, b, 1)
    assert counts[99] > 10000
    id_t = torch.zeros(n + 2, 8, device="cuda", requires_grad=True)
    t = torch.zeros(100, 8, device="cuda", requires_grad=True)
    out = euler_b200.shallow_encode(nodes, id_t, [], [("u64_0", t, 99)], "concat")
    out.backward(torch.ones_like(out))
    assert np.array_equal(t.grad[:, 0].cpu().numpy(), counts)
    assert np.array_equal(id_t.grad[:, 0].cpu().numpy(), np.bincount(nodes, minlength=n + 2))
    t2 = t.detach().clone().requires_grad_(True)
    euler_b200.sparse_feature_embedding(nodes, "u64_0", t2, 99, sparse_grad=True).backward(torch.ones(n, 8, device="cuda"))
    assert t2.grad.is_sparse and np.array_equal(t2.grad.to_dense()[:, 0].cpu().numpy(), counts)


@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_sparse_feature_embedding_sparse_grad_equals_dense(env, combiner):
    import euler_b200
    nodes = env["nodes"]
    table = _table(N_ROWS, 16)
    grad = torch.randn(len(nodes), 16, generator=torch.Generator().manual_seed(4)).cuda()
    dense, sparse = table.clone().requires_grad_(True), table.clone().requires_grad_(True)
    euler_b200.sparse_feature_embedding(nodes, "u64_0", dense, N_ROWS - 1, combiner).backward(grad)
    out = euler_b200.sparse_feature_embedding(nodes, "u64_0", sparse, N_ROWS - 1, combiner, sparse_grad=True)
    assert torch.equal(out, euler_b200.sparse_feature_embedding(nodes, "u64_0", table, N_ROWS - 1, combiner))
    s, = torch.autograd.grad(out, sparse, grad)
    assert s.is_sparse and s.is_coalesced()
    assert torch.equal(s.to_dense(), dense.grad)
    g = env["g"]
    named = {v for b in er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, 0, N_ROWS - 1) for v in b}
    assert s.indices()[0].tolist() == sorted(named)


def test_sparse_backward_on_a_large_table_allocates_little(env):
    """a 50M-row slot table: the sparse backward's allocator peak stays under a tenth of the table"""
    import euler_b200
    nodes = torch.as_tensor(env["nodes"], device="cuda")
    n_rows, dim = 50_000_000, 4
    table = torch.zeros(n_rows, dim, device="cuda").requires_grad_(True)
    for sparse_grad in (True, False):
        out = euler_b200.shallow_encode(nodes, None, [], [("u64_0", table, n_rows - 1)], "concat", sparse_grad=sparse_grad)
        grad = torch.ones_like(out)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        g, = torch.autograd.grad(out, table, grad)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        if sparse_grad:
            assert g.is_sparse and peak < table.numel() * 4 / 10, peak
            sparse_rows = g.coalesce().indices()[0]
        else:
            assert peak >= table.numel() * 4
            assert torch.equal(torch.nonzero(g.abs().sum(1) > 0).reshape(-1), sparse_rows)
        del g, out


def test_two_hop_sage_step_matches_the_composition(env):
    """sample_fanout -> ShallowEncoder (ids, dense and sparse slots) -> mean over each hop's neighbours -> Dense -> SGD, fused
    against fused=False: the same embeddings, gradients and updated tables"""
    import euler_b200
    from euler_b200.encoders import Dense, ShallowEncoder
    g = env["g"]
    seeds = g["ids"][:64].astype(np.int64)

    def step(fused, sparse_grad):
        torch.manual_seed(0)
        enc = ShallowEncoder(dim=None, feature_idx=["feat0", "feat1"], feature_dim=[8, 7], max_id=N_ID - 2,
                             sparse_feature_idx=["u64_0", "u64_1"], sparse_feature_max_id=[N_ROWS - 2, 58], embedding_dim=[8, 8, 4],
                             fused=fused, sparse_grad=sparse_grad, device="cuda")
        out_dense = Dense(4 * enc.output_dim, 5, device="cuda")   # two layers of [self | mean]
        euler_b200.seed(7)
        ids, _, _ = euler_b200.sample_fanout(seeds, [[0], [0]], [3, 2], default_node=0)
        h = [enc(x) for x in ids]
        for _ in range(2):
            h = [torch.cat([h[i], h[i + 1].reshape(h[i].shape[0], -1, h[i].shape[1]).mean(1)], 1) for i in range(len(h) - 1)]
        loss = out_dense(h[0]).square().mean()
        opt = torch.optim.SGD(list(enc.parameters()) + list(out_dense.parameters()), lr=0.5)
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss.detach(), [p.detach().clone() for p in enc.parameters()]

    loss_c, p_c = step(False, False)
    for sparse_grad in (False, True):
        loss_f, p_f = step(True, sparse_grad)
        torch.testing.assert_close(loss_f, loss_c, rtol=1e-5, atol=1e-7)
        for a, b in zip(p_f, p_c):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
