"""GPU: the exact outputs of the ops whose library calls, ragged fetches and sparse table gradients share one path in ops.py,
on the tiny Euler directory and on Graph.from_csr graphs: empty inputs, zero totals, nodes that take the default sparse entry,
unknown feature names, exact dense shapes, empty rows of sorted listings and batch adjacencies, and the dense and sparse
table gradients of the four losses."""
import numpy as np
import pytest
import torch

import embedding_reference as er
import graphs
import skipgram_reference as sr

pytestmark = pytest.mark.gpu

ABSENT = 10 ** 12


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def env():
    """a 2-edge-type graph with many empty neighbor groups, two uint64 slots (u64_0 over [0, 50), u64_1 over [0, 8), some
    nodes without values) and one binary slot (some rows empty); nodes to query include an absent id, repeats and a node
    without any neighbor"""
    import euler_b200
    n, T, S = 60, 2, 2
    g = graphs.random_graph(seed=71, n=n, T=T, avg_deg=2, empty_frac=0.4)
    rng = np.random.RandomState(72)
    lens = np.stack([rng.choice([0, 1, 2, 4], size=n), rng.randint(0, 3, size=n)], axis=1).reshape(-1)
    u64_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    u64_val = np.concatenate([rng.randint(0, 50 if k % S == 0 else 8, size=c) for k, c in enumerate(lens)]).astype(np.uint64)
    bin_rows = [bytes(rng.randint(97, 123, size=rng.choice([0, 1, 3])).astype(np.uint8)) for _ in range(n)]
    bin_ptr = np.concatenate([[0], np.cumsum([len(b) for b in bin_rows])]).astype(np.int64)
    bin_val = np.frombuffer(b"".join(bin_rows), np.uint8).copy()
    g.update(u64_ptr=u64_ptr, u64_val=u64_val, S=S, bin_rows=bin_rows)
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=T, cum_w=g["cum_w"], grp_cum=g["grp_cum"],
                                   node_type=g["node_type"], node_w=g["node_w"], u64_ptr=u64_ptr, u64_val=u64_val, n_u64_slots=S,
                                   bin_ptr=bin_ptr, bin_val=bin_val, n_bin_slots=1)
    grp_ptr = g["grp_ptr"]
    lonely = [int(g["ids"][r]) for r in range(n) if grp_ptr[r * T + T] == grp_ptr[r * T]]
    assert lonely, "the fixture needs a node without neighbors"
    nodes = np.concatenate([g["ids"][rng.randint(0, n, size=40)], [ABSENT], g["ids"][:3], g["ids"][:3], lonely[:2]]).astype(np.int64)
    return dict(g=g, gr=gr, og=graphs.oracle_graph(g), nodes=nodes, lonely=np.asarray(lonely, np.int64))


def _install(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)
    return euler_b200


def _sparse_want(bags):
    """(indices, values, dense_shape) of the SparseTensor whose row i holds bags[i]"""
    idx = np.asarray([(i, k) for i, b in enumerate(bags) for k in range(len(b))], np.int64).reshape(-1, 2)
    return idx, np.asarray([v for b in bags for v in b], np.int64), (len(bags), max((len(b) for b in bags), default=0))


def _eq_sparse(got, want, what):
    idx, vals, shape = got
    assert idx.is_cuda and idx.dtype == torch.int64 and vals.dtype == torch.int64, what
    assert tuple(idx.shape) == (len(want[1]), 2) and tuple(vals.shape) == (len(want[1]),), what
    assert np.array_equal(idx.cpu().numpy(), want[0]) and np.array_equal(vals.cpu().numpy(), want[1]), what
    assert shape == want[2] and all(type(x) is int for x in shape), (what, shape, want[2])


def _bags(env, nodes, slot, default):
    g = env["g"]
    return er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, slot, default)


def _listing(env, nodes, et):
    """get_full_neighbor's listing per node: [(ids, weights, types)]"""
    lens, ids, w, t = env["og"].get_full_neighbor(np.asarray(nodes, np.int64).astype(np.uint64), et)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return [(ids[off[i]:off[i + 1]].astype(np.int64), w[off[i]:off[i + 1]], t[off[i]:off[i + 1]]) for i in range(len(lens))]


# ------------------------------------------------------------------------------------ features
def test_node_sparse_and_binary_features(env):
    eb = _install(env)
    nodes = env["nodes"]
    got = eb.get_sparse_feature(nodes, ["u64_0", "u64_1", "nope"], [7, 0, 5])
    for k, (slot, dv) in enumerate(((0, 7), (1, 0), (-1, 5))):
        _eq_sparse(got[k], _sparse_want(_bags(env, nodes, slot, dv)), "slot %d" % slot)
    _eq_sparse(eb.get_sparse_feature(nodes, ["u64_1"])[0], _sparse_want(_bags(env, nodes, 1, 0)), "default_values=None")
    no_values = [int(i) for r, i in enumerate(env["g"]["ids"]) if env["g"]["u64_ptr"][2 * r] == env["g"]["u64_ptr"][2 * r + 1]]
    assert no_values
    _eq_sparse(eb.get_sparse_feature(no_values, ["u64_0"], [9])[0], _sparse_want([[9]] * len(no_values)), "all default")
    _eq_sparse(eb.get_sparse_feature(np.zeros(0, np.int64), ["u64_0"])[0], _sparse_want([]), "empty batch")
    assert eb.get_sparse_feature(nodes, []) == []
    rows = {int(i): b for i, b in zip(env["g"]["ids"], env["g"]["bin_rows"])}
    want = [rows.get(int(i), b"") for i in nodes]
    assert eb.get_binary_feature(nodes, ["bin_0", "nope"]) == [want, [b""] * len(nodes)]
    empty = [int(i) for i, b in rows.items() if not b]
    assert empty and eb.get_binary_feature(empty, ["bin_0"]) == [[b""] * len(empty)]    # a total of zero
    assert eb.get_binary_feature(np.zeros(0, np.int64), ["bin_0"]) == [[]]


def test_tiny_directory_node_and_edge_features(tiny_dir):
    import euler_b200 as eb
    eb.set_graph(eb.Graph.load(tiny_dir))
    _eq_sparse(eb.get_sparse_feature([1, -1, 2], ["f1"], [77])[0], _sparse_want([[11, 12], [77], [21, 22]]), "tiny f1")
    _eq_sparse(eb.get_sparse_feature([1, 2], ["nope"], [5])[0], _sparse_want([[5], [5]]), "tiny unknown")
    edges = [[1, 2, 0], [9, 9, 0], [2, 3, 1]]
    f1, f2, nope = eb.get_edge_sparse_feature(edges, ["f1", "f2", "nope"], [3, 0, 4])
    _eq_sparse(f1, _sparse_want([[121, 122], [3], [231, 232]]), "edge f1")
    _eq_sparse(f2, _sparse_want([[123, 124], [0], [233, 234]]), "edge f2")
    _eq_sparse(nope, _sparse_want([[4], [4], [4]]), "edge unknown")
    _eq_sparse(eb.get_edge_sparse_feature(edges[:1], ["f1"])[0], _sparse_want([[121, 122]]), "edge default_values=None")
    _eq_sparse(eb.get_edge_sparse_feature(np.zeros((0, 3), np.int64), ["f1"])[0], _sparse_want([]), "edge empty")
    assert eb.get_edge_binary_feature(edges, ["f5", "nope"]) == [[b"12a", b"", b"23a"], [b"", b"", b""]]
    assert eb.get_edge_binary_feature(np.zeros((0, 3), np.int64), ["f5"]) == [[]]
    assert eb.get_binary_feature([99, 1], ["f5"]) == [[b"", b"1a"]]
    with pytest.raises(eb.EulerError):
        eb.get_edge_sparse_feature([[1, 2]], ["f1"])


# ------------------------------------------------------------------------------------ full listings
@pytest.mark.parametrize("et", ([0], [1, 0], [0, 1, 1]))
def test_full_and_sorted_listings(env, et):
    eb = _install(env)
    for nodes in (env["nodes"], env["lonely"], np.zeros(0, np.int64)):
        lst = _listing(env, nodes, et)
        ptr = np.concatenate([[0], np.cumsum([len(x[0]) for x in lst])]).astype(np.int64)
        for sort in (False, True):
            got = (eb.get_sorted_full_neighbor(nodes, et) if sort else eb.get_full_neighbor(nodes, et))
            assert [x.dtype for x in got] == [torch.int64, torch.int64, torch.float32, torch.int32]
            assert np.array_equal(got[0].cpu().numpy(), ptr)
            order = [np.argsort(x[0], kind="stable") if sort else np.arange(len(x[0])) for x in lst]
            for j in range(3):
                want = np.concatenate([x[j][o] for x, o in zip(lst, order)] + [np.zeros(0, got[j + 1].cpu().numpy().dtype)])
                assert np.array_equal(got[j + 1].cpu().numpy(), want), (et, sort, j)


def _first_occurrence(ids):
    seen = {}
    for i in ids:
        seen.setdefault(int(i), len(seen))
    return seen


@pytest.mark.parametrize("self_loops", (True, False))
def test_full_neighbor_hop_and_adjacency(env, self_loops):
    eb = _install(env)
    et = [1, 0]
    for nodes in (env["nodes"], env["lonely"], np.zeros(0, np.int64)):
        lst = _listing(env, nodes, et)
        listed = np.concatenate([x[0] for x in lst] + [np.zeros(0, np.int64)])
        pos = _first_occurrence(np.concatenate([listed, nodes]))
        n_id, res, ei, types = eb.full_neighbor_hop(nodes, et, self_loops=self_loops, with_types=True)
        assert n_id.cpu().numpy().tolist() == list(pos)
        assert res.cpu().numpy().tolist() == [pos[int(i)] for i in nodes]
        rows = [r for r, x in enumerate(lst) for _ in x[0]]
        want = [rows, [pos[int(i)] for i in listed]]
        if self_loops:
            want = [want[0] + list(range(len(nodes))), want[1] + [pos[int(i)] for i in nodes]]
        assert ei.dtype == torch.int64 and ei.cpu().numpy().reshape(2, -1).tolist() == want
        assert types.cpu().numpy().tolist() == np.concatenate([x[2] for x in lst] + [np.zeros(0, np.int32)]).tolist()
        nxt, indptr, cols, w = eb.full_neighbor_adjacency(nodes, et)
        col = _first_occurrence(listed)
        assert nxt.cpu().numpy().tolist() == list(col)
        assert indptr.cpu().numpy().tolist() == np.concatenate([[0], np.cumsum([len(x[0]) for x in lst])]).tolist()
        want_c, want_w = [], []
        for ids, ws, _ in lst:
            c = np.asarray([col[int(i)] for i in ids], np.int64)
            o = np.argsort(c, kind="stable")
            want_c += c[o].tolist()
            want_w += ws[o].tolist()
        assert cols.cpu().numpy().tolist() == want_c and w.cpu().numpy().tolist() == want_w


def test_sparse_adjacency_with_an_empty_row(env):
    eb = _install(env)
    et = [0, 1]
    g = env["g"]
    lonely = env["lonely"]
    nodes = np.stack([g["ids"][:4].astype(np.int64), np.repeat(lonely[:1], 4), g["ids"][4:8].astype(np.int64)])
    nb = np.stack([g["nbr"][:3].astype(np.int64), g["ids"][:3].astype(np.int64), np.asarray([ABSENT] * 3)])
    adj_set = [set(x[0].tolist()) for x in _listing(env, nodes.reshape(-1), et)]
    batch, N, M = 3, 4, 3
    want_idx, want_val = [], []
    for b in range(batch):
        hits = [[b, j, k] for j in range(N) for k in range(M) if int(nb[b, k]) in adj_set[b * N + j]]
        want_idx += hits
        want_val += [1] * len(hits)
        if [b, N - 1, M - 1] not in hits:     # the filler that closes the batch row
            want_idx.append([b, N - 1, M - 1])
            want_val.append(0)
    assert [v for i, v in zip(want_idx, want_val) if i[0] == 1] == [0], "row 1 is the empty row"
    idx, vals, shape = eb.sparse_get_adj_coo(nodes.reshape(-1), nb.reshape(-1), et, N, M)
    assert shape == (batch, N, M)
    assert idx.cpu().numpy().tolist() == want_idx and vals.cpu().numpy().tolist() == want_val
    dense = eb.sparse_get_adj(nodes.reshape(-1), nb.reshape(-1), et, N, M).cpu().numpy()
    assert np.argwhere(dense > 0).tolist() == [i for i, v in zip(want_idx, want_val) if v]
    idx, vals, shape = eb.sparse_get_adj_coo(np.zeros(0, np.int64), np.zeros(0, np.int64), et)
    assert tuple(idx.shape) == (0, 3) and vals.numel() == 0 and shape == (0, 0, 0)


# ------------------------------------------------------------------------------------ fanout family and walks
def test_fanout_family_empty_and_lonely_inputs(env):
    eb = _install(env)
    ets, counts = [[0, 1], [1, 0]], [3, 2]
    ids, ws, ts = eb.sample_fanout(np.zeros(0, np.int64), ets, counts)
    assert [tuple(x.shape) for x in ids] == [(0,)] * 3 and [tuple(x.shape) for x in ws + ts] == [(0,)] * 4
    ids, ws, ts = eb.sample_fanout(env["lonely"], ets, counts, default_node=-7)
    B = len(env["lonely"])
    assert (ids[1] == -7).all() and (ids[2] == -7).all() and tuple(ids[2].shape) == (B * 6,)
    assert (ws[1] == 0).all() and (ts[1] == -1).all() and [x.dtype for x in ts] == [torch.int32] * 2
    assert eb.sample_fanout(env["nodes"], [], [])[0][0].shape == (len(env["nodes"]),)
    for bad in ([[0, 1], [1]], [[0]]):
        with pytest.raises(eb.EulerError):
            eb.sample_fanout(env["nodes"], bad, counts)
        with pytest.raises(eb.EulerError):
            eb.sample_fanout_with_feature(env["nodes"], bad, counts, 0, [], [], [], [])
        with pytest.raises(eb.EulerError):    # refused before any engine is needed: unequal lists, or one list for two hops
            eb.sample_fanout_batched(env["nodes"][None], bad, counts)
    assert tuple(eb.random_walk(np.zeros(0, np.int64), [[0], [1]]).shape) == (0, 3)
    assert eb.random_walk(env["lonely"][:2], [[0, 1]], default_node=-3).cpu().numpy().tolist() == [[int(i), -3] for i in env["lonely"][:2]]
    with pytest.raises(eb.EulerError):
        eb.random_walk(env["nodes"], [[0, 1], [1]])


def test_batched_fanout_is_the_single_call(env):
    eb = _install(env)
    ets, counts = [[0, 1], [1, 0]], [4, 3]
    ctx = eb.Context(env["gr"], "minstd", 1)
    ctx.set_engines(2, [31, 32])
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    nodes = np.stack([env["nodes"], env["nodes"][::-1]])
    ids, ws, ts = eb.sample_fanout_batched(nodes, ets, counts, -1, ctx=ctx)
    assert [tuple(x.shape) for x in ids] == [(2, len(env["nodes"]) * k) for k in (1, 4, 12)]
    for b, s in enumerate((31, 32)):
        eb.seed(s)
        one = eb.sample_fanout(nodes[b], ets, counts)
        for got, want in zip(ids + ws + ts, one[0] + one[1] + one[2]):
            assert torch.equal(got[b], want)
    ids, _, _ = eb.sample_fanout_batched(np.zeros((2, 0), np.int64), ets, counts, ctx=ctx)
    assert [tuple(x.shape) for x in ids] == [(2, 0)] * 3


def test_fanout_with_feature_sparse_triples(env):
    eb = _install(env)
    ets, counts, nodes = [[0, 1], [1, 0]], [3, 2], env["nodes"]
    eb.seed(5)
    plain = eb.sample_fanout(nodes, ets, counts, 0)
    eb.seed(5)
    ids, ws, ts, dense, sparse = eb.sample_fanout_with_feature(nodes, ets, counts, 0, [], [], ["u64_0", "nope", "u64_1"], [7, 5, 0])
    assert dense == [] and len(sparse) == 9
    B = len(nodes)
    assert [tuple(x.shape) for x in ws] == [(B, 3), (B, 3, 2)] and [tuple(x.shape) for x in ids] == [(B,), (B * 3,), (B * 6,)]
    for l in range(3):
        assert torch.equal(ids[l], plain[0][l])
        hop = ids[l].cpu().numpy()
        for j, (slot, dv) in enumerate(((0, 7), (-1, 5), (1, 0))):
            _eq_sparse(sparse[3 * l + j], _sparse_want(_bags(env, hop, slot, dv)), "hop %d slot %d" % (l, slot))
    out = eb.sample_fanout_with_feature(np.zeros(0, np.int64), ets, counts, 0, [], [], ["u64_0"], [7])
    for triple in out[4]:
        _eq_sparse(triple, _sparse_want([]), "empty batch")


# ------------------------------------------------------------------------------------ table gradients
def _check_sparse_grad(dense, sparse, touched, what):
    """sparse is the coalesced COO form of dense over exactly the touched rows"""
    assert sparse.is_sparse and sparse.shape == dense.shape, what
    rows = sparse._indices()[0].cpu().numpy()
    assert rows.tolist() == sorted(set(int(r) for r in touched)), what
    assert sparse.to_dense().cpu().numpy().tobytes() == dense.cpu().numpy().tobytes(), what
    untouched = np.setdiff1d(np.arange(dense.shape[0]), rows)
    assert not dense[torch.as_tensor(untouched, device=dense.device)].any(), what


def _leaf(rng, rows, dim):
    return torch.tensor(rng.randint(-8, 9, size=(rows, dim)) / 8.0, dtype=torch.float32, device="cuda", requires_grad=True)


@pytest.mark.parametrize("n_rows", (8, 50))
def test_sparse_embedding_gradients(env, n_rows):
    """u64_1's values lie in [0, 8): with 8 rows the batch has more entries than the table has rows"""
    eb = _install(env)
    rng = np.random.RandomState(n_rows)
    nodes = env["nodes"]
    slot = 1 if n_rows == 8 else 0
    bags = _bags(env, nodes, slot, n_rows - 1)
    g_out = torch.tensor(rng.randint(-4, 5, size=(len(nodes), 3)) / 4.0, dtype=torch.float32, device="cuda")
    grads = []
    for sparse_grad in (False, True):
        t = _leaf(rng, n_rows, 3)
        eb.sparse_feature_embedding(nodes, "u64_%d" % slot, t, n_rows - 1, "mean", sparse_grad=sparse_grad).backward(g_out)
        grads.append(t.grad)
    want = er.grad_f64(g_out.cpu().numpy(), bags, n_rows, "mean")
    assert np.abs(grads[0].cpu().numpy() - want).max() <= 1e-6
    _check_sparse_grad(grads[0], grads[1], [v for b in bags for v in b], "sparse embedding")


@pytest.mark.parametrize("with_id", (True, False))
def test_shallow_encoder_gradients(env, with_id):
    eb = _install(env)
    nodes = env["nodes"][env["nodes"] != ABSENT]
    n_id = int(nodes.max()) + 1
    grads = []
    for sparse_grad in (False, True):
        rs = np.random.RandomState(9)
        tabs = ([_leaf(rs, n_id, 4)] if with_id else []) + [_leaf(rs, 50, 4), _leaf(rs, 8, 4)]
        id_t, s0, s1 = (tabs if with_id else [None] + tabs)
        out = eb.shallow_encode(nodes, id_t, [], [("u64_0", s0, 49), (1, s1, 7, "mean")], "concat", sparse_grad=sparse_grad)
        out.backward(torch.ones_like(out))
        grads.append([None if t is None else t.grad for t in (id_t, s0, s1)])
    touched = [nodes, [v for b in _bags(env, nodes, 0, 49) for v in b], [v for b in _bags(env, nodes, 1, 7) for v in b]]
    for k in range(3):
        if not with_id and k == 0:
            assert grads[0][0] is None and grads[1][0] is None
            continue
        _check_sparse_grad(grads[0][k], grads[1][k], touched[k], "shallow table %d" % k)
    if with_id:
        want = np.zeros((n_id, 4))
        np.add.at(want, nodes, 1.0)
        assert np.array_equal(grads[0][0].cpu().numpy(), want)


@pytest.mark.parametrize("shared", (False, True))
def test_skipgram_gradients(env, shared):
    eb = _install(env)
    rng = np.random.RandomState(11 + shared)
    n_rows, B, P, K = 40, 300, 2, 3
    src, pos, negs = rng.randint(0, n_rows, size=B), rng.randint(0, n_rows // 2, size=(B, P)), rng.randint(0, n_rows, size=(B, K))
    grads = []
    for sparse_grad in (False, True):
        rs = np.random.RandomState(5)
        t = _leaf(rs, n_rows, 6)
        c = t if shared else _leaf(rs, n_rows, 6)
        loss, _ = eb.skipgram_xent_loss(src, pos, negs, t, c, sparse_grad=sparse_grad)
        loss.backward()
        grads.append((t.grad, None if shared else c.grad))
    wt, wc = sr.grads64(t.detach().cpu().numpy(), c.detach().cpu().numpy(), src, sr.context_ids(pos, negs), P)
    ctx_rows = np.concatenate([pos.reshape(-1), negs.reshape(-1)])
    if shared:
        assert grads[0][1] is None and grads[1][1] is None
        assert np.abs(grads[0][0].cpu().numpy() - (wt + wc)).max() <= 1e-5 * np.abs(wt + wc).max()
        _check_sparse_grad(grads[0][0], grads[1][0], np.concatenate([src, ctx_rows]), "shared table")
        return
    assert np.abs(grads[0][0].cpu().numpy() - wt).max() <= 1e-5 * np.abs(wt).max()
    assert np.abs(grads[0][1].cpu().numpy() - wc).max() <= 1e-5 * np.abs(wc).max()
    _check_sparse_grad(grads[0][0], grads[1][0], src, "target table")
    _check_sparse_grad(grads[0][1], grads[1][1], ctx_rows, "context table")


@pytest.mark.parametrize("model", ("transe", "transd"))
def test_kg_gradients(env, model):
    eb = _install(env)
    rng = np.random.RandomState(21)
    n_ent, n_rel, dim, B, K = 60, 7, 5, 200, 3
    src, dst, rel = rng.randint(0, n_ent - 3, size=B), rng.randint(0, n_ent - 3, size=B), rng.randint(0, n_rel - 1, size=B)
    neg = rng.randint(0, n_ent - 3, size=(B, K))
    shapes = [(n_ent, dim), (n_rel, dim)] + ([(n_ent, dim), (n_rel, dim)] if model == "transd" else [])
    grads = []
    for sparse_grad in (False, True):
        rs = np.random.RandomState(4)
        tabs = [_leaf(rs, *sh) for sh in shapes]
        loss, _ = eb.kg_margin_loss(src, dst, neg, rel, tabs, model, margin=4.0, sparse_grad=sparse_grad)
        loss.backward()
        grads.append([t.grad for t in tabs])
    from euler_b200.knowledge import composed_kg_loss     # the torch composition, differentiated in float64
    t64 = [t.detach().double().requires_grad_(True) for t in tabs]
    d = lambda a: torch.as_tensor(a, dtype=torch.int64, device="cuda")   # noqa: E731
    composed_kg_loss(model, t64, d(src), d(dst), d(neg), d(rel), margin=4.0)[0].backward()
    ent_rows = np.concatenate([src, dst, neg.reshape(-1)])
    for k in range(len(shapes)):
        assert grads[0][k].any(), (model, k)
        want = t64[k].grad
        assert float((grads[0][k].double() - want).abs().max()) <= 1e-5 * float(want.abs().max()), (model, k)
        _check_sparse_grad(grads[0][k], grads[1][k], ent_rows if k % 2 == 0 else rel, "%s table %d" % (model, k))
