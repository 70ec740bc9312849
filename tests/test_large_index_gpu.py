"""GPU: the table- and feature-reading kernels on tables and feature matrices past 2^31 elements, and the stochastic rounding
of bf16 tables past 2^32 elements, where a row's element offset no longer fits an int and, for bf16 tables, the Philox
counter's second word (element >> 32) is non-zero.  These are the sizes the bf16 features and tables exist for (tens of
millions of rows of width 128 or 256); the rest of the suite uses small tables.

Every test asserts that its largest touched row times the row width reaches the threshold it claims.  Ids include row 0,
the last row under the threshold, the first row at or above it, the last row, several hundred random rows above it, and one
high row repeated more than 256 times (the sparse gradients' distinct-row sums then span several chunks).  Tables are filled
on the device with random values, chunk by chunk.

References.  Dense features: the host's generator oracle.pyoracle.rmat_feat_rows (rounded to bf16 for a bf16 graph), the
reductions restated in their documented f32 order.  Id tables: the same op on the compact table T_big[touched] with the ids
remapped by searchsorted(touched, ids) -- the remap keeps row order, so the op's fixed summation order is unchanged and the
outputs, losses, ranks and sparse gradient values must be the same bits; the small-table ops themselves are checked against
float64 by the other test files.  Optimizers: optim_reference (f32) and sr_reference.step (bf16) on picked rows, the touched
rows and sampled untouched ones.

Each test needs at most about 26 GB of device memory (arithmetic, noted per test), frees it at the end, and skips when the
device has less free.  The dense optimizer form at 2^32 elements is left out: a bf16 var, slots and f32 gradient of that size
need 34 GB or more, and k_opt_dense computes its element index as the sparse path does, which runs past 2^32 here."""
import gc

import numpy as np
import pytest
import torch

import bf16_reference as bf
import embedding_reference as er
import graphs  # noqa: F401  (sys.path)
import optim_reference as ref
import sr_reference as sr

pytestmark = pytest.mark.gpu
T31, T32 = 1 << 31, 1 << 32
D = 128
N31 = (1 << 24) + (1 << 13)   # rows of a width-128 table past 2^31 + 2^20 elements
N32 = (1 << 25) + (1 << 13)   # past 2^32 + 2^20
GB = float(1 << 30)
SEED = 0xDEADBEEF12345678
ESIZE = {torch.float32: 4, torch.bfloat16: 2}


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _need(nbytes):
    """skip unless the device has nbytes free, with 1 GB to spare for the op's own buffers"""
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + (1 << 30):
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (nbytes / GB, free / GB))


def _rand(shape, dtype, lo=-1.0, hi=1.0, seed=0, offset=0):
    """a contiguous device tensor of uniform random values in [lo, hi), filled 2^28 elements at a time; offset puts its data
    that many elements into its buffer"""
    n = int(np.prod(shape))
    buf = torch.empty(n + offset, dtype=dtype, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    step = 1 << 28
    for a in range(offset, n + offset, step):
        buf[a:min(a + step, n + offset)].uniform_(lo, hi, generator=g)
    return buf[offset:].view(shape)


def _pick(rng, n, first, k=300):
    """row 0, the last row under `first`, `first`, the last row and k random rows in [first, n)"""
    return np.concatenate([[0, first - 1, first, n - 1], rng.randint(first, n, size=k)]).astype(np.int64)


def _reached(ids, width, threshold):
    assert int(np.max(np.asarray(ids))) * width >= threshold, "the largest touched row stays under the claimed threshold"


def _dev(x, dtype=torch.int64):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).cuda()


def _compact(ids):
    """(touched: the sorted unique ids i64 on the device, remap(ids) -> the same ids as rows of T_big[touched])"""
    touched = torch.unique(torch.cat([_dev(i).reshape(-1) for i in ids]))
    return touched, lambda i: torch.searchsorted(touched, _dev(i).reshape(-1)).reshape(np.shape(i))


def _same(a, b, what):
    a, b = a.detach(), b.detach()
    assert a.dtype == b.dtype and a.shape == b.shape, what
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    assert torch.equal(a, b), what


def _same_sparse(big, small, touched, what):
    """a sparse gradient (rows, values) of T_big equals the one of T_small: rows mapped back, values to the bit"""
    (rb, vb), (rs, vs) = big, small
    assert torch.equal(rb, touched[rs]), what + " rows"
    _same(vb, vs, what + " values")


def _coo(g):
    g = g.coalesce() if not g.is_coalesced() else g
    return g._indices()[0], g._values()


@pytest.fixture
def eb():
    import euler_b200
    g = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    return euler_b200


# ------------------------------------------------------------------------------------------------ skip-gram
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("K", [5, 0])
def test_skipgram_on_tables_past_2_31(eb, dtype, K):
    """target and context both [2^24 + 2^13, 128]: 17.2 GB in f32, 8.6 GB in bf16"""
    from euler_b200 import ops
    _need(2 * N31 * D * ESIZE[dtype])
    rng = np.random.RandomState(1 + K)
    pool = _pick(rng, N31, T31 // D)
    B = 1000
    src, pos, negs = rng.choice(pool, B), rng.choice(pool, (B, 1)), rng.choice(pool, (B, K))
    src[:4], pos[:4, 0] = pool[:4], pool[:4][::-1]
    hot = pool[3]
    src[100:400] = hot
    if K:
        negs[:400, 2] = hot
    else:
        pos[:400, 0] = hot
    _reached(np.concatenate([src, pos.reshape(-1), negs.reshape(-1)]), D, T31)
    target, context = _rand((N31, D), dtype, seed=1), _rand((N31, D), dtype, seed=2)
    touched, remap = _compact([src, pos, negs])
    t_small, c_small = target[touched], context[touched]
    big = ops._raw_skipgram(_dev(src), _dev(pos), _dev(negs).reshape(B, K), target, context)
    small = ops._raw_skipgram(remap(src), remap(pos), remap(negs).reshape(B, K), t_small, c_small)
    for a, b, nm in zip(big, small, ("logits", "rank", "loss")):
        _same(a, b, nm)
    lb, mb, gb = ops.skipgram_xent_loss_sparse_grads(_dev(src), _dev(pos), _dev(negs).reshape(B, K), target, context)
    ls, ms, gs = ops.skipgram_xent_loss_sparse_grads(remap(src), remap(pos), remap(negs).reshape(B, K), t_small, c_small)
    _same(lb, ls, "loss")
    _same(mb, ms, "metric")
    for k, (a, b) in enumerate(zip(gb, gs)):
        _same_sparse(a, b, touched, "table %d gradient" % k)
    assert int((gb[0][0] == hot).sum()) == 1
    del target, context, t_small, c_small, big, small, gb, gs


# ------------------------------------------------------------------------------------------------ knowledge graphs
# per model: the tables' shapes and which ids index each ('e' entities, 'r' relations)
_KG = {
    'transe': ([(N31, D), (1000, D)], 'er'),
    'distmult': ([(N31, D), (1000, D)], 'er'),
    'transd': ([(N31, D), (1000, D), (N31, D), (1000, D)], 'erer'),
    'transr': ([(4096, D), (131200, D), (131200, D * D)], 'err'),
}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("model", sorted(_KG))
def test_kg_margin_loss_on_tables_past_2_31(eb, dtype, model):
    """TransE / DistMult: the entity table [2^24 + 2^13, 128] (8.6 GB f32); TransD: entity and entity_transfer (17.2 GB
    f32); TransR: transfer [131200, 128 x 128], 2^31 + 2^20 elements (8.6 GB f32), offsets rb * ent_dim * rel_dim"""
    from euler_b200 import ops
    shapes, kinds = _KG[model]
    _need(sum(r * c for r, c in shapes) * ESIZE[dtype])
    rng = np.random.RandomState(len(model))
    n_ent, n_rel = shapes[0][0], shapes[1][0]
    B, K = 600, 5
    ent_pool = _pick(rng, n_ent, T31 // D) if n_ent > T31 // D else np.arange(n_ent)
    rel_pool = _pick(rng, n_rel, T31 // (D * D)) if model == 'transr' else np.arange(n_rel)
    src, dst, neg = rng.choice(ent_pool, B), rng.choice(ent_pool, B), rng.choice(ent_pool, (B, K))
    rel = rng.choice(rel_pool, B)
    src[:4], dst[:4], rel[:4] = ent_pool[:4], ent_pool[:4][::-1], rel_pool[:4]
    neg[:400, 1] = ent_pool[3]   # one entity in 400 corruptions (and twice that under 'both')
    if model == 'transr':
        rel[100:400] = rel_pool[3]
        _reached(rel, D * D, T31)
    else:
        _reached(np.concatenate([src, dst, neg.reshape(-1)]), D, T31)
    tables = [_rand(s, dtype, -0.5, 0.5, seed=k) for k, s in enumerate(shapes)]
    te, remap_e = _compact([src, dst, neg])
    tr, remap_r = _compact([rel])
    touched = [te if c == 'e' else tr for c in kinds]
    small = [t[i] for t, i in zip(tables, touched)]
    args_big = (_dev(src), _dev(dst), _dev(neg), _dev(rel))
    args_small = (remap_e(src), remap_e(dst), remap_e(neg), remap_r(rel))
    lb, mb, gb, eb_ = ops.kg_margin_loss_sparse_grads(*args_big, tables, model, with_embeddings=True)
    ls, ms, gs, es = ops.kg_margin_loss_sparse_grads(*args_small, small, model, with_embeddings=True)
    _same(lb, ls, "loss")
    _same(mb, ms, "metric")
    for k, (a, b) in enumerate(zip(eb_, es)):
        _same(a, b, "embedding %d" % k)
    for k, (a, b) in enumerate(zip(gb, gs)):
        _same_sparse(a, b, touched[k], "%s table %d gradient" % (model, k))
    del tables, small, gb, gs


# ------------------------------------------------------------------------------------------------ ShallowEncoder's id table
def _id_table(dtype):
    t = _rand((N31, D), dtype, seed=5)
    return t.requires_grad_() if dtype == torch.float32 else t


def _table_grad(run, table, dtype):
    """(forward output, the sparse gradient (rows, values) of `table`) of run(table, proxies) for an upstream gradient of
    random values"""
    from euler_b200 import ops
    proxy = ops.table_proxy(table) if dtype == torch.bfloat16 else None
    out = run(table, proxy)
    g_out = torch.empty_like(out).uniform_(-1, 1, generator=torch.Generator(device="cuda").manual_seed(9))
    leaf = proxy if proxy is not None else table
    g, = torch.autograd.grad(out, leaf, g_out)
    return out.detach(), _coo(g)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("pool", [None, 'mean'])
def test_shallow_encode_id_table_past_2_31(eb, dtype, pool):
    """id_table [2^24 + 2^13, 128]: 8.6 GB in f32, 4.3 GB in bf16"""
    import euler_b200
    _need(N31 * D * ESIZE[dtype])
    rng = np.random.RandomState(7)
    ids = rng.choice(_pick(rng, N31, T31 // D), 1500)
    ids[:4] = _pick(rng, N31, T31 // D, 0)
    ids[200:500] = ids[3]
    _reached(ids, D, T31)
    table = _id_table(dtype)
    touched, remap = _compact([ids])
    small = table.detach()[touched]
    small = small.requires_grad_() if dtype == torch.float32 else small

    def run(nodes):
        if pool is None:
            return lambda t, q: euler_b200.shallow_encode(nodes, id_table=t, sparse_grad=True,
                                                          proxies=None if q is None else [q])
        return lambda t, q: euler_b200.shallow_encode_pool(nodes, 5, id_table=t, pool=pool, sparse_grad=True,
                                                           proxies=None if q is None else [q])
    ob, gb = _table_grad(run(_dev(ids)), table, dtype)
    os_, gs = _table_grad(run(remap(ids)), small, dtype)
    _same(ob, os_, "rows")
    if pool is None:   # the rows themselves, read by torch's int64 indexing
        _same(ob, table.detach()[_dev(ids)].float(), "rows vs torch")
    _same_sparse(gb, gs, touched, "id table gradient")
    del table, small, ob, gb, gs


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_sparse_feature_embedding_table_past_2_31(dtype):
    """a slot graph whose uint64 values are rows of a [2^24 + 2^13, 128] table: 8.6 GB in f32, 4.3 GB in bf16"""
    import euler_b200
    _need(N31 * D * ESIZE[dtype])
    rng = np.random.RandomState(11)
    vals = _pick(rng, N31, T31 // D)
    hot = int(vals[3])
    sg = er.slot_graph(5, 400, [lambda r, n: r.randint(0, 6, size=n)],
                       [lambda r, k: np.where(r.rand(k) < 0.3, hot, r.choice(vals, size=k))])
    default = int(vals[2])
    _reached(np.append(sg["u64_val"].astype(np.int64), default), D, T31)
    touched, remap = _compact([sg["u64_val"].astype(np.int64), [default]])
    nodes = _dev(sg["ids"][rng.randint(0, 400, size=2000)].astype(np.int64))
    table = _id_table(dtype)
    small = table.detach()[touched]
    small = small.requires_grad_() if dtype == torch.float32 else small

    def graph(u64_val):
        return euler_b200.Graph.from_csr(sg["ids"], sg["grp_ptr"], sg["nbr"], n_edge_types=sg["T"], node_type=sg["node_type"],
                                         node_w=sg["node_w"], cum_w=sg["cum_w"], u64_ptr=sg["u64_ptr"], u64_val=u64_val,
                                         n_u64_slots=sg["S"])
    outs = []
    for vals_, dv, t in ((sg["u64_val"], default, table), (remap(sg["u64_val"].astype(np.int64)).cpu().numpy(),
                                                           int(remap([default])[0]), small)):
        euler_b200.set_graph(graph(np.asarray(vals_, np.uint64)), rng="minstd", seed=1)
        outs.append(_table_grad(lambda tb, q: euler_b200.sparse_feature_embedding(nodes, "u64_0", tb, dv, 'mean',
                                                                                  sparse_grad=True, proxy=q), t, dtype))
    (ob, gb), (os_, gs) = outs
    assert int((gb[0] == hot).sum()) == 1
    _same(ob, os_, "rows")
    _same_sparse(gb, gs, touched, "table gradient")
    del table, small, outs, ob, gb, gs


# ------------------------------------------------------------------------------------------------ embedding stores
def test_store_exchange_and_accumulate_past_2_31(eb):
    """store and grad store [2^24 + 2^13, 128] f32: 17.2 GB"""
    from euler_b200 import ops
    _need(2 * N31 * D * 4)
    rng = np.random.RandomState(13)
    pool = _pick(rng, N31, T31 // D)
    ids = rng.choice(pool, 1500)
    ids[:4] = pool[:4]
    ids[300:700] = pool[3]   # repeats: the last occurrence wins the exchange; the accumulation sums 400 entries
    _reached(ids, D, T31)
    untouched = np.setdiff1d(np.concatenate([rng.randint(0, N31, size=200), [N31 - 2, T31 // D + 1]]), ids)
    store, gstore = _rand((N31, D), torch.float32, seed=1), _rand((N31, D), torch.float32, seed=2)
    touched, remap = _compact([ids])
    s_small, g_small = store[touched], gstore[touched]
    keep = [store[_dev(untouched)], gstore[_dev(untouched)]]
    rows = torch.empty((ids.size, D), device="cuda").uniform_(-1, 1)
    _same(ops.store_exchange(store, gstore, _dev(ids), rows), ops.store_exchange(s_small, g_small, remap(ids), rows), "taken")
    _same(store[touched], s_small, "store")
    _same(gstore[touched], g_small, "grad store")
    grad = torch.empty((ids.size // 5, D), device="cuda").uniform_(-1, 1)
    ops.store_accumulate(gstore, _dev(ids), grad, count=5, pool='mean')
    ops.store_accumulate(g_small, remap(ids), grad, count=5, pool='mean')
    _same(gstore[touched], g_small, "accumulated grad store")
    _same(store[_dev(untouched)], keep[0], "untouched store rows")
    _same(gstore[_dev(untouched)], keep[1], "untouched grad store rows")
    del store, gstore, s_small, g_small


# ------------------------------------------------------------------------------------------------ adjacency mean
def test_adjacency_mean_over_rows_past_2_31(eb):
    """x_neigh [2^24 + 2^13, 128] f32 (8.6 GB), the whole-graph matrix GCNEncoder.infer builds; a small CSR of high columns"""
    from euler_b200 import ops
    _need(N31 * D * 4)
    rng = np.random.RandomState(17)
    pool = _pick(rng, N31, T31 // D)
    deg = rng.randint(0, 12, size=400)
    deg[[5, 9]] = [300, 600]   # rows summed in several chunks
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    cols = rng.choice(pool, int(indptr[-1]))
    cols[:4] = pool[:4]
    cols[indptr[9]:indptr[10]] = pool[3]
    _reached(cols, D, T31)
    x = _rand((N31, D), torch.float32, seed=3)
    touched, remap = _compact([cols])
    x_small = x[touched]
    out = ops.adjacency_mean(x, (_dev(indptr), _dev(cols)))
    _same(out, ops.adjacency_mean(x_small, (_dev(indptr), remap(cols))), "mean")
    # rows of at most 256 entries: the plain left-to-right f32 sum over max(deg, 1e-7)
    xs, c = x_small.cpu().numpy(), remap(cols).cpu().numpy()
    want = np.zeros((deg.size, D), np.float32)
    for i in np.nonzero(deg <= 256)[0]:
        s = np.zeros(D, np.float32)
        for k in range(indptr[i], indptr[i + 1]):
            s = s + xs[c[k]]
        want[i] = s / np.float32(max(deg[i], 1e-7))
    short = torch.from_numpy(np.nonzero(deg <= 256)[0]).cuda()
    _same(out[short].cpu(), torch.from_numpy(want[deg <= 256]), "restated mean")
    del x, x_small, out


# ------------------------------------------------------------------------------------------------ gather and scatter
def test_gather_params_past_2_31(eb):
    """params [2^24 + 2^13, 128] f32: 8.6 GB"""
    from euler_b200 import ops
    _need(N31 * D * 4)
    rng = np.random.RandomState(19)
    idx = rng.choice(_pick(rng, N31, T31 // D), 2000)
    idx[:4] = _pick(rng, N31, T31 // D, 0)
    idx[500:900] = idx[3]
    _reached(idx, D, T31)
    params = _rand((N31, D), torch.float32, seed=4)
    _same(ops.gather(params, _dev(idx, torch.int32)), params[_dev(idx)], "gather")
    del params


@pytest.mark.parametrize("op", ["scatter_add", "scatter_max"])
@pytest.mark.parametrize("order", ["sorted", "unsorted"])
def test_scatter_output_past_2_31(eb, op, order):
    """out [2^24 + 2^13, 128] f32: 8.6 GB.  Unsorted scatter_add adds with atomics in any order: its updates are small
    integers, whose sums are exact in every order."""
    from euler_b200 import ops
    _need(N31 * D * 4)
    rng = np.random.RandomState(23 + len(op) + len(order))
    pool = _pick(rng, N31, T31 // D)
    idx = rng.choice(pool, 3000)
    idx[:4] = pool[:4]
    idx[1000:1400] = pool[3]
    if order == "sorted":
        idx = np.sort(idx)
    _reached(idx, D, T31)
    if op == "scatter_add" and order == "unsorted":
        upd = torch.from_numpy(rng.randint(-64, 65, size=(idx.size, D)).astype(np.float32)).cuda()
    else:
        upd = torch.empty((idx.size, D), device="cuda").uniform_(-1, 1)
    fn = getattr(ops, op)
    touched, remap = _compact([idx])
    out = fn(upd, _dev(idx, torch.int32), N31)
    small = fn(upd, remap(idx).to(torch.int32), touched.numel())
    _same(out[touched], small, op)
    u, i = upd.cpu().numpy(), remap(idx).cpu().numpy()
    want = np.full((touched.numel(), D), 0 if op == "scatter_add" else -1e9, np.float64 if op == "scatter_add" else np.float32)
    (np.add if op == "scatter_add" else np.maximum).at(want, i, u)
    if op == "scatter_add":   # within 1e-5 of the terms' magnitudes; exact on the integer updates
        mag = np.zeros_like(want)
        np.add.at(mag, i, np.abs(u))
        assert np.all(np.abs(small.cpu().numpy() - want) <= 1e-5 * mag)
        if order == "unsorted":
            np.testing.assert_array_equal(small.cpu().numpy(), want.astype(np.float32))
    else:
        np.testing.assert_array_equal(small.cpu().numpy(), want)
    rest = _dev(np.setdiff1d(np.concatenate([rng.randint(0, N31, size=300), [N31 - 2, T31 // D + 1]]), idx))
    assert bool((out[rest] == (0.0 if op == "scatter_add" else -1e9)).all()), "untouched rows"
    del out, small


# ------------------------------------------------------------------------------------------------ optimizers
def _sparse(rows, vals, shape):
    return torch.sparse_coo_tensor(_dev(rows)[None], vals, shape, is_coalesced=True, check_invariants=False)


@pytest.mark.parametrize("name", ["momentum", "adagrad"])
def test_f32_sparse_optimizer_past_2_31(eb, name):
    """var and accumulator [2^24 + 2^13, 128] f32: 17.2 GB"""
    from euler_b200 import ops
    _need(2 * N31 * D * 4)
    rng = np.random.RandomState(29 + len(name))
    rows = np.unique(_pick(rng, N31, T31 // D))
    _reached(rows, D, T31)
    untouched = np.setdiff1d(np.concatenate([rng.randint(0, N31, size=300), [T31 // D - 2, T31 // D + 1, N31 - 2]]), rows)
    pick = np.concatenate([rows, untouched])
    var, acc = _rand((N31, D), torch.float32, seed=6), _rand((N31, D), torch.float32, 0.1, 1.0, seed=7)
    w0, a0 = var[_dev(pick)].cpu().numpy(), acc[_dev(pick)].cpu().numpy()
    vals = rng.randn(rows.size, D).astype(np.float32)
    grad = _sparse(rows, torch.from_numpy(vals).cuda(), (N31, D))
    if name == "momentum":
        ops.optim_momentum_(var, acc, grad, 0.05, 0.9)
        ref.momentum(w0, a0, (np.arange(rows.size), vals), 0.05, 0.9)
    else:
        ops.optim_adagrad_(var, acc, grad, 0.3)
        ref.adagrad(w0, a0, (np.arange(rows.size), vals), 0.3)
    _same(var[_dev(pick)].cpu(), torch.from_numpy(w0), "var")
    _same(acc[_dev(pick)].cpu(), torch.from_numpy(a0), "accumulator")
    del var, acc, grad


def _bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _bf16_slots(name, n, offset=0):
    """the bf16 slots of an optimizer over n x 128 rows: random, adagrad's accumulator and adam's v positive"""
    if name == "momentum":
        return [_rand((n, D), torch.bfloat16, -0.1, 0.1, seed=21, offset=offset)]
    if name == "adagrad":
        return [_rand((n, D), torch.bfloat16, 0.1, 1.0, seed=22, offset=offset)]
    return [_rand((n, D), torch.bfloat16, -0.1, 0.1, seed=23, offset=offset),
            _rand((n, D), torch.bfloat16, 0.0, 0.01, seed=24, offset=offset)]


def _bf16_step(name, var, slots, grad, powers, step):
    from euler_b200 import ops
    kw = dict(seed=SEED, step=step, tensor=3)
    if name == "adam":
        ops.optim_adam_(var, slots[0], slots[1], grad, powers, 0.01, 0.9, 0.999, 1e-8, **kw)
    elif name == "adagrad":
        ops.optim_adagrad_(var, slots[0], grad, 0.3, **kw)
    else:
        ops.optim_momentum_(var, slots[0], grad, 0.05, 0.9, **kw)


@pytest.mark.parametrize("name", ["momentum", "adagrad", "adam"])
def test_bf16_sparse_optimizer_past_2_32(eb, name):
    """var and slots [2^25 + 2^13, 128] bf16, 2^32 + 2^20 elements: 17.2 GB (momentum, adagrad), 25.8 GB (adam).  Rows on
    both sides of 2^32 / 128 draw their rounding bits with element high words 0 and 1."""
    _need((2 if name != "adam" else 3) * N32 * D * 2)
    rng = np.random.RandomState(31 + len(name))
    first = T32 // D
    rows = np.unique(np.concatenate([_pick(rng, N32, first), rng.randint(first - 2000, first, size=50)]))
    _reached(rows, D, T32)
    untouched = np.setdiff1d(np.concatenate([rng.randint(0, N32, size=200), rng.randint(first - 500, first + 500, size=50),
                                             [first - 2, first + 1, N32 - 2]]), rows)
    assert (untouched < first).any() and (untouched >= first).any()
    pick = np.concatenate([rows, untouched])
    var = _rand((N32, D), torch.bfloat16, -1, 1, seed=20)
    slots = _bf16_slots(name, N32)
    tables = [_bits(t[_dev(pick)]) for t in [var] + slots]
    vals = rng.randn(rows.size, D).astype(np.float32)
    powers = torch.tensor([0.9 ** 3, 0.999 ** 3], dtype=torch.float32, device="cuda")
    adam = None
    if name == "adam":
        adam = ref.Adam(0.01, 0.9, 0.999, 1e-8)
        adam.powers = powers.cpu().numpy()
    step = torch.tensor(7, dtype=torch.int64, device="cuda")
    _bf16_step(name, var, slots, _sparse(rows, torch.from_numpy(vals).cuda(), (N32, D)), powers, step)
    sr.step(name, tables, (np.arange(rows.size), vals), SEED, 7, 3, {"momentum": 0.05, "adagrad": 0.3}.get(name, 0.01),
            adam=adam, momentum=0.9, rows=pick)
    for k, t in enumerate([var] + slots):
        got = _bits(t[_dev(pick)])
        bad = pick[(got != tables[k]).any(axis=1)]
        assert bad.size == 0, "table %d: %d rows differ, %d of them under row 2^32 / D, the first %s" % (
            k, bad.size, int((bad < first).sum()), np.sort(bad)[:8])
    del var, slots


@pytest.mark.parametrize("name", ["momentum", "adam"])
@pytest.mark.parametrize("offset", [0, 1])
def test_bf16_dense_optimizer_past_2_31(eb, name, offset):
    """var and slots [2^24 + 2^13, 128] bf16 with an f32 gradient of that shape: 17.2 GB (momentum), 21.5 GB (adam); offset 1
    puts every table one element past its buffer's start, which takes the scalar path"""
    _need((2 if name == "momentum" else 3) * N31 * D * 2 + N31 * D * 4)
    rng = np.random.RandomState(37 + len(name) + offset)
    pick = np.unique(_pick(rng, N31, T31 // D, 400))
    _reached(pick, D, T31)
    var = _rand((N31, D), torch.bfloat16, -1, 1, seed=30, offset=offset)
    slots = _bf16_slots(name, N31, offset)
    grad = _rand((N31, D), torch.float32, seed=31, offset=offset)
    tables = [_bits(t[_dev(pick)]) for t in [var] + slots]
    g = grad[_dev(pick)].cpu().numpy()
    powers = torch.tensor([0.9 ** 2, 0.999 ** 2], dtype=torch.float32, device="cuda")
    adam = None
    if name == "adam":
        adam = ref.Adam(0.01, 0.9, 0.999, 1e-8)
        adam.powers = powers.cpu().numpy()
    step = torch.tensor(4, dtype=torch.int64, device="cuda")
    _bf16_step(name, var, slots, grad, powers, step)
    sr.step(name, tables, g, SEED, 4, 3, 0.05 if name == "momentum" else 0.01, adam=adam, momentum=0.9, rows=pick)
    for k, t in enumerate([var] + slots):
        np.testing.assert_array_equal(_bits(t[_dev(pick)]), tables[k], err_msg="table %d" % k)
    del var, slots, grad


# ------------------------------------------------------------------------------------------------ dense node features
FN, FE, FD = 8_500_000, 20_000_000, 256   # 2.18G feature elements: 8.7 GB as f32, 4.35 GB as bf16
FIRST = T31 // FD + 1                       # the first id whose row (id - 1) starts at or past 2^31 elements


@pytest.fixture(scope="module", params=["float32", "bfloat16"])
def feat_graph(request):
    import euler_b200
    _need(FN * FD * (4 if request.param == "float32" else 2) + (2 << 30))
    g = euler_b200.Graph.rmat(FN, FE, feat_dim=FD, feat_dtype=request.param)
    euler_b200.set_graph(g, rng="minstd", seed=1)
    probe = torch.tensor([1, FIRST - 1, FIRST, FN, 0, FN + 1], device="cuda")
    assert euler_b200.graph_node_rows(probe).tolist() == [0, FIRST - 2, FIRST - 1, FN - 1, -1, -1]   # row r is id r + 1
    assert FN * FD >= T31 + (1 << 20)
    yield euler_b200, request.param
    small = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(small), rng="minstd", seed=1)
    del g
    gc.collect()
    torch.cuda.empty_cache()


def _feat(ids, dtype, dim=FD):
    """the generator's rows of ids (zeros for non-nodes) as the graph stores them, f32[len(ids), dim] (zero-padded past FD)"""
    import oracle.pyoracle as po
    ids = np.asarray(ids, np.int64).reshape(-1)
    u, inv = np.unique(ids, return_inverse=True)
    rows = po.rmat_feat_rows(u, FN, FD, 7)
    if dtype == "bfloat16":
        rows = bf.rounded(rows)
    out = np.zeros((u.size, dim), np.float32)
    out[:, :min(dim, FD)] = rows[:, :min(dim, FD)]
    return out[inv.reshape(-1)]


def _feat_ids(rng, k=400):
    """node 1 (row 0), the last id under the threshold, the first at it, the last node, k random ids past it, and absent
    ids 0 and FN + 1"""
    return np.concatenate([[1, FIRST - 1, FIRST, FN], rng.randint(FIRST, FN + 1, size=k), [0, FN + 1]]).astype(np.int64)


@pytest.mark.parametrize("dim", [FD, 255, 300])
def test_dense_feature_rows_past_2_31(feat_graph, dim):
    eb, dt = feat_graph
    from euler_b200 import _lib
    ids = _feat_ids(np.random.RandomState(dim))
    _reached(ids - 1, FD, T31)
    want = _feat(ids, dt, dim)
    got = eb.get_dense_feature(_dev(ids), [0], [dim])[0]
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    if dim == FD:   # the host-buffer entry point
        out = np.zeros((ids.size, dim), np.float32)
        _lib.check(_lib.load().eu_get_dense_feature_host(eb.context()._h, ids.ctypes.data, ids.size, 0, dim, out.ctypes.data))
        np.testing.assert_array_equal(out, want)


@pytest.mark.parametrize("dim", [FD, 254])
@pytest.mark.parametrize("rows", [1000, (1 << 17) + 64])
def test_sage_mean_past_2_31(feat_graph, dim, rows):
    """dim 256 takes the 4-wide k_sage_mean, 254 k_sage_mean_generic; 2^17 rows and more take the dedup / broadcast path"""
    import oracle.pyoracle as po
    eb, dt = feat_graph
    rng = np.random.RandomState(dim + rows)
    count = 5 if rows < (1 << 17) else 2
    pool = np.concatenate([_feat_ids(rng, 20000), [0, FN + 7]])
    ids = rng.choice(pool, rows * count)
    ids[:4] = pool[:4]
    ids[count * 10:count * 600] = np.tile(ids[count * 9:count * 10], 590)   # one segment repeated 591 times
    _reached(ids - 1, FD, T31)
    got = eb.sage_mean_aggregate(_dev(ids), count, dim).cpu().numpy()
    want = po.scatter_mean(_feat(ids, dt, min(dim, FD)), np.repeat(np.arange(rows), count).astype(np.int32), rows)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("k", [3, 8, 16])
def test_neighbor_top_k_feature_past_2_31(feat_graph, k):
    eb, dt = feat_graph
    rng = np.random.RandomState(k)
    pool = _feat_ids(rng, 2000)
    B, count = 300, 20
    nodes, nbrs = rng.choice(pool, B), rng.choice(pool, (B, count))
    nodes[:6], nbrs[0, :6] = pool[[0, 1, 2, 3, -2, -1]], pool[[0, 1, 2, 3, -2, -1]]
    nbrs[1:4] = pool[3]   # a row of one neighbour: ties everywhere
    _reached(np.concatenate([nodes, nbrs.reshape(-1)]) - 1, FD, T31)
    got = eb.neighbor_top_k_feature(_dev(nodes), _dev(nbrs), 0, FD, k).cpu().numpy()
    x = _feat(nbrs, dt).reshape(B, count, FD)
    top = -np.sort(-x, axis=1, kind="stable")[:, :k]
    np.testing.assert_array_equal(got[:, 0], _feat(nodes, dt))
    np.testing.assert_array_equal(got[:, 1:], top)


@pytest.mark.parametrize("pool", [None, 'mean'])
def test_shallow_encode_dense_slot_past_2_31(feat_graph, pool):
    eb, dt = feat_graph
    rng = np.random.RandomState(41)
    ids = rng.choice(_feat_ids(rng), 1000)
    ids[:6] = _feat_ids(rng, 0)
    _reached(ids - 1, FD, T31)
    rows = _feat(ids, dt)
    if pool is None:
        got = eb.shallow_encode(_dev(ids), dense=[(0, FD)])
        np.testing.assert_array_equal(got.cpu().numpy(), rows)
        return
    got = eb.shallow_encode_pool(_dev(ids), 5, dense=[(0, FD)], pool=pool).cpu().numpy()
    r = rows.reshape(-1, 5, FD)
    s = r[:, 0].copy()
    for j in range(1, 5):   # left to right from the segment's first row, one division by count
        s = s + r[:, j]
    np.testing.assert_array_equal(got, s / np.float32(5))


def test_sample_fanout_with_feature_past_2_31(feat_graph):
    eb, dt = feat_graph
    rng = np.random.RandomState(43)
    seeds = _feat_ids(rng, 20000)[:-2]   # nodes only
    _reached(seeds - 1, FD, T31)
    nbrs, _, _, dense, _ = eb.sample_fanout_with_feature(_dev(seeds), [[0]], [10], -1, [0], [FD], [], [])
    hop = nbrs[1].cpu().numpy()
    assert (hop >= FIRST).any(), "no sampled id past the threshold"
    np.testing.assert_array_equal(dense[0].cpu().numpy(), _feat(seeds, dt))
    np.testing.assert_array_equal(dense[1].cpu().numpy(), _feat(hop, dt))
