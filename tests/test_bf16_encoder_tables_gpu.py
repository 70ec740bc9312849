"""GPU: the node encoders' bfloat16 tables.  sparse_feature_embedding, shallow_encode and shallow_encode_pool on bf16 tables
give the f32 op's bits on the widened tables (both feature dtypes, aligned and offset tables, every combiner and width, CUDA-
graph replay); each table's proxy receives, coalesced, the sparse gradient an f32 table holding the widened values gets with
sparse_grad=True, alone and summed over several uses in one graph, the same on every run; one optimizers.minimize step of
each model over ShallowEncoders equals the f32 step on widened tables, the bf16 tables and slots being tests/sr_reference.py's
rounding of that update; infer reads bf16 tables; 300 Adam steps track f32 training; refusals and bad ids change nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import bf16_reference as bf
import embedding_reference as er
import optim_reference as ref
import sr_reference as sr

pytestmark = pytest.mark.gpu
F32 = np.float32
N_NODES, N_ROWS, N_ID = 600, 1000, 1000   # graph ids 1 .. 600; slot u64_0's table rows; the ops' id table rows
SLOT_DIMS = (5, 12, 3)                     # dense slots feat0, feat1, feat2 (feat2 holds 0 / 1 labels)
ABSENT = (0, 650, 999)                     # ids the graph does not hold, inside the id table
DIMS = (1, 3, 4, 16, 128, 200)
DENSE = [("feat0", 8), ("feat1", 7), ("feat2", 3), (99, 2)]   # padded, clipped, as stored, unknown
MAX_ID = 700                               # the encoders' max_id: id table of 702 rows, default node 701
SLOT_MAX = [N_ROWS - 1, 59]                # the encoders' sparse_feature_max_id (tables of max + 2 rows)


def _lens_mixed(rng, n):   # 0 (default), 1, ordinary, and bags of more than 256 values
    k = rng.choice([0, 1, 2, 3, 5, 9], size=n, p=[0.3, 0.2, 0.2, 0.15, 0.1, 0.05])
    k[rng.choice(n, size=3, replace=False)] = [257, 300, 700]
    return k


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = er.slot_graph(5, N_NODES, [_lens_mixed, lambda rng, n: rng.randint(1, 4, size=n)],
                      [lambda rng, k: rng.randint(0, N_ROWS - 1, size=k), lambda rng, k: rng.randint(0, 50, size=k)],
                      feat_dim=sum(SLOT_DIMS))
    g["feat"] = np.ascontiguousarray(g["feat"], F32)
    g["feat"][:, 17:20] = (g["feat"][:, 17:20] > 0).astype(F32)
    graphs = {dt: euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                            node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=list(SLOT_DIMS),
                                            u64_ptr=g["u64_ptr"], u64_val=g["u64_val"], n_u64_slots=g["S"], feat_dtype=dt)
              for dt in ("float32", "bfloat16")}
    rng = np.random.RandomState(2)
    nodes = np.concatenate([g["ids"][rng.randint(0, N_NODES, size=700)], ABSENT, g["ids"][:5], g["ids"][:5]]).astype(np.int64)
    return dict(g=g, graphs=graphs, nodes=torch.as_tensor(nodes, device="cuda"))


def _install(env, feat="float32"):
    import euler_b200
    euler_b200.set_graph(env["graphs"][feat], rng="minstd", seed=1)


@pytest.fixture(autouse=True)
def _installed(env):
    _install(env)


def _bf16(n, dim, seed, offset=0, scale=0.3):
    """a bf16 table [n, dim] of rounded normal draws whose data lies `offset` elements past an 8-byte boundary"""
    bits = bf.round_bits(np.random.RandomState(seed).randn(n, dim).astype(F32) * F32(scale)).reshape(-1)
    buf = torch.zeros(bits.size + offset, dtype=torch.int16, device="cuda")
    buf[offset:] = torch.from_numpy(bits.view(np.int16)).cuda()
    return buf.view(torch.bfloat16)[offset:].view(n, dim)


def _bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    x, y = (a.view(torch.int32), b.view(torch.int32)) if a.dtype == torch.float32 else (a, b)
    assert torch.equal(x, y), what


def _same_sparse(a, b, what):
    a, b = a.coalesce(), b.coalesce()
    assert a.shape == b.shape, what
    assert torch.equal(a.indices(), b.indices()), what
    _same(a.values(), b.values(), what)


SLOTS = [("u64_0", N_ROWS, N_ROWS - 1, "sum"), ("u64_1", 60, 55, "mean"), ("no_such_slot", 20, 7, "sqrtn")]


def _sparse(n, dim, offset, seed=10, dims=None):
    """n sparse slots over SLOTS, cycled: [(name, bf16 table, default, combiner)]"""
    out = []
    for k in range(n):
        name, rows, dv, c = SLOTS[k % len(SLOTS)]
        out.append((name, _bf16(rows, dims[k] if dims else dim, seed + k, offset), dv, c))
    return out


def _widened(sparse):
    return [(n, t.float(), dv, c) for n, t, dv, c in sparse]


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("dim", DIMS)
def test_sparse_feature_embedding_forward(env, dim):
    import euler_b200
    for feat in ("float32", "bfloat16"):
        _install(env, feat)
        for off in (0, 1, 4):   # aligned; scalar; 8-byte aligned only (bf16's 4-wide path, which f32 would not take)
            t16 = _bf16(N_ROWS, dim, dim + off, off)
            t32 = t16.float()
            for comb in ("sum", "mean", "sqrtn"):
                for slot, dv in (("u64_0", N_ROWS - 1), ("no_such_slot", 3)):
                    a = euler_b200.sparse_feature_embedding(env["nodes"], slot, t16, dv, comb)
                    b = euler_b200.sparse_feature_embedding(env["nodes"], slot, t32, dv, comb)
                    _same(a, b, (feat, dim, off, comb, slot))


@pytest.mark.parametrize("dim", DIMS)
def test_shallow_encode_forward(env, dim):
    import euler_b200
    for feat in ("float32", "bfloat16"):
        _install(env, feat)
        for off in (0, 1, 4):
            id16 = _bf16(N_ID, dim, 1, off)
            for n in (1, 2, 3, 8):
                sp = _sparse(n, dim, off, dims=[dim if k % 2 == 0 else max(1, dim // 2) for k in range(n)])
                for dense in (DENSE, []):
                    a = euler_b200.shallow_encode(env["nodes"], id16, dense, sp, "concat")
                    b = euler_b200.shallow_encode(env["nodes"], id16.float(), dense, _widened(sp), "concat")
                    _same(a, b, (feat, dim, off, n, len(dense), "concat"))
                sp = _sparse(n, dim, off)
                a, fa = euler_b200.shallow_encode(env["nodes"], id16, DENSE, sp, "add")
                b, fb = euler_b200.shallow_encode(env["nodes"], id16.float(), DENSE, _widened(sp), "add")
                _same(a, b, (feat, dim, off, n, "add"))
                _same(fa, fb, (feat, dim, off, n, "add feats"))
                a = euler_b200.shallow_encode(env["nodes"], None, DENSE[:2], sp, "concat")   # no id table
                b = euler_b200.shallow_encode(env["nodes"], None, DENSE[:2], _widened(sp), "concat")
                _same(a, b, (feat, dim, off, n, "no id"))


@pytest.mark.parametrize("count", (1, 2, 5, 25, 64, 512))
def test_shallow_encode_pool_forward(env, count):
    import euler_b200
    rng = np.random.RandomState(count)
    R = max(2, 1024 // count)
    pool_ids = np.concatenate([env["g"]["ids"].astype(np.int64), ABSENT, [MAX_ID + 1]])
    nodes = torch.as_tensor(rng.choice(pool_ids, size=R * count), device="cuda")
    for feat in ("float32", "bfloat16"):
        _install(env, feat)
        for dim in (3, 16, 128):
            for off in (0, 1, 4):
                id16 = _bf16(N_ID, dim, 2, off)
                sp = _sparse(3, dim, off)
                for pool in ("sum", "mean"):
                    a = euler_b200.shallow_encode_pool(nodes, count, id16, DENSE, sp, pool)
                    b = euler_b200.shallow_encode_pool(nodes, count, id16.float(), DENSE, _widened(sp), pool)
                    _same(a, b, (feat, count, dim, off, pool))


def test_forward_captures_in_a_cuda_graph(env):
    import euler_b200
    nodes = env["nodes"]
    id16, sp = _bf16(N_ID, 16, 3, 4), _sparse(3, 16, 4)
    pool_nodes = nodes[:700]
    calls = [lambda: euler_b200.shallow_encode(nodes, id16, DENSE, sp, "concat"),
             lambda: euler_b200.shallow_encode_pool(pool_nodes, 7, id16, DENSE, sp, "mean"),
             lambda: euler_b200.sparse_feature_embedding(nodes, "u64_0", sp[0][1], N_ROWS - 1, "mean")]
    for k, fn in enumerate(calls):
        eager = fn()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
            cg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(cg, stream=s):
                out = fn()
        torch.cuda.current_stream().wait_stream(s)
        out.zero_()
        cg.replay()
        torch.cuda.synchronize()
        _same(out, eager, k)


# ------------------------------------------------------------------------------------------------ gradients
def _proxy_grads(fn, tables):
    """fn(tables, proxies) -> output; the proxies' .grad (coalesced) after backward of sum(out * G)"""
    import euler_b200
    proxies = [None if t is None else euler_b200.table_proxy(t) for t in tables]
    out = fn(tables, proxies)
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(4)).cuda()
    (out * G).sum().backward()
    return [None if q is None or q.grad is None else q.grad.coalesce() for q in proxies]


def _f32_grads(fn, tables):
    leaves = [None if t is None else t.float().requires_grad_() for t in tables]
    out = fn(leaves, None)
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(4)).cuda()
    (out * G).sum().backward()
    return [None if t is None or t.grad is None else t.grad.coalesce() for t in leaves]


def _check_grads(fn, tables, what):
    g16 = _proxy_grads(fn, tables)
    g32 = _f32_grads(fn, tables)
    again = _proxy_grads(fn, tables)
    for k, (a, b, c) in enumerate(zip(g16, g32, again)):
        if a is None:
            continue
        assert a.is_sparse and a.dtype == torch.float32
        _same_sparse(a, b, what + (k,))
        _same_sparse(a, c, what + (k, "repeat"))


@pytest.mark.parametrize("dim", (3, 16, 128))
def test_op_gradients_reach_the_proxies(env, dim):
    import euler_b200
    nodes = env["nodes"]
    for off in (0, 4):
        tables = [_bf16(N_ID, dim, 5, off)] + [t for _, t, _, _ in _sparse(3, dim, off)]
        meta = [(n, dv, c) for n, _, dv, c in SLOTS]

        def sp(ts):
            return [(n, t, dv, c) for (n, dv, c), t in zip(meta, ts[1:])]

        for comb in ("sum", "mean", "sqrtn"):
            _check_grads(lambda ts, qs: euler_b200.sparse_feature_embedding(
                nodes, "u64_0", ts[1], N_ROWS - 1, comb, sparse_grad=qs is None, proxy=qs and qs[1]), tables, ("sfe", comb, off))
        for combiner in ("concat", "add"):
            def enc(ts, qs, combiner=combiner):
                res = euler_b200.shallow_encode(nodes, ts[0], DENSE, sp(ts), combiner, sparse_grad=qs is None, proxies=qs)
                return res if combiner == "concat" else res[0]
            _check_grads(enc, tables, ("encode", combiner, off))
        for pool in ("sum", "mean"):
            _check_grads(lambda ts, qs: euler_b200.shallow_encode_pool(
                nodes[:700], 7, ts[0], DENSE, sp(ts), pool, sparse_grad=qs is None, proxies=qs), tables, ("pool", pool, off))


def _encoder_kw(dt, **kw):
    return dict(feature_idx=["feat0", "feat1"], feature_dim=[5, 12], max_id=MAX_ID, use_id=True,
                sparse_feature_idx=["u64_0", "u64_1"], sparse_feature_max_id=SLOT_MAX, embedding_dim=[16, 8, 4],
                device="cuda", table_dtype=dt, **kw)


def _pair(build):
    """(bf16 model, f32 model with sparse_grad=True holding the same parameters, its tables the widened bf16 ones)"""
    torch.manual_seed(0)
    m16 = build(torch.bfloat16, {})
    torch.manual_seed(0)
    m32 = build(torch.float32, {"sparse_grad": True})
    m32.load_state_dict(m16.state_dict())
    return m16, m32


def _table_pairs(m16, m32):
    """[(bf16 table, its proxy, the f32 table)] of every ShallowEncoder in m16"""
    from euler_b200.encoders import ShallowEncoder
    names = {id(p): n for n, p in m16.named_parameters()}
    p32 = dict(m32.named_parameters())
    out, seen = [], set()
    for e in m16.modules():
        if isinstance(e, ShallowEncoder):
            for t, q in e.table_proxies():
                if id(t) not in seen:
                    seen.add(id(t))
                    out.append((t, q, p32[names[id(t)]]))
    return out


@pytest.mark.parametrize("shuffle", (False, True))
def test_repeated_reads_sum_into_the_proxy(env, shuffle):
    """SageEncoder reads its node encoder's tables at every hop and through the pooled deepest hop; ShuffleSageEncoder does
    that twice.  Each proxy's gradient is the f32 table's sparse one, and repeats run to run."""
    import euler_b200
    from euler_b200.encoders import SageEncoder, ShuffleSageEncoder
    cls = ShuffleSageEncoder if shuffle else SageEncoder
    seeds = torch.as_tensor(env["g"]["ids"][:48].astype(np.int64), device="cuda")
    m16, m32 = _pair(lambda dt, kw: cls([[0], [0]], [4, 3], 16, aggregator="mean", **_encoder_kw(dt, **kw)))
    assert m16._pools_deepest_hop()
    grads = []
    for m in (m16, m32, m16):
        for t, q, t32 in _table_pairs(m16, m32):
            q.grad = t32.grad = None
        euler_b200.seed(3)
        out = m(seeds, torch.Generator().manual_seed(1)) if shuffle else m(seeds)
        out = torch.cat(out, 0) if shuffle else out
        G = torch.randn(out.shape, generator=torch.Generator().manual_seed(4)).cuda()
        (out * G).sum().backward()
        grads.append([(q.grad if m is m16 else t32.grad).coalesce() for _, q, t32 in _table_pairs(m16, m32)])
    assert len(grads[0]) == 3
    for k, (a, b, c) in enumerate(zip(*grads)):
        _same_sparse(a, b, (shuffle, k))
        _same_sparse(a, c, (shuffle, k, "repeat"))


# ------------------------------------------------------------------------------------------------ one minimize step
def _sup_sage(aggregator):
    from euler_b200.encoders import SageEncoder
    from euler_b200.supervised import SuperviseModel

    class SupSage(SuperviseModel):
        def __init__(self, dt, kw):
            super().__init__("feat2", 3, dim=16, device="cuda")
            self.enc = SageEncoder([[0], [0]], [4, 3], 16, aggregator=aggregator, **_encoder_kw(dt, **kw))

        def embed(self, n_id):
            return self.enc(n_id)

    return lambda dt, kw: SupSage(dt, kw)


def _geniepath(dt, kw):
    from euler_b200.supervised import GeniePath
    k = _encoder_kw(dt, **kw)
    k.pop("embedding_dim")
    return GeniePath(16, [[0], [0]], "feat2", 3, use_residual=True, head_num=2, **k)


def _dgi(dt, kw):
    from euler_b200.unsupervised import DGI
    k = _encoder_kw(dt, **kw)
    return DGI(0, [0], k.pop("max_id"), [[0], [0]], [4, 3], 16, **k)


def _gae(dt, kw):
    from euler_b200.autoencoder import GraphAutoEncoder
    from euler_b200.encoders import SageEncoder
    return GraphAutoEncoder(SageEncoder([[0], [0]], [3, 2], 16, **_encoder_kw(dt, **kw)), 0, [0], MAX_ID, num_negs=3)


MODELS = {"sage_mean": _sup_sage("mean"), "sage_gcn": _sup_sage("gcn"), "sage_meanpool": _sup_sage("meanpool"),
          "geniepath": _geniepath, "dgi": _dgi, "gae": _gae}
LR = 0.01


def _loss(m, seeds):
    out = m(seeds, torch.Generator().manual_seed(1)) if type(m).__name__ == "DGI" else m(seeds)
    return out[1]


@pytest.mark.parametrize("opt", ("adam", "momentum"))
@pytest.mark.parametrize("model", sorted(MODELS))
def test_minimize_step_equals_f32_step(env, model, opt):
    import euler_b200
    from euler_b200 import optimizers
    seeds = torch.as_tensor(env["g"]["ids"][100:164].astype(np.int64), device="cuda")
    m16, m32 = _pair(MODELS[model])
    o16 = optimizers.get(opt)(list(m16.parameters()), LR, seed=9)
    o32 = optimizers.get(opt)(list(m32.parameters()), LR)
    pairs = _table_pairs(m16, m32)
    assert pairs and all(t.dtype == torch.bfloat16 for t, _, _ in pairs)
    before = [_bits(t) for t, _, _ in pairs]
    losses = []
    for m, o in ((m16, o16), (m32, o32)):
        euler_b200.seed(7)
        loss = _loss(m, seeds)
        optimizers.minimize(o, loss, m)
        losses.append(loss.detach())
    _same(losses[0], losses[1], "loss")
    for (n, a), (_, b) in zip(m16.named_parameters(), m32.named_parameters()):
        if a.dtype == torch.float32:
            _same(a.detach(), b.detach(), (model, opt, n))
    index = {id(p): i for i, p in enumerate(m16.parameters())}
    for (t, q, t32), bits in zip(pairs, before):
        g = q.grad.coalesce()
        _same_sparse(g, t32.grad, (model, opt, "table gradient"))
        rows, vals = g.indices()[0].cpu().numpy(), g.values().cpu().numpy()
        slots = ["m", "v"] if opt == "adam" else ["momentum"]
        want = [bits.copy()] + [np.zeros_like(bits) for _ in slots]
        adam = ref.Adam(LR, 0.9, 0.999, 1e-8) if opt == "adam" else None
        sr.step(opt, want, (rows, vals), 9, 0, index[id(t)], LR, adam=adam, momentum=0.9)
        got = [_bits(t)] + [_bits(o16.state[t][s]) for s in slots]
        for k, (x, y) in enumerate(zip(got, want)):
            np.testing.assert_array_equal(x, y, err_msg=str((model, opt, k)))
    assert int(o16.sr_step) == 1


def test_gcn_infer_reads_bf16_tables(env):
    from euler_b200.encoders import GCNEncoder
    m16, m32 = _pair(lambda dt, kw: GCNEncoder([[0], [0]], 16, aggregator="mean", **_encoder_kw(dt, **kw)))
    ids = torch.as_tensor(np.concatenate([env["g"]["ids"][:200].astype(np.int64), [MAX_ID + 1]]), device="cuda")
    _same(m16.infer(ids), m32.infer(ids), "infer")
    _same(m16.infer(), m32.infer(), "infer, every node")


# ------------------------------------------------------------------------------------------------ training
def test_training_tracks_f32(env):
    """300 Adam steps at lr 0.001 of a supervised SageEncoder with use_id and a sparse slot, from the same tables and draws:
    the mean loss of the last 50 bf16 steps lies within 2 % of f32 training's, and the bf16 tables move.  (At lr 0.01 both
    memorise the 600 nodes' labels and the loss falls to 1e-4, where 2 % says nothing.)"""
    import euler_b200
    from euler_b200 import optimizers
    from euler_b200.encoders import SageEncoder
    from euler_b200.supervised import SuperviseModel

    class SupSage(SuperviseModel):
        def __init__(self, dt, kw):
            super().__init__("feat2", 3, dim=32, device="cuda")
            self.enc = SageEncoder([[0], [0]], [5, 3], 32, aggregator="mean", feature_idx="feat1", feature_dim=12,
                                   max_id=MAX_ID, use_id=True, sparse_feature_idx=["u64_1"], sparse_feature_max_id=[59],
                                   embedding_dim=16, device="cuda", table_dtype=dt, **kw)

        def embed(self, n_id):
            return self.enc(n_id)

    m16, m32 = _pair(lambda dt, kw: SupSage(dt, kw))
    o16 = optimizers.get("adam")(list(m16.parameters()), 0.001, seed=5)
    o32 = optimizers.get("adam")(list(m32.parameters()), 0.001)
    start = [t.float().clone() for t, _, _ in _table_pairs(m16, m32)]
    ids = env["g"]["ids"].astype(np.int64)
    l16, l32 = [], []
    for s in range(300):
        seeds = torch.as_tensor(np.random.RandomState(s).choice(ids, 64), device="cuda")
        for m, o, out in ((m16, o16, l16), (m32, o32, l32)):
            euler_b200.seed(1000 + s)
            loss = _loss(m, seeds)
            optimizers.minimize(o, loss, m)
            out.append(loss.detach())
    a = np.array([float(x) for x in l16])
    b = np.array([float(x) for x in l32])
    assert b[:10].mean() - b[-50:].mean() > 0.02, (b[:10].mean(), b[-50:].mean())
    assert abs(a[-50:].mean() - b[-50:].mean()) <= 0.02 * b[-50:].mean(), (a[-50:].mean(), b[-50:].mean())
    moved = np.mean([float((t.float() != s).float().mean()) for (t, _, _), s in zip(_table_pairs(m16, m32), start)])
    assert moved > 0.2, moved


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_write_nothing(env):
    import euler_b200
    from euler_b200 import EulerError, _lib, ops
    lib = _lib.load()
    nodes = env["nodes"]
    id16, sp = _bf16(N_ID, 8, 1), _sparse(2, 8, 0)
    euler_b200.shallow_encode(nodes, id16, [], sp, "concat")
    torch.cuda.synchronize()
    n0 = lib.eu_launch_count()
    with pytest.raises(EulerError, match="one dtype"):
        euler_b200.shallow_encode(nodes, id16.float(), [], sp, "concat")
    with pytest.raises(EulerError, match="autograd"):
        euler_b200.shallow_encode(nodes, id16.clone().requires_grad_(), [], sp, "concat")
    with pytest.raises(EulerError, match="autograd"):
        euler_b200.sparse_feature_embedding(nodes, "u64_0", sp[0][1].clone().requires_grad_(), N_ROWS - 1)
    with pytest.raises(EulerError, match="one dtype"):
        euler_b200.shallow_encode_pool(nodes[:700], 7, id16, [], _widened(sp), "mean")
    assert lib.eu_launch_count() == n0
    # an unknown table dtype at the C ABI: EU_ERR_INVALID, the output untouched
    p = er.shallow_problem(nodes, id16, [], sp)
    out = torch.full((nodes.numel(), 24), 7.0, device="cuda")
    for sym, args in (("eu_shallow_encode_dtype", (C.byref(p), 2, out, None)),
                      ("eu_shallow_encode_pool_dtype", (C.byref(p), 2, 1, 0, out)),
                      ("eu_sparse_embedding_lookup_dtype", (nodes, nodes.numel(), 0, 3, sp[0][1], N_ROWS, 8, 0, 2, out))):
        with pytest.raises(EulerError, match="dtype"):
            ops._call(sym, *args)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    assert lib.eu_launch_count() == n0


def test_out_of_range_id_leaves_tables_slots_and_step(env):
    import euler_b200
    from euler_b200 import EulerError, optimizers
    m16, _ = _pair(_sup_sage("mean"))
    opt = optimizers.get("adam")(list(m16.parameters()), LR, seed=9)
    seeds = torch.as_tensor(env["g"]["ids"][:32].astype(np.int64), device="cuda")
    euler_b200.seed(1)
    optimizers.minimize(opt, _loss(m16, seeds), m16)   # the slots exist from here
    torch.cuda.synchronize()
    tables = [t for t, _, _ in _table_pairs(m16, m16)]

    def state():
        return [_bits(t) for t in tables] + [_bits(opt.state[t][s]) for t in tables for s in ("m", "v")] + \
            [p.detach().cpu().numpy().copy() for p in m16.parameters() if p.dtype == torch.float32]

    before, step, powers = state(), int(opt.sr_step), opt.beta_powers.clone()
    bad = seeds.clone()
    bad[5] = MAX_ID + 50
    with pytest.raises(EulerError, match="outside"):
        optimizers.minimize(opt, _loss(m16, bad), m16)
    torch.cuda.synchronize()
    for a, b in zip(state(), before):
        np.testing.assert_array_equal(a, b)
    assert int(opt.sr_step) == step and torch.equal(opt.beta_powers, powers)
