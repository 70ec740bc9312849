"""GPU: the fused optimizer updates (ops.optim_momentum_, optim_adagrad_, optim_adam_: eu_optim_*) bit for bit against the
numpy float32 restatement of TF 1.x (tests/optim_reference.py) over consecutive steps, dense and sparse, at every row width,
aligned and offset; the sparse table gradients the library's backward passes produce; repeat bits, no host synchronisation,
CUDA-graph replay, a table above 2^31 elements, host refusals, and whole training steps against fused=False."""
import copy

import numpy as np
import pytest
import torch

import embedding_reference as er
import graphs  # noqa: F401  (sys.path)
import optim_reference as ref

pytestmark = pytest.mark.gpu
F32 = np.float32
NAMES = ['sgd', 'momentum', 'adagrad', 'adam']
LR = {'sgd': 0.1, 'momentum': 0.05, 'adagrad': 0.3, 'adam': 0.01}


@pytest.fixture(scope="module")
def eb():
    import euler_b200
    g = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    return euler_b200


def _bits(x):
    return np.ascontiguousarray(np.asarray(x, F32)).view(np.int32)


def _assert_bits(got, want, what):
    np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=what)


def _values(rng, shape):
    """gradient values with zeros, subnormals and large entries among ordinary ones"""
    g = rng.randn(*shape).astype(F32)
    flat = g.reshape(-1)
    k = flat.size
    flat[rng.rand(k) < 0.1] = 0
    flat[rng.rand(k) < 0.05] = F32(3e-39) * rng.choice([-1, 1])
    flat[rng.rand(k) < 0.05] = F32(1e18) * rng.choice([-1, 1])
    return g


def _dev(x, offset):
    """x on the device, contiguous; offset puts its data one float past a 16-byte boundary"""
    x = np.ascontiguousarray(x, F32)
    if not offset:
        return torch.from_numpy(x).cuda()
    buf = torch.empty(x.size + 1, dtype=torch.float32, device="cuda")
    t = buf[1:].view(x.shape)
    t.copy_(torch.from_numpy(x))
    return t


def _sparse(rows, vals, shape, offset):
    return torch.sparse_coo_tensor(torch.from_numpy(rows).cuda()[None], _dev(vals, offset), shape, is_coalesced=True,
                                   check_invariants=False)


def _sparse_steps(rng, N):
    """the rows of five steps: a few with 0 and N - 1, none, one (N - 1), every row, a few"""
    few = lambda: np.unique(np.concatenate([[0, N - 1], rng.choice(N, size=min(N, 5), replace=False)]))  # noqa: E731
    return [few(), np.zeros(0, np.int64), np.array([N - 1]), np.arange(N), few()]


def _step_op(name, var, slots, grad, powers=None):
    from euler_b200 import ops
    if name == 'adam':
        ops.optim_adam_(var, slots[0], slots[1], grad, powers, LR[name], 0.9, 0.999, 1e-8)
        powers.mul_(torch.tensor([0.9, 0.999], dtype=torch.float32, device="cuda"))
    elif name == 'adagrad':
        ops.optim_adagrad_(var, slots[0], grad, LR[name])
    else:
        ops.optim_momentum_(var, slots[0], grad, LR[name], 0.0 if name == 'sgd' else 0.9)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("form", ["dense", "sparse"])
@pytest.mark.parametrize("D", [1, 3, 4, 16, 128, 200])
@pytest.mark.parametrize("offset", [False, True])
def test_bit_exact_vs_restatement(eb, name, form, D, offset):
    N = 9000 if D <= 4 else 300   # several sparse-Adam CTAs at every width
    rng = np.random.RandomState(D * 31 + len(name) + (7 if offset else 0))
    shape = (N, D) if D > 1 else (N,)
    var0 = (rng.randn(*shape) * 2).astype(F32)
    want_var = var0.copy()
    nslots = 2 if name == 'adam' else 1
    init = F32(0.1) if name == 'adagrad' else F32(0)
    want_slots = [np.full(shape, init, F32) for _ in range(nslots)]
    var = _dev(var0, offset)
    slots = [_dev(s, offset) for s in want_slots]
    powers = torch.tensor([0.9, 0.999], dtype=torch.float32, device="cuda")
    adam = ref.Adam(LR['adam'])
    steps = _sparse_steps(rng, N) if form == "sparse" else [None] * 5
    for k, rows in enumerate(steps):
        if form == "dense":
            g = _values(rng, shape)
            grad, rg = _dev(g, offset), g
        else:
            vals = _values(rng, (rows.size,) + shape[1:])
            grad, rg = _sparse(rows, vals, shape, offset), (rows, vals)
        before = [var.cpu().numpy()] + [s.cpu().numpy() for s in slots]
        _step_op(name, var, slots, grad, powers)
        if name == 'adam':
            adam.step([(want_var, want_slots[0], want_slots[1], rg)])
        elif name == 'adagrad':
            ref.adagrad(want_var, want_slots[0], rg, LR[name])
        else:
            ref.momentum(want_var, want_slots[0], rg, LR[name], 0.0 if name == 'sgd' else 0.9)
        what = "%s %s D=%d offset=%s step %d" % (name, form, D, offset, k)
        _assert_bits(var.cpu().numpy(), want_var, what + " var")
        for s, w in zip(slots, want_slots):
            _assert_bits(s.cpu().numpy(), w, what + " slot")
        if name == 'adam':
            _assert_bits(powers.cpu().numpy(), adam.powers, what + " powers")
        elif form == "sparse":   # Momentum and Adagrad leave untouched rows alone, bit for bit
            untouched = np.setdiff1d(np.arange(N), rows)
            for got, was in zip([var] + slots, before):
                _assert_bits(got.cpu().numpy()[untouched], was[untouched], what + " untouched rows")


def _coo_ok(g, what):
    """a COO gradient of whole rows whose rows are strictly increasing.  (Its is_coalesced() flag may be lost on the way to
    .grad: torch's gradient accumulation can rebuild the tensor without it; the optimizers then coalesce() it.)"""
    assert g is not None and g.is_sparse and g.sparse_dim() == 1, what
    rows = g._indices()[0].cpu().numpy()
    bad = np.nonzero(np.diff(rows) <= 0)[0]
    assert bad.size == 0, "%s: rows not strictly increasing at %s: %s" % (what, bad[:8], rows[bad[:4, None] + [0, 1]])


@pytest.mark.parametrize("producer", ["skipgram", "shallow_encode", "shallow_encode_pool", "kg", "sparse_feature_embedding"])
def test_library_sparse_gradients_arrive_sorted_and_unique(eb, producer):
    import euler_b200
    from euler_b200 import encoders, knowledge, unsupervised as un
    euler_b200.set_graph(eb.get_graph(), rng="minstd", seed=1)
    torch.manual_seed(0)
    inputs = torch.as_tensor(np.random.RandomState(1).randint(1, 500, size=300), device="cuda")
    if producer == "skipgram":   # DeepWalk
        dw = un.DeepWalk(0, [0], 500, 16, walk_len=3, num_negs=5, sparse_grad=True, device="cuda")
        dw(inputs)[1].backward()
        grads = [p.grad for p in dw.parameters()]
    elif producer == "shallow_encode":   # ShallowEncoder over an id table
        se = encoders.ShallowEncoder(dim=8, feature_idx=-1, max_id=500, sparse_grad=True, device="cuda")
        se(inputs).sum().backward()
        grads = [se.embedding.embeddings.grad]
    elif producer == "shallow_encode_pool":   # SageEncoder's deepest hop; SageEncoder itself adds one such gradient per hop
        table = torch.randn(502, 8, device="cuda", requires_grad=True)
        out = euler_b200.shallow_encode_pool(inputs, 3, id_table=table, pool='mean', sparse_grad=True)
        grads = [torch.autograd.grad(out.sum(), table)[0]]
    elif producer == "kg":   # TransE
        euler_b200.set_graph(_kg_graph(), rng="minstd", seed=3)
        te = knowledge.TransE(0, 0, 199, 5, 16, 16, num_negs=4, sparse_grad=True, device="cuda")
        te(euler_b200.sample_edge(64, 0)).loss.backward()
        grads = [p.grad for p in te.parameters()]
    else:   # over a uint64 slot
        sg = er.slot_graph(5, 400, [lambda rng, n: rng.randint(0, 4, size=n)], [lambda rng, k: rng.randint(0, 99, size=k)])
        euler_b200.set_graph(euler_b200.Graph.from_csr(sg["ids"], sg["grp_ptr"], sg["nbr"], n_edge_types=sg["T"],
                                                       node_type=sg["node_type"], node_w=sg["node_w"], cum_w=sg["cum_w"],
                                                       u64_ptr=sg["u64_ptr"], u64_val=sg["u64_val"], n_u64_slots=sg["S"]),
                             rng="minstd", seed=1)
        table = torch.randn(100, 8, device="cuda", requires_grad=True)
        nodes = torch.as_tensor(sg["ids"][np.random.RandomState(4).randint(0, 400, size=500)], device="cuda")
        euler_b200.sparse_feature_embedding(nodes, "u64_0", table, 99, sparse_grad=True).sum().backward()
        grads = [table.grad]
    for k, g in enumerate(grads):
        _coo_ok(g, "%s gradient %d" % (producer, k))


def _kg_graph(n_ent=200, n_rel=6, n_edges=3000, seed=0):
    """a knowledge graph: entities of node type 0, triples of edge type 0 with the relation id in the edge slot 'id'"""
    import euler_b200
    rng = np.random.RandomState(seed)
    src, dst, rel = rng.randint(0, n_ent, n_edges), rng.randint(0, n_ent, n_edges), rng.randint(0, n_rel, n_edges)
    order = np.lexsort((dst, src))
    src, dst, rel = src[order], dst[order], rel[order]
    ptr = np.cumsum(np.concatenate([[0], np.bincount(src, minlength=n_ent)])).astype(np.int64)
    g = euler_b200.Graph.from_csr(np.arange(n_ent), ptr, dst, w=np.ones(n_edges, np.float32))
    g.set_edges(src, dst, np.zeros(n_edges, np.int32), dense=rel.reshape(-1, 1).astype(np.float32), dense_names=['id'])
    return g


@pytest.fixture
def graph500():
    import euler_b200
    g = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    return euler_b200


@pytest.mark.parametrize("name", NAMES)
def test_uncoalesced_gradient_matches_coalesce_then_restatement(graph500, name):
    """a table two ops used in one step: the sum of their COO gradients is uncoalesced"""
    from euler_b200 import optimizers
    rng = np.random.RandomState(8)
    N, D = 700, 12
    var0 = rng.randn(N, D).astype(F32)
    p = torch.nn.Parameter(torch.from_numpy(var0.copy()).cuda())
    opt = optimizers.get(name)([p], LR[name])
    want = var0.copy()
    grads = []
    for s in range(3):
        parts = []
        for _ in range(2):
            rows = np.sort(rng.choice(N, size=40, replace=False))
            parts.append(_sparse(rows, _values(rng, (40, D)), (N, D), False))
        g = parts[0] + parts[1]
        assert not g.is_coalesced()
        c = g.coalesce()
        grads.append((c._indices()[0].cpu().numpy(), c._values().cpu().numpy()))
        p.grad = g
        opt.step()
    want, _, powers = ref.run(name, want, grads, LR[name])
    _assert_bits(p.detach().cpu().numpy(), want, name)
    if name == 'adam':
        _assert_bits(opt.beta_powers.cpu().numpy(), powers, "powers")


def _table_step(name, N=200000, D=64, R=3000, seed=0, steps=2):
    """a table, fused, after `steps` sparse steps then one dense step: the var and slot bits"""
    from euler_b200 import optimizers
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.nn.Parameter(torch.randn(N, D, generator=g, device="cuda"))
    opt = optimizers.get(name)([p], LR[name])
    for s in range(steps):
        rows = torch.randperm(N, generator=g, device="cuda")[:R].sort().values
        p.grad = torch.sparse_coo_tensor(rows[None], torch.randn(R, D, generator=g, device="cuda"), (N, D), is_coalesced=True)
        opt.step()
    p.grad = torch.randn(N, D, generator=g, device="cuda")
    opt.step()
    return [p.detach().clone()] + [t.clone() for t in opt.state[p].values()]


@pytest.mark.parametrize("name", NAMES)
def test_two_runs_give_identical_bits(graph500, name):
    a, b = _table_step(name), _table_step(name)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def _mixed_params(rng):
    """a dense weight, a bias and a sparse table, with their gradients"""
    w = torch.nn.Parameter(torch.from_numpy(rng.randn(33, 17).astype(F32)).cuda())
    b = torch.nn.Parameter(torch.from_numpy(rng.randn(17).astype(F32)).cuda())
    t = torch.nn.Parameter(torch.from_numpy(rng.randn(5000, 32).astype(F32)).cuda())
    rows = np.sort(rng.choice(5000, size=300, replace=False))
    grads = [torch.from_numpy(_values(rng, (33, 17))).cuda(), torch.from_numpy(_values(rng, (17,))).cuda(),
             _sparse(rows, _values(rng, (300, 32)), (5000, 32), False)]
    return [w, b, t], grads


@pytest.mark.parametrize("name", NAMES)
def test_step_never_synchronises(graph500, name):
    from euler_b200 import optimizers
    params, grads = _mixed_params(np.random.RandomState(4))
    opt = optimizers.get(name)(params, LR[name])
    for p, g in zip(params, grads):
        p.grad = g
    opt.step()   # the first step allocates the slots and the Context
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.step()
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", NAMES)
def test_graph_replay_gives_eager_bits(graph500, name):
    from euler_b200 import optimizers
    rng = np.random.RandomState(6)
    params, grads = _mixed_params(rng)
    eager = [torch.nn.Parameter(p.detach().clone()) for p in params]
    o_eager = optimizers.get(name)(eager, LR[name])
    o_graph = optimizers.get(name)(params, LR[name])
    for ps in (params, eager):
        for p, g in zip(ps, grads):
            p.grad = g
    o_eager.step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o_graph.step()   # warm-up on the capture stream: slots, the Context bound to it
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            o_graph.step()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(4):
        cg.replay()
        o_eager.step()
    torch.cuda.synchronize()
    for p, q in zip(params, eager):
        assert torch.equal(p.detach().view(torch.int32), q.detach().view(torch.int32))
        for a, b in zip(o_graph.state[p].values(), o_eager.state[q].values()):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    if name == 'adam':   # five steps each: the warm-up and four replays
        want = ref.Adam()
        for _ in range(5):
            want.finish()
        _assert_bits(o_graph.beta_powers.cpu().numpy(), want.powers, "replayed powers")
        _assert_bits(o_eager.beta_powers.cpu().numpy(), want.powers, "eager powers")


def test_sparse_adam_above_2_31_elements(graph500):
    """one sparse Adam step on a table of 2^31 + 1000 single-float rows: touched rows, sampled untouched rows, the last row"""
    from euler_b200 import ops
    N = (1 << 31) + 1000
    var = torch.empty(N, device="cuda").uniform_(-1, 1)
    m = torch.full((N,), 0.25, device="cuda")
    v = torch.full((N,), 0.5, device="cuda")
    rng = np.random.RandomState(3)
    rows = np.unique(np.concatenate([rng.randint(0, N, size=2000), [0, (1 << 31) - 1, 1 << 31, N - 2]])).astype(np.int64)
    vals = _values(rng, (rows.size,))
    untouched = np.setdiff1d(np.concatenate([rng.randint(0, N, size=2000), [N - 1, (1 << 31) + 1]]), rows)
    pick = np.concatenate([rows, untouched])
    pick_t = torch.from_numpy(pick).cuda()
    w0, m0, v0 = (t[pick_t].cpu().numpy() for t in (var, m, v))
    powers = torch.tensor([0.9, 0.999], dtype=torch.float32, device="cuda")
    ops.optim_adam_(var, m, v, _sparse(rows, vals, (N,), False), powers, 0.01, 0.9, 0.999, 1e-8)
    adam = ref.Adam(0.01)
    adam.update(w0, m0, v0, (np.arange(rows.size), vals))   # rows are independent: the update of the picked rows alone
    got = [t[pick_t].cpu().numpy() for t in (var, m, v)]
    for g, w, nm in zip(got, (w0, m0, v0), ('var', 'm', 'v')):
        _assert_bits(g, w, nm)
    del var, m, v
    torch.cuda.empty_cache()


def test_host_refusals_write_nothing(graph500):
    import euler_b200
    from euler_b200 import ops
    N, D = 50, 8
    var, a, b = (torch.randn(N, D, device="cuda") for _ in range(3))
    powers = torch.tensor([0.9, 0.999], device="cuda")
    keep = [t.clone() for t in (var, a, b, powers)]
    good = torch.randn(N, D, device="cuda")
    cases = [
        lambda: ops.optim_momentum_(var, a[:, :4], good, 0.1, 0.9),                          # slot shape
        lambda: ops.optim_momentum_(var, a, good.double(), 0.1, 0.9),                        # grad dtype
        lambda: ops.optim_momentum_(var, a, good.cpu(), 0.1, 0.9),                           # grad device
        lambda: ops.optim_adagrad_(var, a.t().contiguous().t(), good, 0.1),                                   # non-contiguous slot
        lambda: ops.optim_adagrad_(var, a.half(), good, 0.1),                                # slot dtype
        lambda: ops.optim_adagrad_(var, a, good[:10], 0.1),                                  # grad shape
        lambda: ops.optim_adam_(var, a, b, good, powers[:1], 0.1, 0.9, 0.999, 1e-8),         # powers shape
        lambda: ops.optim_adam_(var, a, b, good, powers.double(), 0.1, 0.9, 0.999, 1e-8),    # powers dtype
        lambda: ops.optim_adam_(var, a, b.cpu(), good, powers, 0.1, 0.9, 0.999, 1e-8),       # slot device
        lambda: ops.optim_adam_(var, a, b, good.to_sparse(2), powers, 0.1, 0.9, 0.999, 1e-8),  # two sparse dims
    ]
    for k, call in enumerate(cases):
        with pytest.raises(euler_b200.EulerError):
            call()
        for t, w in zip((var, a, b, powers), keep):
            assert torch.equal(t, w), k


def _close(a, b, what):
    scale = max(float(b.abs().max()), 1e-30)
    assert float((a - b).abs().max()) <= 1e-5 * scale, what


def _compare_steps(make_model, run_step, name, lr, steps=3):
    """the model trained `steps` steps with the fused optimizer and with fused=False, from the same parameters and draws"""
    from euler_b200 import optimizers
    import euler_b200
    m1 = make_model()
    m2 = copy.deepcopy(m1)
    for m, fused in ((m1, True), (m2, False)):
        opt = optimizers.get(name)(m.parameters(), lr, fused=fused)
        for s in range(steps):
            euler_b200.seed(100 + s)
            opt.zero_grad()
            run_step(m, s).backward()
            opt.step()
    for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        _close(p.detach(), q.detach(), n)


def test_deepwalk_sparse_adam_steps(graph500):
    from euler_b200 import unsupervised as un
    torch.manual_seed(1)
    inputs = torch.as_tensor(np.random.RandomState(2).randint(1, 500, size=256), device="cuda")
    _compare_steps(lambda: un.DeepWalk(0, [0], 500, 32, walk_len=3, num_negs=5, sparse_grad=True, device="cuda"),
                   lambda m, s: m(inputs)[1], 'adam', 0.01)


def test_transe_adagrad_steps():
    import euler_b200
    from euler_b200 import knowledge
    euler_b200.set_graph(_kg_graph(), rng="minstd", seed=3)
    torch.manual_seed(0)
    edges = euler_b200.sample_edge(128, 0)
    _compare_steps(lambda: knowledge.TransE(0, 0, 199, 5, 16, 16, num_negs=4, device="cuda"),
                   lambda m, s: m(edges).loss, 'adagrad', 0.1)


def test_supervised_sage_momentum_steps():
    import euler_b200
    from euler_b200 import encoders
    from euler_b200.supervised import SuperviseModel
    max_id, feat = 3000, 16
    g = graphs.random_graph(seed=49, n=max_id, T=1, avg_deg=5, feat_dim=feat)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)

    class Model(SuperviseModel):
        def __init__(self):
            super().__init__(0, 3, dim=8, device="cuda")
            self.enc = encoders.SageEncoder([[0], [0]], [5, 2], 8, 'mean', feature_idx=0, feature_dim=feat, max_id=max_id,
                                            use_id=True, sparse_grad=True, device="cuda")

        def embed(self, n_id):
            return self.enc(n_id)

    torch.manual_seed(2)
    inputs = torch.as_tensor(np.random.RandomState(5).randint(1, max_id + 1, size=512), device="cuda")
    probe = Model()
    probe(inputs)[1].backward()
    kinds = {p.grad.is_sparse for p in probe.parameters() if p.grad is not None}
    assert kinds == {True, False}   # dense layers and a sparse id table in one step
    _compare_steps(Model, lambda m, s: m(inputs)[1], 'momentum', 0.1)
