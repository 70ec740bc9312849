"""GPU: the skip-gram step and tf_euler's optimizers over bfloat16 id tables.  The forward and backward of bf16 tables give
the f32 op's bits on the widened tables; every optimizer update, dense and sparse, is bit for bit sr_reference's restatement
(f32 update on widened values, then stochastic rounding); repeated runs and CUDA-graph replays repeat the bits; DeepWalk
and LINE trained on bf16 tables track f32 training, where round to nearest would stall; refusals write nothing."""
import numpy as np
import pytest
import torch

import bf16_reference as bf
import graphs  # noqa: F401  (sys.path)
import optim_reference as ref
import skipgram_reference as sk
import sr_reference as sr

pytestmark = pytest.mark.gpu
F32 = np.float32
LR = {'momentum': 0.05, 'adagrad': 0.3, 'adam': 0.01}
SLOTS = {'momentum': ('momentum',), 'adagrad': ('accumulator',), 'adam': ('m', 'v')}
SEED = 0xDEADBEEF12345678


@pytest.fixture(scope="module")
def graph():
    import euler_b200
    g = euler_b200.Graph.rmat(4096, 40000, seed=11)
    euler_b200.set_graph(g, rng="minstd", seed=1)
    return euler_b200


def _bf16(bits, offset=0):
    """uint16 bf16 bits [N, D] on the device; offset puts the data `offset` elements past an 8-byte boundary"""
    bits = np.ascontiguousarray(bits, np.uint16)
    buf = torch.zeros(bits.size + offset, dtype=torch.int16, device="cuda")
    buf[offset:] = torch.from_numpy(bits.reshape(-1).view(np.int16)).cuda()
    return buf.view(torch.bfloat16)[offset:].view(bits.shape)


def _bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _table(rng, n, dim, offset, scale=0.1):
    """(a bf16 table, the same table widened to f32, contiguous)"""
    t = _bf16(bf.round_bits(rng.randn(n, dim).astype(F32) * F32(scale)), offset)
    return t, t.float()


def _ids(src, pos, negs):
    d = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.int64).cuda().contiguous()   # noqa: E731
    return d(src).reshape(-1), d(pos), d(negs).reshape(len(src), np.asarray(negs).shape[1])


def _same(a, b, what):
    assert a.dtype == b.dtype and torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                              b.view(torch.int32) if b.dtype == torch.float32 else b), what


# ------------------------------------------------------------------------------------------------ forward and backward
@pytest.mark.parametrize("dim", [1, 3, 4, 16, 128, 200, 512, 513])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("P,K", [(1, 0), (1, 5), (3, 0), (3, 5)])
def test_forward_is_the_f32_op_on_widened_tables(graph, dim, offset, P, K):
    from euler_b200 import ops
    rng = np.random.RandomState(dim * 7 + offset + 31 * P + K)
    n, B = 300, 37
    t16, t32 = _table(rng, n, dim, offset)
    c16, c32 = _table(rng, n, dim, offset)
    src, pos, negs = sk.pair_ids(rng, B, P, K, n)
    ids = _ids(src, pos, negs)
    lg16, rk16, ls16 = ops._raw_skipgram(*ids, t16, c16)
    lg32, rk32, ls32 = ops._raw_skipgram(*ids, t32, c32)
    _same(lg16, lg32, "logits")
    assert torch.equal(rk16, rk32)
    _same(ls16, ls32, "loss")
    _, l64 = sk.forward64(t32.cpu().numpy(), c32.cpu().numpy(), src, sk.context_ids(pos, negs), P)
    assert abs(float(ls16) - l64) <= 1e-6
    loss, metric = ops.skipgram_xent_loss(*ids, t16, c16, metric='mrr')   # the public op on bf16 tables
    loss32, metric32 = ops.skipgram_xent_loss(*ids, t32, c32, metric='mrr')
    _same(loss, loss32, "public loss")
    _same(metric, metric32, "public metric")


@pytest.mark.parametrize("dim", [3, 16, 128, 200])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("n", [300, 5])   # 5 rows: every row's entries span several 256-entry chunks
def test_backward_is_the_f32_op_on_widened_tables(graph, dim, offset, shared, n):
    from euler_b200 import ops
    rng = np.random.RandomState(dim + 3 * offset + 5 * shared + n)
    B, P, K = 400, 1, 5
    t16, t32 = _table(rng, n, dim, offset)
    c16, c32 = (t16, t32) if shared else _table(rng, n, dim, offset)
    src, pos, negs = sk.pair_ids(rng, B, P, K, n)
    ids = _ids(src, pos, negs)
    logits = ops._raw_skipgram(*ids, t16, c16)[0]
    g = torch.tensor([0.75], dtype=torch.float32, device="cuda")
    sp16 = ops._raw_skipgram_sparse_grads(*ids, t16, c16, logits, g, shared)
    sp32 = ops._raw_skipgram_sparse_grads(*ids, t32, c32, logits, g, shared)
    assert len(sp16) == len(sp32) == (1 if shared else 2)
    for (r16, v16), (r32, v32) in zip(sp16, sp32):
        assert torch.equal(r16, r32)
        _same(v16, v32, "sparse values")
    dense = {}
    for name, (t, c, sym, extra) in {"bf16": (t16, c16, "eu_skipgram_loss_backward_dtype", (1,)),
                                     "f32": (t32, c32, "eu_skipgram_loss_backward", ())}.items():
        gt = torch.full((n, dim), 7.0, device="cuda")
        gc = gt if shared else torch.full((n, dim), 7.0, device="cuda")
        ops._call(sym, g, *ids, B, P, K, t, c, n, dim, *extra, logits, gt, gc)
        dense[name] = (gt, gc)
    for a, b in zip(dense["bf16"], dense["f32"]):
        _same(a, b, "dense gradient")


# ------------------------------------------------------------------------------------------------ optimizer updates
def _grad_values(rng, shape):
    g = rng.randn(*shape).astype(F32)
    g.reshape(-1)[rng.rand(g.size) < 0.1] = 0
    return g


def _f32_dev(x, offset):
    x = np.ascontiguousarray(x, F32)
    buf = torch.zeros(x.size + offset, dtype=torch.float32, device="cuda")
    buf[offset:] = torch.from_numpy(x.reshape(-1)).cuda()
    return buf[offset:].view(x.shape)


def _init_slots(name, rng, N, D):
    """random slot bits of a dense test: adagrad's accumulator and adam's v positive"""
    if name == 'momentum':
        return [bf.round_bits(rng.randn(N, D).astype(F32) * F32(0.1))]
    if name == 'adagrad':
        return [bf.round_bits(np.abs(rng.randn(N, D)).astype(F32) + F32(0.1))]
    return [bf.round_bits(rng.randn(N, D).astype(F32) * F32(0.1)), bf.round_bits(np.abs(rng.randn(N, D)).astype(F32) * F32(0.01))]


def _steps_rows(rng, N):
    few = lambda: np.unique(np.concatenate([[0, N - 1], rng.choice(N, size=min(N, 5), replace=False)]))  # noqa: E731
    return [few(), np.zeros(0, np.int64), np.array([N - 1]), np.arange(N), few()]


@pytest.mark.parametrize("name", ['momentum', 'adagrad', 'adam'])
@pytest.mark.parametrize("form", ["dense", "sparse"])
@pytest.mark.parametrize("D", [1, 3, 4, 16, 128])
@pytest.mark.parametrize("offset", [0, 1])
def test_updates_match_the_restatement(graph, name, form, D, offset):
    """five steps; var and slots bit-equal to sr_reference.step after each.  Sparse: through the optimizer's apply_sparse,
    the table the second of two parameters (tensor index 1), the first never updated; dense: through ops.optim_*_"""
    from euler_b200 import ops, optimizers
    rng = np.random.RandomState(D * 11 + offset + len(name) + (form == "dense"))
    N = 64
    var_bits = bf.round_bits(rng.randn(N, D).astype(F32) * F32(0.5))
    adam_ref = ref.Adam(LR['adam'], 0.9, 0.999, 1e-8) if name == 'adam' else None
    if form == "sparse":
        other = torch.nn.Parameter(_bf16(bf.round_bits(rng.randn(7, D).astype(F32))), requires_grad=False)
        other_bits = _bits(other)
        var = torch.nn.Parameter(_bf16(var_bits, offset), requires_grad=False)
        opt = optimizers.get(name)([other, var], LR[name], seed=SEED)
        if name == 'adagrad':
            slot_bits = [bf.round_bits(np.full((N, D), F32(0.1)))]
        else:
            slot_bits = [np.zeros((N, D), np.uint16) for _ in SLOTS[name]]
        row_sets = _steps_rows(rng, N)
    else:
        var = _bf16(var_bits, offset)
        slot_bits = _init_slots(name, rng, N, D)
        slots = [_bf16(b, offset) for b in slot_bits]
        step = torch.zeros((), dtype=torch.int64, device="cuda")
        powers = torch.tensor([0.9, 0.999], dtype=torch.float32, device="cuda")
    tables = [var_bits.copy()] + [b.copy() for b in slot_bits]
    for k in range(5):
        if form == "sparse":
            rows = row_sets[k]
            vals = _grad_values(rng, (len(rows), D))
            grad = (rows, vals)
            opt.apply_sparse(var, torch.from_numpy(rows).cuda(), _f32_dev(vals, offset))
            dev_slots = [opt.state[var][s] for s in SLOTS[name]]
        else:
            grad = _grad_values(rng, (N, D))
            g = _f32_dev(grad, offset)
            kw = dict(seed=SEED, step=step, tensor=1)
            if name == 'adam':
                ops.optim_adam_(var, slots[0], slots[1], g, powers, LR[name], 0.9, 0.999, 1e-8, **kw)
                powers.mul_(torch.tensor([0.9, 0.999], dtype=torch.float32, device="cuda"))
            elif name == 'adagrad':
                ops.optim_adagrad_(var, slots[0], g, LR[name], **kw)
            else:
                ops.optim_momentum_(var, slots[0], g, LR[name], 0.9, **kw)
            step.add_(1)
            dev_slots = slots
        sr.step(name, tables, grad, SEED, k, 1, LR[name], adam=adam_ref, momentum=0.9)
        if adam_ref is not None:
            adam_ref.finish()
        np.testing.assert_array_equal(_bits(var), tables[0], err_msg="var, step %d" % k)
        for i, s in enumerate(dev_slots):
            np.testing.assert_array_equal(_bits(s), tables[1 + i], err_msg="slot %d, step %d" % (i, k))
    if form == "sparse":
        np.testing.assert_array_equal(_bits(other), other_bits, err_msg="a parameter never updated")
        assert int(opt.sr_step) == 5


@pytest.mark.parametrize("name", ['momentum', 'adagrad', 'adam'])
@pytest.mark.parametrize("D", [4, 3])
def test_rows_outside_the_table_are_never_written(graph, name, D):
    """guard rows before and after var (and its slots) keep their bits when the gradient names rows -1 and N"""
    from euler_b200 import ops
    rng = np.random.RandomState(40 + D)
    N = 50
    bufs = [_bf16(bf.round_bits(np.abs(rng.randn(N + 2, D)).astype(F32) + F32(0.1))) for _ in SLOTS[name] + ('var',)]
    before = [_bits(b) for b in bufs]
    views = [b[1:N + 1] for b in bufs]
    rows = torch.tensor([-1, 3, 17, N], dtype=torch.int64, device="cuda")
    vals = torch.ones((4, D), dtype=torch.float32, device="cuda")
    step = torch.zeros((), dtype=torch.int64, device="cuda")
    powers = torch.tensor([0.9, 0.999], dtype=torch.float32, device="cuda")
    var = views[-1]
    if name == 'adam':
        ops._call("eu_optim_adam_dtype", var, views[0], views[1], N, D, vals, rows, 4, powers, 0.01, 0.9, 0.999, 1e-8, 1, 1,
                  step, 0)
    elif name == 'adagrad':
        ops._call("eu_optim_adagrad_dtype", var, views[0], N, D, vals, rows, 4, 0.3, 1, 1, step, 0)
    else:
        ops._call("eu_optim_momentum_dtype", var, views[0], N, D, vals, rows, 4, 0.05, 0.9, 1, 1, step, 0)
    for b, w in zip(bufs, before):
        got = _bits(b)
        np.testing.assert_array_equal(got[[0, N + 1]], w[[0, N + 1]], err_msg="guard rows")
        if name != 'adam':   # sparse momentum / adagrad: only rows 3 and 17 change
            untouched = np.setdiff1d(np.arange(1, N + 1), [4, 18])
            np.testing.assert_array_equal(got[untouched], w[untouched], err_msg="untouched rows")


def _table_run(name, graph_replay):
    """an optimizer over two bf16 tables stepped five times through apply_sparse from fixed gradients: eager, or one
    warm-up step and four replays of a captured step.  Returns (bits of every table and slot, the step counter)."""
    from euler_b200 import optimizers
    rng = np.random.RandomState(9)
    params = [torch.nn.Parameter(_bf16(bf.round_bits(rng.randn(n, 16).astype(F32) * F32(0.2))), requires_grad=False)
              for n in (3000, 700)]
    rows = [torch.from_numpy(np.unique(rng.randint(0, p.shape[0], size=400))).cuda() for p in params]
    vals = [torch.from_numpy(rng.randn(len(r), 16).astype(F32) * F32(1e-3)).cuda() for r in rows]
    opt = optimizers.get(name)(params, LR[name], seed=77)
    if not graph_replay:
        for _ in range(5):
            opt.apply_sparse(params, rows, vals)
    else:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            opt.apply_sparse(params, rows, vals)   # warm-up on the capture stream: slots, the Context bound to it
            cg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(cg, stream=s):
                opt.apply_sparse(params, rows, vals)
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(4):
            cg.replay()
    torch.cuda.synchronize()
    out = [_bits(p) for p in params] + [_bits(t) for p in params for t in opt.state[p].values()]
    return out, int(opt.sr_step)


@pytest.mark.parametrize("name", ['momentum', 'adagrad', 'adam'])
def test_repeat_and_graph_replay_give_the_same_bits(graph, name):
    a, sa = _table_run(name, False)
    b, sb = _table_run(name, False)
    c, sc = _table_run(name, True)
    assert sa == sb == sc == 5
    for x, y, z in zip(a, b, c):
        np.testing.assert_array_equal(x, y, err_msg="repeat")
        np.testing.assert_array_equal(x, z, err_msg="graph replay")


# ------------------------------------------------------------------------------------------------ training
def _models(kind, dim=32):
    from euler_b200 import unsupervised as un
    out = []
    for dt in (torch.bfloat16, torch.float32):
        torch.manual_seed(3)
        if kind == "deepwalk":
            out.append(un.DeepWalk(0, [0], 4096, dim, walk_len=3, num_negs=5, device="cuda", table_dtype=dt))
        else:
            out.append(un.Line(0, [0], 4096, dim, num_negs=5, order=2, device="cuda", table_dtype=dt))
    m16, m32 = out
    with torch.no_grad():   # one starting point: the f32 tables hold the bf16 tables' widened values
        for p16, p32 in zip(m16.parameters(), m32.parameters()):
            p32.copy_(p16.float())
    return m16, m32


@pytest.mark.parametrize("kind", ["deepwalk", "line"])
def test_training_tracks_f32(graph, kind):
    """300 Adam steps (lr 0.01) from the same tables and draws: the mean loss of the last 50 steps of bf16 training lies
    within 2 % of f32 training's, and both learn (the loss falls by more than 0.02 from the first 10 steps)"""
    import euler_b200
    from euler_b200 import optimizers
    m16, m32 = _models(kind)
    o16 = optimizers.get('adam')(list(m16.parameters()), 0.01, seed=5)
    o32 = optimizers.get('adam')(list(m32.parameters()), 0.01)
    rng = np.random.RandomState(4)
    l16, l32 = [], []
    for s in range(300):
        batch = torch.as_tensor(rng.randint(1, 4097, size=256), device="cuda")
        for m, o, out in ((m16, o16, l16), (m32, o32, l32)):
            euler_b200.seed(1000 + s)
            out.append(m.train_step(batch, o)[0])
    a = np.array([float(x) for x in l16])
    b = np.array([float(x) for x in l32])
    assert b[:10].mean() - b[-50:].mean() > 0.02, (b[:10].mean(), b[-50:].mean())
    assert a[:10].mean() - a[-50:].mean() > 0.02, (a[:10].mean(), a[-50:].mean())
    assert abs(a[-50:].mean() - b[-50:].mean()) <= 0.02 * b[-50:].mean(), (a[-50:].mean(), b[-50:].mean())
    assert m16.target_encoder.embeddings.dtype == torch.bfloat16


def test_stochastic_rounding_keeps_updates_round_to_nearest_drops(graph):
    """one plain SGD step whose typical update is 1/50 of a bf16 ulp: round to nearest (the control) leaves more than 90 %
    of the touched elements unchanged, while stochastic rounding's step, projected on the f32 step, has its full length"""
    import euler_b200
    from euler_b200 import ops, optimizers
    m16, _ = _models("deepwalk")
    euler_b200.seed(7)
    batch = torch.as_tensor(np.random.RandomState(8).randint(1, 4097, size=512), device="cuda")
    src, pos, negs = m16.to_sample(batch)
    tables = [m16.target_encoder.embeddings, m16.context_encoder.embeddings]
    _, _, grads = ops.skipgram_xent_loss_sparse_grads(src, pos, negs, *tables)
    old = [t.float() for t in tables]
    touched = [o[r] for o, (r, _) in zip(old, grads)]
    ulp = torch.cat([(2.0 ** (torch.floor(torch.log2(x.abs().clamp_min(1e-30))) - 7)).reshape(-1) for x in touched])
    gabs = torch.cat([v.abs().reshape(-1) for _, v in grads])
    lr = float(0.02 * ulp.median() / gabs[gabs > 0].median())
    delta = [-lr * v for _, v in grads]
    opt = optimizers.get('sgd')(tables, lr, seed=11)
    opt.apply_sparse(tables, [r for r, _ in grads], [v for _, v in grads])
    num = den = 0.0
    stalled = moved = 0
    for t, o, (r, _), d in zip(tables, old, grads, delta):
        sr_change = t.float()[r] - o[r]
        rn_change = (o[r] + d).to(torch.bfloat16).float() - o[r]   # the f32 SGD step, rounded to nearest
        nz = d != 0
        num += float((sr_change * d).sum())
        den += float((d * d).sum())
        stalled += int(((rn_change == 0) & nz).sum())
        moved += int(nz.sum())
    assert moved > 10000
    assert stalled > 0.9 * moved, (stalled, moved)
    assert 0.85 < num / den < 1.15, num / den


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_leave_every_table_untouched(graph):
    from euler_b200 import EulerError, ops, optimizers
    rng = np.random.RandomState(12)
    t16, _ = _table(rng, 50, 8, 0)
    s16, _ = _table(rng, 50, 8, 0)
    before = [_bits(t16), _bits(s16)]
    step = torch.zeros((), dtype=torch.int64, device="cuda")
    g = torch.ones((50, 8), dtype=torch.float32, device="cuda")
    src, pos, negs = _ids(*sk.pair_ids(rng, 10, 1, 2, 50))
    leaf = t16.clone().requires_grad_(True)
    with pytest.raises(EulerError, match="autograd"):
        ops.skipgram_xent_loss(src, pos, negs, leaf, leaf)
    with pytest.raises(EulerError, match="one dtype"):
        ops.skipgram_xent_loss(src, pos, negs, t16, t16.float())
    with pytest.raises(EulerError, match="step"):
        ops.optim_momentum_(t16, s16, g, 0.1, 0.9)                      # no step counter
    with pytest.raises(EulerError):
        ops.optim_momentum_(t16, s16.float(), g, 0.1, 0.9, step=step)   # a slot of another dtype
    with pytest.raises(EulerError):
        ops.optim_adagrad_(t16, s16, g.to(torch.bfloat16), 0.1, step=step)   # a bf16 gradient
    with pytest.raises(EulerError, match="dtype"):
        ops._call("eu_optim_momentum_dtype", t16, s16, 50, 8, g, None, -1, 0.1, 0.9, 7, 0, step, 0)
    with pytest.raises(EulerError, match="dtype"):
        ops._call("eu_skipgram_loss_dtype", src, pos, negs, 10, 1, 2, t16, t16, 50, 8, 5,
                  torch.empty((10, 3), device="cuda"), torch.empty(10, dtype=torch.int32, device="cuda"),
                  torch.empty((), device="cuda"))
    p = torch.nn.Parameter(t16, requires_grad=False)
    opt = optimizers.get('adam')([p], 0.01, seed=1)
    with pytest.raises(ValueError, match="float32"):
        opt.apply_sparse(p, torch.tensor([1], device="cuda"), torch.ones((1, 8), dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(ValueError, match="not one of"):
        opt.apply_sparse(torch.nn.Parameter(s16, requires_grad=False), torch.tensor([1], device="cuda"),
                         torch.ones((1, 8), device="cuda"))
    torch.cuda.synchronize()
    assert int(step) == 0 and int(opt.sr_step) == 0
    np.testing.assert_array_equal(_bits(t16), before[0])
    np.testing.assert_array_equal(_bits(s16), before[1])
