"""CPU: the node encoders' bfloat16 tables without a device -- the constructors' refusals, the tables' dtypes, the proxies
(neither parameters nor state), optimizers' step(sparse_grads=) against .grad, and minimize's wiring on a stand-in op."""
import pytest
import torch

from euler_b200 import encoders, optimizers, ops, supervised, unsupervised


def _shallow(dt, **kw):
    torch.manual_seed(0)
    return encoders.ShallowEncoder(feature_idx=-1, max_id=20, sparse_feature_idx=['a', 'b'], sparse_feature_max_id=[9, 4],
                                   embedding_dim=[8, 4, 4], table_dtype=dt, **kw)


def test_constructor_refusals():
    with pytest.raises(ValueError, match="table_dtype"):
        _shallow(torch.float16)
    with pytest.raises(ValueError, match="fused=True"):
        _shallow(torch.bfloat16, fused=False)
    with pytest.raises(ValueError, match="fused=True"):
        encoders.SageEncoder([[0]], [3], 8, max_id=20, use_id=True, fused=False, table_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="float32 tables only"):
        encoders.ScalableSageEncoder(0, 3, 2, 8, max_id=20, use_id=True, table_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="float32 tables only"):
        encoders.ScalableGCNEncoder(0, 2, 8, max_id=20, use_id=True, table_dtype=torch.bfloat16)


def test_table_dtypes_and_proxies():
    e16, e32 = _shallow(torch.bfloat16), _shallow(torch.float32)
    tables16 = [e16.embedding.embeddings] + [s.embeddings for s in e16.sparse_embeddings]
    tables32 = [e32.embedding.embeddings] + [s.embeddings for s in e32.sparse_embeddings]
    for a, b in zip(tables16, tables32):
        assert a.dtype == torch.bfloat16 and not a.requires_grad
        assert b.dtype == torch.float32 and b.requires_grad
        assert torch.equal(a, b.to(torch.bfloat16))   # initialised in f32 and rounded once to nearest
    assert e32.table_proxies() == []
    pairs = e16.table_proxies()
    assert [t for t, _ in pairs] == tables16
    for t, q in pairs:
        assert q.dtype == torch.float32 and q.shape == t.shape and q.requires_grad and q.is_leaf
        assert q.untyped_storage().nbytes() == 4   # one element, strides 0
    assert [q for _, q in e16.table_proxies()] == [q for _, q in pairs]   # made once
    params = {id(p) for p in e16.parameters()}
    assert not any(id(q) in params for _, q in pairs)
    state = e16.state_dict()
    assert sorted(state) == ['embedding.embeddings', 'sparse_embeddings.0.embeddings', 'sparse_embeddings.1.embeddings']
    assert all(v.dtype == torch.bfloat16 for v in state.values())


def test_models_pass_table_dtype():
    sage = encoders.SageEncoder([[0], [0]], [3, 2], 8, max_id=20, use_id=True, table_dtype=torch.bfloat16)
    gcn = encoders.GCNEncoder([[0]], 8, max_id=20, use_id=True, use_residual=True, table_dtype=torch.bfloat16)
    genie = supervised.GeniePath(8, [[0]], 'label', 2, max_id=20, use_id=True, table_dtype=torch.bfloat16)
    dgi = unsupervised.DGI(0, 0, 20, [[0]], [3], 8, use_id=True, table_dtype=torch.bfloat16)
    for m in (sage, gcn, genie, dgi):
        tables = [p for p in m.parameters() if p.dim() == 2 and p.shape[0] == 22]
        assert tables and all(t.dtype == torch.bfloat16 for t in tables)


def test_proxy_refusals_before_device_work():
    t16 = torch.zeros(5, 4, dtype=torch.bfloat16)
    with pytest.raises(ops.EulerError, match="one dtype"):
        ops._check_tables("op", [("a", t16), ("b", torch.zeros(5, 4))])
    with pytest.raises(ops.EulerError, match="autograd"):
        ops._check_tables("op", [("a", t16.clone().requires_grad_())])
    with pytest.raises(ops.EulerError, match="bfloat16 table only"):
        ops._check_tables("op", [("a", torch.zeros(5, 4))], [ops.table_proxy(torch.zeros(5, 4))])
    with pytest.raises(ops.EulerError, match="shape"):
        ops._check_tables("op", [("a", t16)], [ops.table_proxy(torch.zeros(6, 4))])
    with pytest.raises(ops.EulerError, match="one entry per table"):
        ops._check_tables("op", [("a", t16)], [])
    assert ops._check_tables("op", [("a", None), ("b", t16)])[0] == torch.bfloat16


def _sparse(rows, vals, shape):
    return torch.sparse_coo_tensor(torch.tensor([rows]), torch.tensor(vals, dtype=torch.float32), shape).coalesce()


@pytest.mark.parametrize("name", ['sgd', 'momentum', 'adagrad', 'adam'])
def test_step_sparse_grads_equals_grad(name):
    """step(sparse_grads={p: g}) is p.grad = g; step(), bit for bit; Adam's powers advance once per step"""
    res = []
    for via_keyword in (True, False):
        torch.manual_seed(1)
        table = torch.nn.Parameter(torch.randn(6, 3))
        dense = torch.nn.Parameter(torch.randn(3, 2))
        opt = optimizers.get(name)([table, dense], 0.1, fused=False)
        for s in range(3):
            g = _sparse([1, 4, 1], [[0.5 + s, -1.0, 2.0], [3.0, 0.25, -0.5], [1.0, 1.0, 1.0]], (6, 3))
            dense.grad = torch.full((3, 2), 0.125 * (s + 1))
            if via_keyword:
                table.grad = None
                opt.step(sparse_grads={table: g})
            else:
                table.grad = g
                opt.step()
        res.append((table.detach().clone(), dense.detach().clone(), getattr(opt, 'beta_powers', None)))
    (a, b, pa), (c, d, pc) = res
    assert torch.equal(a.view(torch.int32), c.view(torch.int32)) and torch.equal(b.view(torch.int32), d.view(torch.int32))
    if name == 'adam':
        assert torch.equal(pa, pc)
        assert torch.equal(pa, torch.tensor([0.9, 0.999], dtype=torch.float32) ** 4)


def test_step_sparse_grads_refusals():
    p = torch.nn.Parameter(torch.zeros(4, 2))
    opt = optimizers.get('sgd')([p], 0.1, fused=False)
    with pytest.raises(ValueError, match="not one of"):
        opt.step(sparse_grads={torch.nn.Parameter(torch.zeros(4, 2)): _sparse([0], [[1.0, 1.0]], (4, 2))})
    with pytest.raises(ValueError, match="sparse COO"):
        opt.step(sparse_grads={p: torch.zeros(4, 2)})


class _StandIn(torch.autograd.Function):
    """a CPU stand-in for the fused ops: the widened rows of `ids`, the coalesced sparse gradient to the proxy"""

    @staticmethod
    def forward(ctx, proxy, table, ids):
        ctx.save_for_backward(ids)
        ctx.shape = tuple(table.shape)
        return table.float()[ids]

    @staticmethod
    def backward(ctx, g):
        ids, = ctx.saved_tensors
        return torch.sparse_coo_tensor(ids.reshape(1, -1), g, ctx.shape).coalesce(), None, None


class _Model(torch.nn.Module):
    """two uses of one shared bf16 encoder (as SageEncoder's hops), then a dense layer"""

    def __init__(self):
        super().__init__()
        self.enc = _shallow(torch.bfloat16)
        self.also = self.enc   # a shared node encoder is collected once
        self.fc = torch.nn.Linear(16, 1)

    def forward(self, ids):
        outs = []
        for use in (ids, ids.flip(0)):
            id_table, _, sparse, proxies = self.enc._op_inputs()
            tables = [id_table] + [s[1] for s in sparse]
            outs.append(torch.cat([_StandIn.apply(q, t, use % t.shape[0]) for t, q in zip(tables, proxies)], 1))
        return self.fc(outs[0] + outs[1]).square().sum()


class _Recorder:
    def __init__(self, params):
        self.params, self.calls = params, []

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    def step(self, sparse_grads=None):
        self.calls.append(({id(k): v for k, v in sparse_grads.items()}, [p.grad for p in self.params]))


def test_minimize_wiring():
    m = _Model()
    pairs = m.enc.table_proxies()
    for _, q in pairs:
        q.grad = ops.table_proxy(q).detach()   # stale: minimize clears it before the backward pass
    dense = [p for p in m.parameters() if p.requires_grad]
    opt = _Recorder(dense)
    ids = torch.tensor([3, 7, 3, 1])
    loss = m(ids)
    assert optimizers.minimize(opt, loss, m) is loss
    assert len(opt.calls) == 1
    got, dense_grads = opt.calls[0]
    assert sorted(got) == sorted(id(t) for t, _ in pairs)
    assert all(g is not None for g in dense_grads)
    # the reference: f32 tables holding the widened values, sparse gradients through the same graph
    ref = _Model()
    ref.load_state_dict(m.state_dict())
    tables = [t.detach().float().requires_grad_() for t, _ in pairs]
    outs = []
    for use in (ids, ids.flip(0)):
        outs.append(torch.cat([torch.nn.functional.embedding(use % t.shape[0], t, sparse=True) for t in tables], 1))
    ref.fc(outs[0] + outs[1]).square().sum().backward()
    for (t, _), r in zip(pairs, tables):
        g = got[id(t)]
        assert g.is_sparse and g.shape == t.shape
        # the two sides add a repeated row's entries in different orders: the wiring is checked, not the rounding
        torch.testing.assert_close(g.coalesce().to_dense(), r.grad.coalesce().to_dense(), rtol=1e-6, atol=1e-7)


def test_minimize_without_bf16_tables_is_zero_grad_backward_step():
    torch.manual_seed(2)
    lin = torch.nn.Linear(3, 1)
    opt = optimizers.get('sgd')(list(lin.parameters()), 0.5, fused=False)
    x = torch.randn(4, 3)
    want = [p.detach().clone() for p in lin.parameters()]
    loss = lin(x).sum()
    grads = torch.autograd.grad(loss, list(lin.parameters()), retain_graph=True)
    for w, g in zip(want, grads):
        w.sub_(0.5 * g)
    for p in lin.parameters():
        p.grad = torch.full_like(p, 9.0)   # stale
    optimizers.minimize(opt, loss, lin)
    for p, w in zip(lin.parameters(), want):
        assert torch.equal(p.detach(), w)
