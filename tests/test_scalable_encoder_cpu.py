"""CPU: ScalableSageEncoder / ScalableGCNEncoder (constructor, widths, store shapes, the keyword decision, training=False,
and three consecutive training steps of the literal composition on a CPU stand-in of the graph ops), each step against a
float64 restatement of upstream's call (encoders.py:294-408, 629-748) with the pinned step order: the neighbour store rows
read at the start of the step, the exchange after the last layer (write keep-last, read, clear), then the accumulation
and both optimizers from the same parameters."""
import copy

import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import ops
from euler_b200.encoders import GCNEncoder, SageEncoder, ScalableGCNEncoder, ScalableSageEncoder, ShallowEncoder
from test_gcn_encoder_cpu import _multi_hop
from test_sage_encoder_cpu import _sample_fanout
from test_shallow_encoder_cpu import _dense_feature, _sparse_feature


@pytest.fixture
def cpu_ops(monkeypatch):
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    monkeypatch.setattr(ops, "get_sparse_feature", _sparse_feature)
    monkeypatch.setattr(ops, "sample_fanout", _sample_fanout)
    monkeypatch.setattr(ops, "get_multi_hop_neighbor", _multi_hop)


KW = dict(feature_idx=['f1', 'f2'], feature_dim=[4, 2], max_id=12, use_id=True, sparse_feature_idx=['s1', 's2'],
          sparse_feature_max_id=[9, 4], embedding_dim=[3, 2, 5], fused=False)


def test_constructor_errors_widths_and_stores():
    with pytest.raises(ValueError, match="divided exactly"):
        ScalableSageEncoder([0], 3, 2, 7, concat=True, **KW)
    with pytest.raises(ValueError, match="stores"):
        ScalableGCNEncoder([0], 2, 6, 'attention', head_num=4, **KW)            # layer 0 is 4 wide, the store 6
    with pytest.raises(ValueError, match="use_residual"):
        ScalableGCNEncoder([0], 2, 6, 'attention', head_num=4, use_residual=True, **KW)
    ScalableGCNEncoder([0], 1, 6, 'attention', head_num=4, **KW)               # one layer: nothing is stored
    for L in (1, 2, 3):
        s = ScalableSageEncoder([0], 3, L, 8, **KW)
        assert s.dims == [16] + [8] * L and s.metapath == [[0]] * L and s.fanouts == [3] * L
        assert [tuple(t.shape) for t in s.stores] == [(14, 8)] * (L - 1) == [tuple(t.shape) for t in s.gradient_stores]
        assert all(((t >= 0) & (t < 0.05)).all() for t in s.stores) and all((t == 0).all() for t in s.gradient_stores)
        g = ScalableGCNEncoder([0], L, 8, 'attention', head_num=2, **KW)
        assert g.dims == [16] + [8] * L and [tuple(t.shape) for t in g.stores] == [(14, 8)] * (L - 1)
        assert not any(k.startswith(('store', 'gradient_store')) for k in list(s.state_dict()) + list(g.state_dict()))
        assert isinstance(s.store_optimizer, torch.optim.Adam) and s.store_optimizer.defaults['lr'] == 0.001
    a = ScalableSageEncoder([0], 3, 2, 8, store_init_maxval=0.5, generator=torch.Generator().manual_seed(5), **KW)
    b = ScalableSageEncoder([0], 3, 2, 8, store_init_maxval=0.5, generator=torch.Generator().manual_seed(5), **KW)
    assert torch.equal(a.stores[0], b.stores[0]) and a.stores[0].max() > 0.05


def test_shared_node_encoder_and_use_residual_mean_what_they_say():
    # upstream passes (shared_node_encoder, use_residual) into SageEncoder's (use_residual, shared_node_encoder) slots
    shared = ShallowEncoder(feature_idx='f1', feature_dim=4, fused=False)
    enc = ScalableSageEncoder([0], 3, 2, 8, shared_node_encoder=shared, max_id=12, fused=False)
    assert enc._node_encoder is shared and enc.dims == [4, 8, 8]
    assert ScalableSageEncoder([0], 3, 2, 8, use_residual=True, **KW)._node_encoder is not shared


# ---------------------------------------------------------------------------- float64 restatement of one training step
class _Ref:
    """upstream's call and the pinned step in float64: a float64 copy of the encoder's layers (their math is checked
    against numpy in test_sage_encoder_cpu / test_gcn_encoder_cpu), the tables as numpy arrays, SGD and torch's Adam
    restated"""

    def __init__(self, enc, head, sage):
        self.m = copy.deepcopy(enc).double()
        self.head = head.detach().double().clone()
        self.sage = sage
        self.S = [s.double().numpy().copy() for s in enc.stores]
        self.G = [g.double().numpy().copy() for g in enc.gradient_stores]
        self.adam = {}

    def params(self):
        return [p for p in self.m.parameters() if p.requires_grad]

    def step(self, inputs, lr, store_lr):
        m = self.m
        L = m.num_layers
        if self.sage:
            node, neighbor = _sample_fanout(inputs, [m.edge_type], [m.fanout], default_node=m.max_id + 1)[0]
        else:
            (node, neighbor), (adj,) = _multi_hop(inputs, [m.edge_type])
        head = self.head.clone().requires_grad_()
        h, nb = _encode_f64(m._node_encoder, node), _encode_f64(m._node_encoder, neighbor)
        embs, leaves = [], []
        for layer in range(L):
            a = m.aggregators[layer]
            if self.sage:
                h = a((h, nb.reshape(-1, m.fanout, m.dims[layer])))
            else:
                out = a((h, nb, adj))
                h = h + out if m.use_residual else out
            embs.append(h)
            if layer < L - 1:
                nb = torch.tensor(self.S[layer][neighbor.numpy()], requires_grad=True)   # the store as the step began
                leaves.append(nb)
        taken = []
        for l in range(L - 1):                                   # the exchange, one id at a time in input order
            taken.append(self.G[l][node.numpy()].copy())
            for i, v in enumerate(node.tolist()):
                self.S[l][v] = embs[l][i].detach().numpy()       # a later occurrence overwrites: the last one wins
            self.G[l][node.numpy()] = 0
        store_loss = sum(((embs[l] * torch.tensor(taken[l])).sum() for l in range(L - 1)), torch.zeros((), dtype=torch.float64))
        loss = _loss(h, head)
        params = self.params()
        if leaves:
            for l, g in enumerate(torch.autograd.grad(loss + store_loss, leaves, retain_graph=True)):
                for e, v in enumerate(neighbor.tolist()):
                    self.G[l][v] += g[e].numpy()
        g_store = (torch.autograd.grad(store_loss, params, retain_graph=True, allow_unused=True) if store_loss.requires_grad
                   else [None] * len(params))
        g_loss = torch.autograd.grad(loss, params + [head], allow_unused=True)
        with torch.no_grad():
            for p, g in zip(params + [head], g_loss):
                if g is not None:
                    p -= lr * g
            for k, (p, g) in enumerate(zip(params, g_store)):   # torch.optim.Adam's defaults
                if g is None:
                    continue
                mt, vt, t = self.adam.get(k, (torch.zeros_like(p), torch.zeros_like(p), 0))
                t += 1
                mt = 0.9 * mt + 0.1 * g
                vt = 0.999 * vt + 0.001 * g * g
                p -= store_lr * (mt / (1 - 0.9 ** t)) / ((vt / (1 - 0.999 ** t)).sqrt() + 1e-8)
                self.adam[k] = (mt, vt, t)
        self.head = head.detach()
        return store_loss.item()


def _encode_f64(node_encoder, nodes):
    """the float64 node encoder, its dense features read in float64 ('add' maps them through its float64 Dense layer)"""
    mp = pytest.MonkeyPatch()
    mp.setattr(ops, "get_dense_feature", lambda *a, **k: [t.double() for t in _dense_feature(*a, **k)])
    try:
        return node_encoder(nodes)
    finally:
        mp.undo()


def _loss(h, head):
    return torch.tanh(h @ head).square().mean()


def _check(enc, head, ref, store_loss):
    f64 = lambda t: t.detach().double().numpy()   # noqa: E731
    for a, b in zip(enc.stores + enc.gradient_stores, ref.S + ref.G):
        np.testing.assert_allclose(f64(a), b, rtol=1e-5, atol=1e-5)
    for a, b in zip([p for p in enc.parameters() if p.requires_grad], ref.params()):
        np.testing.assert_allclose(f64(a), f64(b), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(f64(head), f64(ref.head), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(enc.store_loss.item(), store_loss, rtol=1e-5, atol=1e-5)


# seeds repeat (3, 5) and are neighbours of one another: 1 -> 3, 4 -> 12 (the default 13), 7 -> 8 (Sage); 3 -> 9, 10 (GCN)
BATCHES = [[3, 5, 11, 3, 7, 1], [9, 5, 5, 8, 2, 4], [3, 10, 6, 0, 9, 3]]


def _train(enc, sage):
    torch.manual_seed(7)
    head = torch.randn(enc.dims[-1], 1) * 0.5
    ref = _Ref(enc, head, sage)
    head.requires_grad_()
    opt = torch.optim.SGD(list(enc.parameters()) + [head], lr=0.05)
    for batch in BATCHES:
        inputs = torch.as_tensor(batch, dtype=torch.int64)
        out = enc(inputs, training=True)
        assert out.shape == (len(batch), enc.dims[-1])
        enc.train_step(_loss(out, head), opt)
        _check(enc, head, ref, ref.step(inputs, 0.05, 0.01))
    assert any((g != 0).any() for g in enc.gradient_stores) or enc.num_layers == 1


@pytest.mark.parametrize("layers", (1, 2, 3))
@pytest.mark.parametrize("aggregator", ("mean", "gcn", "meanpool"))
def test_sage_training_steps_against_float64(cpu_ops, aggregator, layers):
    torch.manual_seed(0)
    enc = ScalableSageEncoder([0], 3, layers, 6, aggregator=aggregator, store_learning_rate=0.01, store_init_maxval=0.5,
                              generator=torch.Generator().manual_seed(1), **KW)
    _train(enc, True)


@pytest.mark.parametrize("use_residual", (False, True))
@pytest.mark.parametrize("aggregator", ("gcn", "mean", "attention"))
def test_gcn_training_steps_against_float64(cpu_ops, aggregator, use_residual):
    torch.manual_seed(0)
    enc = ScalableGCNEncoder([0], 3, 8, aggregator, use_residual=use_residual, head_num=2, store_learning_rate=0.01,
                             store_init_maxval=0.5, generator=torch.Generator().manual_seed(1), **KW)
    _train(enc, False)


def test_inference_is_the_plain_encoder(cpu_ops):
    torch.manual_seed(0)
    s = ScalableSageEncoder([0], 3, 2, 6, aggregator='gcn', **KW)
    plain = SageEncoder([[0]] * 2, [3, 3], 6, aggregator='gcn', **KW)
    plain.load_state_dict(s.state_dict())
    inputs = torch.as_tensor([[3, 5], [11, 8]], dtype=torch.int64)
    assert torch.equal(s(inputs), plain(inputs))
    g = ScalableGCNEncoder([0], 2, 8, 'attention', head_num=2, use_residual=True, **KW)
    gplain = GCNEncoder([[0]] * 2, 8, 'attention', head_num=2, use_residual=True, **KW)
    gplain.load_state_dict(g.state_dict())
    assert torch.equal(g(inputs), gplain(inputs))
    assert s.store_loss is None and g.store_loss is None          # inference touches no store
