"""CPU: the sparse aggregators' composition (fused=False), GCNEncoder / GenieEncoder (constructor, widths, the literal
composition on a CPU stand-in of get_multi_hop_neighbor) and GeniePath's step, each against a float64 numpy restatement of
upstream's sparse_aggregators.py / encoders.py."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import ops, sparse_aggregators
from euler_b200.encoders import GCNEncoder, GenieEncoder
from euler_b200.supervised import GeniePath, f1_score
from test_shallow_encoder_cpu import _dense_feature, _sparse_feature, _restated as _shallow_f64


def f64(t):
    return t.detach().double().numpy()


def relu(x):
    return np.maximum(x, 0)


def _act(fn):
    return relu if fn is not None else (lambda v: v)


# ---------------------------------------------------------------------------- float64 restatement of sparse_aggregators.py
def _adj_sum_f64(nb, indptr, cols):
    n = len(indptr) - 1
    out = np.zeros((n, nb.shape[1]))
    for i in range(n):
        for k in range(indptr[i], indptr[i + 1]):
            out[i] += nb[cols[k]]
    return out, np.diff(indptr).astype(np.float64)[:, None]


def _head_f64(x, nb, indptr, cols, kernel, w_self, w_neigh, renorm):
    """SingleAttentionAggregator.call before its activation, for one head"""
    n = len(x)
    if renorm:
        fa = np.concatenate([x, nb]) @ kernel
        fs = fa[:n]
        rows = [[i] + [c + n for c in cols[indptr[i]:indptr[i + 1]]] for i in range(n)]
    else:
        fa, fs = nb @ kernel, x @ kernel
        rows = [list(cols[indptr[i]:indptr[i + 1]]) for i in range(n)]
    sw, aw = fs @ w_self, fa @ w_neigh
    out = np.zeros((n, kernel.shape[1]))
    for i, r in enumerate(rows):
        if not r:
            continue
        u = np.array([sw[i, 0] + aw[c, 0] for c in r])
        u = np.where(u > 0, u, 0.2 * u)
        a = np.exp(u - u.max())
        a /= a.sum()
        out[i] = sum(a_k * fa[c] for a_k, c in zip(a, r))
    return out if renorm else fs + out


def _aggregate_f64(a, x, nb, indptr, cols):
    if isinstance(a, sparse_aggregators.GCNAggregator):
        S, deg = _adj_sum_f64(nb, indptr, cols)
        agg = (x + S) / (1 + deg) if a.renorm else x + S / np.maximum(deg, 1e-7)
        return _act(a.dense.activation)(agg @ f64(a.dense.kernel))
    if isinstance(a, sparse_aggregators.MeanAggregator):
        S, deg = _adj_sum_f64(nb, indptr, cols)
        act = _act(a.self_layer.activation)
        s, m = act(x @ f64(a.self_layer.kernel)), act((S / np.maximum(deg, 1e-7)) @ f64(a.neigh_layer.kernel))
        return np.concatenate([s, m], 1) if a.concat else s + m
    heads = a.attentions if isinstance(a, sparse_aggregators.AttentionAggregator) else [a]
    out = np.concatenate([_head_f64(x, nb, indptr, cols, f64(h.dense.kernel), f64(h.self_layer.kernel), f64(h.neigh_layer.kernel),
                                    a.renorm) for h in heads], 1)
    return _act(a.activation)(out)


def _adjacency(n, m, seed=0):
    """rows of 0 .. 5 entries with repeated columns (multi-edges); row 1 always empty"""
    rng = np.random.RandomState(seed)
    lens = rng.randint(0, 6, size=n) if m else np.zeros(n, np.int64)
    lens[1] = 0
    cols = [np.sort(rng.randint(0, m, size=k)) for k in lens] if m else []
    if m and lens.max() >= 2:
        r = int(np.argmax(lens))
        cols[r][1] = cols[r][0]                 # a duplicate entry
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    cols = np.concatenate(cols).astype(np.int64) if m else np.zeros(0, np.int64)
    return indptr, cols


def _build(name, kw):
    torch.manual_seed(1)
    return sparse_aggregators.get(name)(7, 8, fused=False, **kw)


CASES = [("gcn", dict()), ("gcn", dict(renorm=True)), ("gcn", dict(activation=None)),
         ("mean", dict()), ("mean", dict(concat=True)), ("mean", dict(activation=None)),
         ("attention", dict(head_num=1)), ("attention", dict(head_num=2, activation=None)), ("attention", dict(head_num=4)),
         ("attention", dict(head_num=2, renorm=True)), ("attention", dict(head_num=4, renorm=True, activation=None))]


@pytest.mark.parametrize("m", (9, 0))
@pytest.mark.parametrize("name,kw", CASES)
def test_aggregators_against_float64(name, kw, m):
    a = _build(name, kw)
    n = 6
    indptr, cols = _adjacency(n, m)
    x, nb = torch.randn(n, 7), torch.randn(m, 7)
    adj = (torch.as_tensor(indptr), torch.as_tensor(cols), torch.ones(len(cols)))
    out = a((x, nb, adj))
    assert out.shape == (n, a.output_dim) and out.dtype == torch.float32
    want = _aggregate_f64(a, f64(x), f64(nb), indptr, cols)
    np.testing.assert_allclose(f64(out), want, rtol=1e-5, atol=1e-6)
    out.square().sum().backward()                                        # the composition is differentiable
    assert all(p.grad is not None for p in a.parameters())


def test_single_attention_is_one_head_and_widths():
    torch.manual_seed(0)
    one = sparse_aggregators.SingleAttentionAggregator(7, 5, fused=False)
    assert one.dense.bias is None and tuple(one.self_layer.kernel.shape) == (5, 1) and one.output_dim == 5
    x, nb = torch.randn(4, 7), torch.randn(6, 7)
    indptr, cols = _adjacency(4, 6, seed=3)
    np.testing.assert_allclose(f64(one((x, nb, (torch.as_tensor(indptr), torch.as_tensor(cols))))),
                               _aggregate_f64(one, f64(x), f64(nb), indptr, cols), rtol=1e-5, atol=1e-6)
    assert sparse_aggregators.AttentionAggregator(7, 10, head_num=4, fused=False).output_dim == 8    # 4 * (10 // 4)
    assert sparse_aggregators.MeanAggregator(7, 7, concat=True, fused=False).output_dim == 6         # upstream rounds down
    assert sparse_aggregators.get('gcn') is sparse_aggregators.GCNAggregator
    assert sparse_aggregators.get('maxpool') is None
    assert sparse_aggregators.GCNAggregator(7, 3, head_num=4).output_dim == 3    # head_num is taken and ignored


# ---------------------------------------------------------------------------- encoders on a CPU stand-in
def _multi_hop(nodes, edge_types, sampler=None):
    """a deterministic stand-in of get_multi_hop_neighbor: node v lists (3 v + k) % 13 for k < v % 4, and (3 v) % 13 once
    more when v % 4 == 3 (a multi-edge); columns in first-occurrence order, each row's entries ordered by column"""
    nodes = torch.as_tensor(nodes, dtype=torch.int64).reshape(-1)
    nodes_list, adj_list = [nodes], []
    for _ in edge_types:
        listing = [[(3 * v + k) % 13 for k in range(v % 4)] + ([(3 * v) % 13] if v % 4 == 3 else []) for v in nodes.tolist()]
        uniq = list(dict.fromkeys(x for row in listing for x in row))
        pos = {v: i for i, v in enumerate(uniq)}
        rows = [sorted(pos[x] for x in row) for row in listing]
        indptr = torch.as_tensor(np.concatenate([[0], np.cumsum([len(r) for r in rows])]), dtype=torch.int64)
        cols = torch.as_tensor([c for r in rows for c in r], dtype=torch.int64)
        nodes = torch.as_tensor(uniq, dtype=torch.int64)
        nodes_list.append(nodes)
        adj_list.append((indptr, cols, torch.ones(len(cols))))
    return nodes_list, adj_list


@pytest.fixture
def cpu_ops(monkeypatch):
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    monkeypatch.setattr(ops, "get_sparse_feature", _sparse_feature)
    monkeypatch.setattr(ops, "get_multi_hop_neighbor", _multi_hop)


KW = dict(feature_idx=['f1', 'f2'], feature_dim=[4, 2], max_id=12, use_id=True, sparse_feature_idx=['s1', 's2'],
          sparse_feature_max_id=[9, 4], embedding_dim=[3, 2, 5], fused=False)


def test_constructor_errors_and_widths():
    with pytest.raises(AssertionError):
        GCNEncoder([[0], [0]], 8, head_num=[4])
    with pytest.raises(ValueError, match="head_num"):
        GCNEncoder([[0]], 8, head_num='4')
    with pytest.raises(ValueError, match="use_residual"):
        GCNEncoder([[0]], 6, 'attention', head_num=4, use_residual=True, **KW)        # width 4 != dim 6
    with pytest.raises(NotImplementedError):
        GCNEncoder([[0]], 8, max_id=5, use_id=True, use_hash_embedding=True)
    enc = GCNEncoder([[0], [0], [0]], 8, 'attention', head_num=[4, 2, 3], **KW)
    assert enc.dims == [16, 8, 8, 6] and enc.head_num == [4, 2, 3] and len(enc.aggregators) == 3
    assert [a.activation is not None for a in enc.aggregators] == [True, True, False]   # relu on all but the last layer
    assert tuple(enc.aggregators[1].attentions[0].dense.kernel.shape) == (8, 4)           # layer 1 reads layer 0's width
    assert GCNEncoder([[0]], 8, feature_idx='f1', feature_dim=4, max_id=12).dims == [4, 8]   # use_id unset: no id embedding
    res = GCNEncoder([[0], [0]], 8, 'gcn', use_residual=True, **KW)
    assert res.dims == [8, 8, 8] and res._node_encoder.combiner == 'add'
    genie = GenieEncoder([[0], [0]], 8, head_num=2, **KW)
    assert genie.dims == [16, 8, 8] and [tuple(d.kernel.shape) for d in genie.depth_fc] == [(16, 8), (8, 8), (8, 8)]
    assert all(torch.all(d.bias == 0.0002) for d in genie.depth_fc)                     # layers.Dense's default bias
    assert tuple(genie.lstm_cell.kernel.shape) == (16, 32)


def _gcn_f64(enc, inputs):
    """GCNEncoder.call's loop (encoders.py:214-233) in float64; also returns each layer's seed rows"""
    nodes, adjs = _multi_hop(inputs, enc.metapath)
    hidden = [_shallow_f64(enc._node_encoder, n.numpy()) for n in nodes]
    seeds = [hidden[0]]
    for layer in range(enc.num_layers):
        a = enc.aggregators[layer]
        nxt = []
        for hop in range(enc.num_layers - layer):
            h = _aggregate_f64(a, hidden[hop], hidden[hop + 1], adjs[hop][0].numpy(), adjs[hop][1].numpy())
            nxt.append(hidden[hop] + h if enc.use_residual else h)
        hidden = nxt
        seeds.append(hidden[0])
    return hidden[0], seeds


@pytest.mark.parametrize("use_residual", (False, True))
@pytest.mark.parametrize("aggregator", ("gcn", "mean", "attention"))
@pytest.mark.parametrize("layers", (1, 2, 3))
def test_gcn_encoder_against_float64(cpu_ops, layers, aggregator, use_residual):
    torch.manual_seed(0)
    enc = GCNEncoder([[0]] * layers, 8, aggregator, use_residual=use_residual, head_num=2, **KW)
    inputs = torch.as_tensor([[3, 5], [11, 8], [2, 7]], dtype=torch.int64)
    out = enc(inputs)
    assert out.shape == (3, 2, 8) and out.dtype == torch.float32
    np.testing.assert_allclose(f64(out).reshape(-1, 8), _gcn_f64(enc, inputs)[0], rtol=1e-5, atol=1e-6)


def _sigmoid(x):
    return 1 / (1 + np.exp(-x))


def _genie_f64(enc, inputs):
    """GenieEncoder.call (encoders.py:262-291) in float64: the LSTM's first step from a zero state"""
    _, seeds = _gcn_f64(enc, inputs)
    x = seeds[0] @ f64(enc.depth_fc[0].kernel) + f64(enc.depth_fc[0].bias)
    z = np.concatenate([x, np.zeros_like(x)], 1) @ f64(enc.lstm_cell.kernel) + f64(enc.lstm_cell.bias)
    i, j, f, o = np.split(z, 4, axis=1)
    c = _sigmoid(i) * np.tanh(j)                   # + sigmoid(f + 1) * 0
    return _sigmoid(o) * np.tanh(c)


@pytest.mark.parametrize("use_residual", (False, True))
def test_genie_encoder_against_float64(cpu_ops, use_residual):
    torch.manual_seed(0)
    enc = GenieEncoder([[0], [0]], 8, use_residual=use_residual, head_num=2, **KW)
    inputs = torch.as_tensor([3, 5, 11, 8, 2, 7], dtype=torch.int64)
    out = enc(inputs)
    assert out.shape == (6, 8)
    np.testing.assert_allclose(f64(out), _genie_f64(enc, inputs), rtol=1e-5, atol=1e-6)
    out.sum().backward()
    assert enc.depth_fc[0].kernel.grad is not None and enc.lstm_cell.kernel.grad is not None
    # outputs[:, 0, :]: the aggregators and the later depth layers never reach the result
    assert all(p.grad is None for p in enc.aggregators.parameters())
    assert all(p.grad is None for d in enc.depth_fc[1:] for p in d.parameters())


def _xent(x, z):
    return np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))


def test_geniepath_step_against_float64(cpu_ops):
    torch.manual_seed(0)
    kw = {k: v for k, v in KW.items() if k != 'fused'}
    model = GeniePath(8, [[0], [0]], 'f1', 3, head_num=2, fused=False, **kw)
    assert isinstance(model._encoder, GenieEncoder) and model._encoder.head_num == [2, 2]
    inputs = torch.as_tensor([3, 5, 11, 8, 2], dtype=torch.int64)
    emb, loss, name, metric = model(inputs)
    h = _genie_f64(model._encoder, inputs)
    logit = h @ f64(model.out_fc.weight).T
    label = _dense_feature(inputs, ['f1'], [3])[0].double().numpy()
    assert name == 'f1' and emb.shape == (5, 8)
    np.testing.assert_allclose(f64(emb), h, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(loss.item(), _xent(logit, label).mean(), rtol=1e-5)
    np.testing.assert_allclose(float(metric), float(f1_score(torch.as_tensor(label), torch.as_tensor(_sigmoid(logit)))), rtol=1e-6)
    loss.backward()
    assert model.out_fc.weight.grad is not None and model._encoder.depth_fc[0].kernel.grad is not None
