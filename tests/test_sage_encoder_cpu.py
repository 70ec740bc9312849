"""CPU: the aggregators, SageEncoder / ShuffleSageEncoder (constructor, dims, the literal composition on a CPU stand-in of the
graph ops), f1_score, SuperviseModel and DGI, each against a float64 numpy restatement of upstream's code."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import aggregators, ops
from euler_b200.encoders import Dense, SageEncoder, ShuffleSageEncoder
from euler_b200.supervised import SuperviseModel, f1_score
from euler_b200.unsupervised import DGI
from test_shallow_encoder_cpu import _dense_feature, _sparse_feature, _restated as _shallow_f64


def f64(t):
    return t.detach().double().numpy()


def relu(x):
    return np.maximum(x, 0)


# ---------------------------------------------------------------------------- aggregators
def _aggregate_f64(a, x, nb):
    """aggregators.py in float64 from the module's parameters; activation: relu where the module has one"""
    act = (lambda v: relu(v)) if getattr(a, 'dense', getattr(a, 'self_layer', None)).activation else (lambda v: v)
    if isinstance(a, aggregators.GCNAggregator):
        return act(np.concatenate([x[:, None], nb], 1).mean(1) @ f64(a.dense.kernel))
    if isinstance(a, aggregators.MeanAggregator):
        agg = nb.mean(1)
    else:
        h = relu(nb @ f64(a.layers[0].kernel) + f64(a.layers[0].bias))
        agg = h.mean(1) if isinstance(a, aggregators.MeanPoolAggregator) else h.max(1)
    s, n = act(x @ f64(a.self_layer.kernel)), act(agg @ f64(a.neigh_layer.kernel))
    return np.concatenate([s, n], 1) if a.concat else s + n


@pytest.mark.parametrize("activation", (torch.relu, None))
@pytest.mark.parametrize("concat", (False, True))
@pytest.mark.parametrize("name", ("gcn", "mean", "meanpool", "maxpool"))
def test_aggregators_against_float64(name, concat, activation):
    torch.manual_seed(1)
    a = aggregators.get(name)(7, 6, activation=activation, concat=concat)
    x, nb = torch.randn(5, 7), torch.randn(5, 4, 7)
    out = a((x, nb))
    assert out.shape == (5, 6) and out.dtype == torch.float32
    np.testing.assert_allclose(f64(out), _aggregate_f64(a, f64(x), f64(nb)), rtol=1e-5, atol=1e-6)
    if name in ("gcn", "mean"):
        pooled = nb.mean(1) if a.pooled_input == 'mean' else nb.sum(1)
        np.testing.assert_allclose(f64(a.forward_pooled(x, pooled, 4)), f64(out), rtol=1e-5, atol=1e-6)
    else:
        assert not hasattr(a, 'forward_pooled')
        assert tuple(a.layers[0].kernel.shape) == (7, 6) and torch.all(a.layers[0].bias == 0.0002)   # the un-halved dim, with bias
        assert a.self_layer.bias is None and a.neigh_layer.bias is None


def test_aggregator_errors_and_lookup():
    for name in ("mean", "meanpool", "maxpool"):
        with pytest.raises(ValueError, match="divided exactly"):
            aggregators.get(name)(4, 5, concat=True)
    assert aggregators.get("lstm") is None
    d = Dense(3, 2, activation=torch.relu, use_bias=True)
    assert torch.all(d.bias == 0.0002) and (d.kernel.abs() <= 0.36).all()
    assert Dense(3, 2).bias is None


# ---------------------------------------------------------------------------- the sample tree on a CPU stand-in
def _sample_fanout(nodes, edge_types, counts, default_node=-1):
    """a deterministic stand-in: neighbour k of node n is (3 n + k) % 13, or default_node where that is 12"""
    ids = [torch.as_tensor(nodes, dtype=torch.int64).reshape(-1)]
    for c in counts:
        nb = (3 * ids[-1][:, None] + torch.arange(c)[None, :]) % 13
        ids.append(torch.where(nb == 12, torch.full_like(nb, default_node), nb).reshape(-1))
    return ids, None, None


@pytest.fixture
def cpu_ops(monkeypatch):
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    monkeypatch.setattr(ops, "get_sparse_feature", _sparse_feature)
    monkeypatch.setattr(ops, "sample_fanout", _sample_fanout)


KW = dict(feature_idx=['f1', 'f2'], feature_dim=[4, 2], max_id=12, use_id=True, sparse_feature_idx=['s1', 's2'],
          sparse_feature_max_id=[9, 4], embedding_dim=[3, 2, 5], fused=False)


def test_constructor_errors_and_dims():
    with pytest.raises(ValueError, match="metapath"):
        SageEncoder([[0]], [3, 2], 8)
    with pytest.raises(ValueError, match="divided exactly"):
        SageEncoder([[0]], [3], 7, concat=True)
    with pytest.raises(NotImplementedError):
        SageEncoder([[0]], [3], 8, max_id=5, use_id=True, use_hash_embedding=True)
    enc = SageEncoder([[0], [0], [0]], [3, 2, 2], 8, **KW)
    assert enc.dims == [16, 8, 8, 8] and enc.num_layers == 3 and len(enc.aggregators) == 3
    assert [bool(a.self_layer.activation) for a in enc.aggregators] == [True, True, False]   # relu on all but the last layer
    assert SageEncoder([[0]], [3], 8, feature_idx='f1', feature_dim=4, max_id=12).dims == [4, 8]   # use_id unset: no id embedding
    shared = enc.aggregators
    assert SageEncoder([[0], [0], [0]], [3, 2, 2], 8, shared_aggregators=shared, **KW).aggregators is shared


def _sage_f64(enc, samples):
    """SageEncoder.call's loop (encoders.py:479-489) in float64"""
    hidden = [_shallow_f64(enc._node_encoder, s.numpy()) for s in samples]
    for layer in range(enc.num_layers):
        a = enc.aggregators[layer]
        hidden = [_aggregate_f64(a, hidden[hop], hidden[hop + 1].reshape(-1, enc.fanouts[hop], enc.dims[layer]))
                  for hop in range(enc.num_layers - layer)]
    return hidden[0]


@pytest.mark.parametrize("aggregator", ("mean", "gcn", "maxpool"))
@pytest.mark.parametrize("fanouts", ([3], [3, 2], [2, 2, 3]))
def test_composition_against_float64(cpu_ops, fanouts, aggregator):
    torch.manual_seed(0)
    enc = SageEncoder([[0]] * len(fanouts), fanouts, 6, aggregator=aggregator, **KW)
    inputs = torch.as_tensor([[3, 5], [11, 8], [2, 3]], dtype=torch.int64)
    out = enc(inputs)
    assert out.shape == (3, 2, 6) and out.dtype == torch.float32
    samples = _sample_fanout(inputs, None, fanouts, default_node=13)[0]
    np.testing.assert_allclose(f64(out).reshape(-1, 6), _sage_f64(enc, samples), rtol=1e-5, atol=1e-6)


def test_shuffling_ids_is_upstreams_shuffle_of_the_rows(cpu_ops):
    """shuffle_samples + the node encoder == encoders.py:502-514 on the encoded rows, under the same permutation"""
    torch.manual_seed(0)
    enc = ShuffleSageEncoder([[0], [0]], [3, 2], 6, **KW)
    inputs = torch.as_tensor([3, 5, 11, 8], dtype=torch.int64)
    samples = enc.sample(inputs)
    shuffled = enc.shuffle_samples(samples, torch.Generator().manual_seed(4))
    assert [s.shape for s in shuffled] == [s.shape for s in samples]                  # split sizes preserved
    perm = torch.randperm(1 + 3 + 6, generator=torch.Generator().manual_seed(4)).numpy()
    assert not np.array_equal(perm, np.arange(10))
    hidden = [f64(enc.node_encoder(s)) for s in samples]
    B, D = 4, enc.dims[0]
    rows = np.concatenate([h.reshape(B, -1, D) for h in hidden], 1).transpose(1, 0, 2)   # [positions, batch, dim]
    rows = rows[perm].transpose(1, 0, 2).reshape(-1, D)                                   # random_shuffle permutes axis 0
    want = np.split(rows, np.cumsum([len(h) for h in hidden])[:-1])
    for s, w in zip(shuffled, want):
        np.testing.assert_array_equal(f64(enc.node_encoder(s)), w)
    h, h_neg = enc(inputs, torch.Generator().manual_seed(4))
    np.testing.assert_allclose(f64(h), _sage_f64(enc, samples), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(f64(h_neg), _sage_f64(enc, shuffled), rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------- models
def test_f1_score_hand_cases():
    def want(tp, fp, fn):
        p, r = tp / (1e-7 + tp + fp), tp / (1e-7 + tp + fn)
        return 2 * p * r / (p + r + 1e-7)
    lab = torch.tensor([[1., 0.], [1., 1.], [0., 0.]])
    assert float(f1_score(lab, torch.zeros(3, 2))) == 0.0                                        # all negative
    np.testing.assert_allclose(float(f1_score(lab, torch.ones(3, 2))), want(3, 3, 0), rtol=1e-6)  # all positive
    pred = torch.tensor([[0.9, 0.6], [0.2, 0.5], [0.49, 0.1]])                                    # floor(p + 0.5): 0.5 rounds up
    np.testing.assert_allclose(float(f1_score(lab, pred)), want(2, 1, 1), rtol=1e-6)
    np.testing.assert_allclose(float(f1_score(lab, lab)), want(3, 0, 0), rtol=1e-6)


def _xent(x, z):
    return np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))


def test_supervise_model_against_float64(cpu_ops):
    class Model(SuperviseModel):
        def __init__(self):
            super().__init__('f1', 3, dim=6)
            self.encoder = SageEncoder([[0], [0]], [3, 2], 6, **KW)

        def embed(self, n_id):
            return self.encoder(n_id)

    with pytest.raises(ValueError, match="f1"):
        SuperviseModel('f1', 3, 'auc', dim=6)
    torch.manual_seed(0)
    model = Model()
    inputs = torch.as_tensor([3, 5, 11, 8, 2], dtype=torch.int64)
    emb, loss, name, metric = model(inputs)
    h = _sage_f64(model.encoder, model.encoder.sample(inputs))
    logit = h @ f64(model.out_fc.weight).T
    label = _dense_feature(inputs, ['f1'], [3])[0].double().numpy()
    assert name == 'f1' and model.out_fc.bias is None
    np.testing.assert_allclose(f64(emb), h, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(loss.item(), _xent(logit, label).mean(), rtol=1e-5)
    np.testing.assert_allclose(float(metric), float(f1_score(torch.as_tensor(label), torch.as_tensor(1 / (1 + np.exp(-logit))))), rtol=1e-6)
    loss.backward()
    assert all(p.grad is not None for p in model.parameters())


def test_dgi_against_float64(cpu_ops):
    torch.manual_seed(0)
    kw = {k: v for k, v in KW.items() if k != 'max_id'}
    model = DGI(0, [0], 12, [[0], [0]], [3, 2], 6, **kw)
    with pytest.raises(ValueError, match="metric"):
        DGI(0, [0], 12, [[0]], [3], 6, metric='f1')
    inputs = torch.as_tensor([3, 5, 11, 8, 2], dtype=torch.int64)
    emb, loss, name, metric = model(inputs, torch.Generator().manual_seed(2))
    enc = model._target_encoder
    samples = enc.sample(inputs.unsqueeze(-1))
    shuffled = enc.shuffle_samples(samples, torch.Generator().manual_seed(2))
    h, h_neg = _sage_f64(enc, samples), _sage_f64(enc, shuffled)
    read = 1 / (1 + np.exp(-h.mean(0)))                       # readout_func: the sigmoid of the batch's mean
    k = f64(model.kernel.kernel)
    lg, nlg = (h @ k) @ read, (h_neg @ k) @ read
    assert emb.shape == (5, 6) and name == 'mrr'
    np.testing.assert_allclose(f64(emb), h, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(loss.item(), np.concatenate([_xent(lg, 1), _xent(nlg, 0)]).mean(), rtol=1e-5)
    np.testing.assert_allclose(float(metric), np.mean(np.where(lg > nlg, 1.0, 0.5)), rtol=1e-6)
    loss.backward()
    assert all(p.grad is not None for p in model.parameters())
