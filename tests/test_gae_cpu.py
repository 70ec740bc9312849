"""CPU: the graph auto-encoders (euler_b200/autoencoder.py) with fused=False over a CPU stand-in encoder and mocked sampling
ops, against a float64 numpy restatement of tf_euler's base_gae.py (GAE) and examples/gae/gae.py (VGAE): loss, acc and every
gradient, the order of the sampling ops and encoder calls, and the constructors' and gae_loss's refusals."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import EulerError, autoencoder as ae, ops

MAX_ID = 40
DIM = 6


class TableEncoder(torch.nn.Module):
    """a stand-in node encoder: rows of a table f32[MAX_ID + 2, DIM], each call's ids recorded in log"""

    def __init__(self, seed, log):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.table = torch.nn.Parameter(torch.randn(MAX_ID + 2, DIM, generator=g) * 0.5)
        self.dims = [DIM]
        self.log = log

    def forward(self, ids):
        self.log.append(('encoder', ids.clone()))
        return self.table[ids]


@pytest.fixture
def sampler(monkeypatch):
    """sample_neighbor and sample_node drawn from a numpy stream, each call recorded"""
    log = []
    rs = np.random.RandomState(5)

    def sample_neighbor(inputs, edge_type, count, default_node=-1):
        log.append(('neighbor', inputs.clone(), edge_type, count, default_node))
        ids = torch.as_tensor(rs.randint(0, MAX_ID + 2, size=(inputs.numel(), count)), dtype=torch.int64)
        return ids, torch.ones(ids.shape), torch.zeros(ids.shape, dtype=torch.int32)

    def sample_node(count, node_type):
        log.append(('node', count, node_type))
        return torch.as_tensor(rs.randint(0, MAX_ID + 1, size=count), dtype=torch.int64)

    monkeypatch.setattr(ops, 'sample_neighbor', sample_neighbor)
    monkeypatch.setattr(ops, 'sample_node', sample_node)
    return log


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _restated(ids, mu_t, lv_t=None, noise=None, radius=0.0):
    """the loss, acc and table gradients of one step in float64: ids = (src [B, 1], pos [B, K], negs [B, K]); mu_t and lv_t
    the tables; noise the three sets' draws (None: emb = mu)"""
    mus = [mu_t[i] for i in ids]
    zs = list(mus)
    if lv_t is not None and noise is not None:
        zs = [m + radius * n * np.sqrt(np.exp(lv_t[i])) for m, n, i in zip(mus, noise, ids)]
    e, p, n = zs
    logits = np.einsum('bod,bkd->bok', e, p)
    neg_logits = np.einsum('bod,bkd->bok', e, n)
    x = np.concatenate([logits.reshape(-1), neg_logits.reshape(-1)])
    z = np.concatenate([np.ones(logits.size), np.zeros(neg_logits.size)])
    loss = np.mean(np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x))))
    acc = np.mean(np.floor(np.concatenate([_sigmoid(logits), _sigmoid(neg_logits)], 2) + 0.5)
                  == np.concatenate([np.ones_like(logits), np.zeros_like(neg_logits)], 2))
    N = x.size
    c_pos, c_neg = (_sigmoid(logits) - 1) / N, _sigmoid(neg_logits) / N          # [B, 1, K]
    dz = [np.einsum('bok,bkd->bod', c_pos, p) + np.einsum('bok,bkd->bod', c_neg, n),
          np.einsum('bok,bod->bkd', c_pos, e), np.einsum('bok,bod->bkd', c_neg, e)]
    g_mu = np.zeros_like(mu_t)
    g_lv = None
    if lv_t is None:
        for i, d in zip(ids, dz):
            np.add.at(g_mu, i, d)
        return loss, acc, g_mu, g_lv
    lvs = [lv_t[i] for i in ids]
    kls = np.concatenate([(-0.5 * (lv - np.exp(lv) - m ** 2 + 1)).reshape(-1) for m, lv in zip(mus, lvs)])
    loss += kls.mean()
    Nk = kls.size
    g_lv = np.zeros_like(lv_t)
    for k, (i, d, m, lv) in enumerate(zip(ids, dz, mus, lvs)):
        np.add.at(g_mu, i, d + m / Nk)
        dzdl = radius * noise[k] * 0.5 * np.sqrt(np.exp(lv)) if noise is not None else 0.0
        np.add.at(g_lv, i, d * dzdl + 0.5 * (np.exp(lv) - 1) / Nk)
    return loss, acc, g_mu, g_lv


def _close(got, want, tol=1e-5):
    got = got.detach().double().numpy() if torch.is_tensor(got) else np.asarray(got, dtype=np.float64)
    scale = max(np.abs(want).max(), 1e-30) if np.size(want) else 1.0
    assert np.abs(got - want).max() <= tol * scale, np.abs(got - want).max() / scale


def _sampled(log):
    """the ids of each encoder call, in order: src, pos, negs, inputs"""
    return [e[1] for e in log if e[0] == 'encoder']


@pytest.mark.parametrize('K', [1, 5, 10])
@pytest.mark.parametrize('B', [1, 7])
def test_gae_matches_restatement(sampler, B, K):
    enc = TableEncoder(1, sampler)
    model = ae.GraphAutoEncoder(enc, node_type=0, edge_type=[0], max_id=MAX_ID, num_negs=K, fused=False)
    inputs = torch.arange(B, dtype=torch.int64) * 3 % (MAX_ID + 1)
    embedding, loss, name, acc = model(inputs)
    assert name == 'acc' and embedding.shape == (B, 1, DIM)
    loss.backward()
    src, pos, negs, last = _sampled(sampler)
    assert torch.equal(last, inputs)
    ids = (src.numpy().reshape(B, 1), pos.numpy().reshape(B, K), negs.numpy().reshape(B, K))
    w, w_acc, g_mu, _ = _restated(ids, enc.table.detach().double().numpy())
    _close(loss, w)
    assert float(acc) == pytest.approx(w_acc, abs=1e-7)
    _close(enc.table.grad, g_mu)
    _close(embedding.reshape(B, DIM), enc.table.detach().double().numpy()[inputs.numpy()], 0)


def _vgae(sampler, K, radius, train):
    enc = TableEncoder(2, sampler)
    gen = torch.Generator().manual_seed(11)
    model = ae.VariationalGraphAutoEncoder(radius, enc, node_type=0, edge_type=[0], max_id=MAX_ID, num_negs=K, train=train,
                                           generator=gen, fused=False)
    with torch.no_grad():
        lv = model.log_var_encoder.embedding.embeddings
        lv.copy_(torch.randn(lv.shape, generator=torch.Generator().manual_seed(3)) * 0.3)
    return enc, model


@pytest.mark.parametrize('radius', [0.0, 1.0])
@pytest.mark.parametrize('K', [1, 5, 10])
@pytest.mark.parametrize('B', [1, 7])
def test_vgae_matches_restatement(sampler, B, K, radius):
    enc, model = _vgae(sampler, K, radius, True)
    inputs = torch.arange(B, dtype=torch.int64) * 5 % (MAX_ID + 1)
    embedding, loss, _, acc = model(inputs)
    loss.backward()
    src, pos, negs, _ = _sampled(sampler)
    ids = (src.numpy().reshape(B, 1), pos.numpy().reshape(B, K), negs.numpy().reshape(B, K))
    replay = torch.Generator().manual_seed(11)     # the model's draws, in its order: src, pos, negs
    noise = [torch.randn((B, n, DIM), generator=replay).double().numpy() for n in (1, K, K)]
    lv_t = model.log_var_encoder.embedding.embeddings
    w, w_acc, g_mu, g_lv = _restated(ids, enc.table.detach().double().numpy(), lv_t.detach().double().numpy(), noise, radius)
    _close(loss, w)
    assert float(acc) == pytest.approx(w_acc, abs=1e-7)
    _close(enc.table.grad, g_mu)
    _close(lv_t.grad, g_lv)
    _close(embedding.reshape(B, DIM), enc.table.detach().double().numpy()[inputs.numpy()], 0)   # the mu rows


@pytest.mark.parametrize('K', [1, 5])
def test_vgae_eval_uses_mu(sampler, K):
    B = 7
    enc, model = _vgae(sampler, K, 1.0, False)
    inputs = torch.arange(B, dtype=torch.int64)
    embedding, loss, _, acc = model(inputs)
    loss.backward()
    src, pos, negs, _ = _sampled(sampler)
    ids = (src.numpy().reshape(B, 1), pos.numpy().reshape(B, K), negs.numpy().reshape(B, K))
    lv_t = model.log_var_encoder.embedding.embeddings
    w, w_acc, g_mu, g_lv = _restated(ids, enc.table.detach().double().numpy(), lv_t.detach().double().numpy(), None, 1.0)
    _close(loss, w)
    assert float(acc) == pytest.approx(w_acc, abs=1e-7)
    _close(enc.table.grad, g_mu)
    _close(lv_t.grad, g_lv)
    assert model.generator.initial_seed() == 11 and torch.equal(
        torch.randn(3, generator=model.generator), torch.randn(3, generator=torch.Generator().manual_seed(11)))   # no draws


@pytest.mark.parametrize('variational', [False, True])
def test_call_order(sampler, variational):
    B, K = 4, 3
    enc = TableEncoder(3, sampler)
    if variational:
        model = ae.VariationalGraphAutoEncoder(0.5, enc, node_type=2, edge_type=[1], max_id=MAX_ID, num_negs=K, fused=False)
    else:
        model = ae.GraphAutoEncoder(enc, node_type=2, edge_type=[1], max_id=MAX_ID, num_negs=K, fused=False)
    inputs = torch.tensor([3, 1, 4, 1], dtype=torch.int64)
    model(inputs)
    kinds = [e[0] for e in sampler]
    assert kinds == ['neighbor', 'node', 'encoder', 'encoder', 'encoder', 'encoder']
    _, nb_inputs, edge_type, count, default_node = sampler[0]
    assert torch.equal(nb_inputs, inputs) and edge_type == [1] and count == K and default_node == MAX_ID + 1
    assert sampler[1][1:] == (B * K, 2)
    calls = [e[1] for e in sampler[2:]]
    assert torch.equal(calls[0], inputs) and torch.equal(calls[3], inputs)
    assert [c.numel() for c in calls] == [B, B * K, B * K, B]


def test_constructor_errors():
    enc = TableEncoder(4, [])
    with pytest.raises(ValueError):
        ae.GraphAutoEncoder(enc, 0, [0], MAX_ID, num_negs=0)
    with pytest.raises(ValueError):
        ae.GraphAutoEncoder(None, 0, [0], MAX_ID)
    with pytest.raises(ValueError):
        ae.VariationalGraphAutoEncoder(float('nan'), enc, 0, [0], MAX_ID, fused=False)
    with pytest.raises(ValueError):
        ae.VariationalGraphAutoEncoder(1.0, lambda ids: ids, 0, [0], MAX_ID, fused=False)   # no row width to read
    m = ae.VariationalGraphAutoEncoder(1.0, lambda ids: ids, 0, [0], MAX_ID, fused=False, dim=5)
    assert m.dim == 5 and m.log_var_encoder.output_dim == 5
    assert ae.GraphAutoEncoder(enc, 0, [0], MAX_ID).num_negs == 5
    assert ae.BaseGraphAutoEncoder(0, [0], MAX_ID).num_negs == 20


def test_gae_loss_refusals_before_the_device():
    e, p = torch.zeros(3, 4), torch.zeros(3, 2, 4)
    for args, kw in [((e, p, torch.zeros(3, 3, 4)), {}), ((e, torch.zeros(3, 0, 4), torch.zeros(3, 0, 4)), {}),
                     ((torch.zeros(2, 4), p, p), {}), ((e, p, p), {'radius': float('inf')}),
                     ((e, p, p), {'noise': (e, p, p)}), ((e, p, p), {'log_var': (e, p)}),
                     ((e, p, p), {'log_var': (e, p, torch.zeros(3, 2, 5))}), ((e.double(), p, p), {})]:
        with pytest.raises(EulerError):
            ops.gae_loss(*args, **kw)
