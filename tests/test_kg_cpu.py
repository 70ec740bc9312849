"""CPU: the torch composition of the knowledge-graph models (knowledge.composed_kg_loss) against a float64 numpy restatement of
upstream's code, the rank's closed form, the hinge and l2_normalize subgradients, TransR's reshape decision and the
constructors' errors."""
import numpy as np
import pytest
import torch

from euler_b200 import knowledge as kn

MODELS = ('transe', 'transh', 'transr', 'transd', 'distmult')


def _n(x):
    return x / np.sqrt(np.maximum((x * x).sum(-1, keepdims=True), 1e-12))


def _numpy_model(model, tabs, src, dst, neg, rel, l1, corrupt, margin):
    """upstream's generate_embedding, calculate_energy and loss_fn in float64 numpy, tile for tile"""
    B, K = neg.shape
    E, R = tabs[0], tabs[1]
    ed, rd = E.shape[1], R.shape[1]
    s, d, ng, r = E[src][:, None], E[dst][:, None], E[neg], R[rel][:, None]
    if model in ('transe', 'distmult'):
        s, d, ng = _n(s), _n(d), _n(ng)
    elif model == 'transh':
        h = tabs[2][rel][:, None]
        hx = np.tile(h, (1, K, 1))
        proj = lambda e, hh: e - (e * _n(hh)).sum(-1, keepdims=True) * _n(hh)   # noqa: E731
        s, d, ng = proj(s, h), proj(d, h), proj(ng, hx)
    elif model == 'transr':
        M = tabs[2][rel].reshape(-1, ed, rd)
        Mx = np.tile(M.reshape(-1, 1, ed * rd), (1, K, 1)).reshape(-1, ed, rd)
        s, d = _n(np.einsum('bi,bij->bj', s[:, 0], M))[:, None], _n(np.einsum('bi,bij->bj', d[:, 0], M))[:, None]
        ng = _n(np.einsum('bi,bij->bj', ng.reshape(-1, ed), Mx)).reshape(B, K, rd)
    else:
        et, rt = tabs[2], tabs[3][rel][:, None]
        proj = lambda e, t, q: _n(e + (e * t).sum(-1, keepdims=True) * q)   # noqa: E731
        s, d = proj(s, et[src][:, None], rt), proj(d, et[dst][:, None], rt)
        ng = proj(ng, et[neg], np.tile(rt, (1, K, 1)))
    r = _n(r)
    if model == 'distmult':
        score = lambda a, q, c: (a * (q * c)).sum(-1)   # noqa: E731
    else:
        score = lambda a, q, c: -(np.abs(a + q - c).sum(-1) if l1 else np.sqrt(((a + q - c) ** 2).sum(-1)))   # noqa: E731
    sx, rx, dx = np.tile(s, (1, K, 1)), np.tile(r, (1, K, 1)), np.tile(d, (1, K, 1))
    pos = score(s, r, d).reshape(B)
    front, tail = score(ng, rx, dx), score(sx, rx, ng)
    negs = {'front': front, 'tail': tail, 'both': np.concatenate([front, tail], -1)}[corrupt]
    loss = np.maximum(margin + negs.mean(-1) - pos, 0).mean()
    return pos, negs, loss


@pytest.mark.parametrize("corrupt", ('front', 'tail', 'both'))
@pytest.mark.parametrize("l1", (True, False))
@pytest.mark.parametrize("model", MODELS)
def test_composed_against_numpy(model, l1, corrupt):
    rng = np.random.RandomState(MODELS.index(model) * 7 + l1)
    ed, rd = (6, 4) if model == 'transr' else (5, 5)
    n_ent, n_rel, B, K = 30, 5, 9, 4
    tabs = [rng.randn(n_ent, ed), rng.randn(n_rel, rd)]
    tabs += {'transh': [rng.randn(n_rel, ed)], 'transr': [rng.randn(n_rel, ed * rd)],
             'transd': [rng.randn(n_ent, ed), rng.randn(n_rel, rd)]}.get(model, [])
    src, dst, rel = rng.randint(0, n_ent, B), rng.randint(0, n_ent, B), rng.randint(0, n_rel, B)
    neg = rng.randint(0, n_ent, (B, K))
    pos, negs, loss = _numpy_model(model, tabs, src, dst, neg, rel, l1, corrupt, 1.5)
    T = lambda a: torch.as_tensor(a)   # noqa: E731
    p, q, _ = kn.composed_kg_scores(model, [T(t) for t in tabs], T(src), T(dst), T(neg), T(rel), l1=l1, corrupt=corrupt)
    np.testing.assert_allclose(p.reshape(-1).numpy(), pos, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(q.reshape(B, -1).numpy(), negs, rtol=1e-12, atol=1e-12)
    got, _, _ = kn.composed_kg_loss(model, [T(t) for t in tabs], T(src), T(dst), T(neg), T(rel), l1=l1, corrupt=corrupt, margin=1.5)
    assert abs(float(got) - loss) <= 1e-12 * max(1.0, abs(loss))


def test_rank_closed_form_is_stable_top_k_with_ties():
    """#{j : neg_j >= pos} is the position of the last entry of concat([neg, pos]) under a stable descending sort, for 2K + 1
    entries with many ties"""
    rng = np.random.RandomState(0)
    for K in (1, 2, 5, 17):
        neg = rng.randint(-3, 4, size=(200, 1, 2 * K)).astype(np.float32)
        pos = rng.randint(-3, 4, size=(200, 1, 1)).astype(np.float32)
        allv = np.concatenate([neg, pos], 2)[:, 0]
        literal = np.array([list(np.argsort(-row, kind='stable')).index(2 * K) for row in allv])
        closed = (neg[:, 0] >= pos[:, 0]).sum(1)
        assert np.array_equal(literal, closed)
        mr = kn.composed_metric(torch.as_tensor(pos), torch.as_tensor(neg), 'mr')
        assert int(mr) == int(literal.sum()) // len(literal)


def test_hinge_subgradient_at_zero_is_taken():
    """TF's maximum(x, 0) sends the gradient to x on equality: a row whose hinge argument is exactly 0 is active"""
    x = torch.tensor([0.0, -1.0, 2.0], dtype=torch.float64, requires_grad=True)
    torch.clamp(x, min=0).sum().backward()
    assert x.grad.tolist() == [1.0, 0.0, 1.0]


def test_l2_normalize_gradient_below_eps():
    """below 1e-12 the maximum passes no gradient to sum x^2: the gradient is rsqrt(1e-12) times the upstream one"""
    x = torch.tensor([[1e-7, -2e-7]], dtype=torch.float64, requires_grad=True)
    g = torch.tensor([[0.3, 0.7]], dtype=torch.float64)
    (kn.l2_normalize(x) * g).sum().backward()
    np.testing.assert_allclose(x.grad.numpy(), g.numpy() * 1e6, rtol=1e-12)
    y = torch.tensor([[3.0, 4.0]], dtype=torch.float64, requires_grad=True)
    (kn.l2_normalize(y) * g).sum().backward()
    yn = np.array([0.6, 0.8])
    want = (g.numpy()[0] - (yn @ g.numpy()[0]) * yn) / 5.0
    np.testing.assert_allclose(y.grad.numpy()[0], want, rtol=1e-12)


def test_transr_relation_reshape_decision():
    """upstream's norm_emb reshapes the relation rows [B, 1, rel_dim] to [-1, ent_dim]: with equal dims that is the per-row
    normalisation used here; with unequal dims it normalises chunks that span triples, which differs"""
    rng = np.random.RandomState(1)
    B = 6
    for ed, rd, same in ((4, 4, True), (4, 6, False)):
        r = rng.randn(B, 1, rd)
        literal = _n(r.reshape(-1, ed)).reshape(B, 1, rd)
        ours = kn.l2_normalize(torch.as_tensor(r)).numpy()
        assert np.allclose(literal, ours) == same


def test_constructor_errors():
    with pytest.raises(ValueError):
        kn.TransE(0, 0, 10, 3, 8, 6)
    with pytest.raises(ValueError):
        kn.TransH(0, 0, 10, 3, 8, 6)
    with pytest.raises(ValueError):
        kn.TransD(0, 0, 10, 3, 8, 6)
    with pytest.raises(ValueError):
        kn.TransE(0, 0, 10, 3, 8, 8, metric_name='hit3')
    for name in ('acc', 'auc', 'f1'):
        with pytest.raises(ValueError):
            kn.DistMult(0, 0, 10, 3, 8, 8, metric_name=name)
    with pytest.raises(ValueError):
        kn.DistMult(0, 0, 10, 3, 8, 8, l2_regular=True, sparse_grad=True)
    m = kn.TransR(0, 0, 10, 3, 8, 6)
    assert m.entity_encoder.embeddings.shape == (12, 8) and m.transfer_matrix.embeddings.shape == (5, 48)
    assert kn.DistMult(0, 0, 10, 3, 8, 8, metric_name='hit3').metric_name == 'hit3'


def test_kg_fixture_shape_on_the_host():
    """tests/golden/kg_euler (make_kg_json.py through the reference's converter): 58 entities, 300 triples, three node and
    three edge types (train, test, valid), as the loader parses it without a device"""
    import ctypes as C
    import os
    from euler_b200 import _lib
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kg_euler")
    nn, ne, T, NT = C.c_int64(0), C.c_int64(0), C.c_int32(0), C.c_int32(0)
    assert _lib.load().eu_graph_load_inspect(path.encode(), 0, 1, C.byref(nn), C.byref(ne), C.byref(T), C.byref(NT), 0, None,
                                             None) == 0
    assert (nn.value, ne.value, T.value, NT.value) == (58, 300, 3, 3)
