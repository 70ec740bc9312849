"""CPU: the solution package (euler_b200/solution.py) on CPU stand-ins of the graph ops -- each logits class, loss and
GetLabelFromFea against float64 numpy restatements of tf_euler/python/solution, and both solutions' shapes, returned tuples
and refusals."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import ops, solution
from euler_b200.encoders import ShallowEncoder
from euler_b200.supervised import f1_score
from test_shallow_encoder_cpu import DENSE, _dense_feature, _row


def f64(t):
    return t.detach().double().numpy()


def _xent(x, z):
    """tf.nn.sigmoid_cross_entropy_with_logits: max(x, 0) - x z + log(1 + exp(-|x|))"""
    return np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))


def _sample_node(count, node_type, condition=''):
    """a deterministic stand-in: draw k is node (5 k + 3 type + 1) % 13"""
    t = int(np.asarray(node_type).reshape(-1)[0]) if not isinstance(node_type, str) else -1
    return (5 * torch.arange(count) + 3 * t + 1) % 13


def _sample_neighbor(nodes, edge_types, count, default_node=-1, condition=''):
    """a deterministic stand-in: neighbour k of node n is (3 n + k) % 13, or default_node where that is 12"""
    nb = (3 * torch.as_tensor(nodes).reshape(-1, 1) + torch.arange(count)[None, :]) % 13
    return torch.where(nb == 12, torch.full_like(nb, default_node), nb), None, None


@pytest.fixture
def cpu_ops(monkeypatch):
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    monkeypatch.setattr(ops, "sample_node", _sample_node)
    monkeypatch.setattr(ops, "sample_neighbor", _sample_neighbor)


# ---------------------------------------------------------------------------- logits, losses, labels
def test_dense_logits_against_float64():
    torch.manual_seed(0)
    logits = solution.DenseLogits(3, dim=5)
    assert logits.out_fc.bias is None and tuple(logits.out_fc.weight.shape) == (3, 5)
    assert (logits.out_fc.weight.abs() <= (6.0 / (5 + 3)) ** 0.5).all()          # glorot uniform bound
    x = torch.randn(4, 5)
    np.testing.assert_allclose(f64(logits(x)), f64(x) @ f64(logits.out_fc.weight).T, rtol=1e-6, atol=1e-6)


def test_pos_neg_and_cosine_logits_against_float64():
    torch.manual_seed(1)
    emb, pos, neg = torch.randn(4, 1, 6), torch.randn(4, 3, 6), torch.randn(4, 5, 6)
    logit, neg_logit = solution.PosNegLogits()(emb, pos, neg)
    np.testing.assert_allclose(f64(logit), np.einsum('bid,bjd->bij', f64(emb), f64(pos)), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(f64(neg_logit), np.einsum('bid,bjd->bij', f64(emb), f64(neg)), rtol=1e-5, atol=1e-6)

    def l2n(v):   # tf.nn.l2_normalize: v * rsqrt(max(sum(v * v), 1e-12))
        return v / np.sqrt(np.maximum((v * v).sum(-1, keepdims=True), 1e-12))

    x, y = torch.randn(7, 6), torch.randn(7, 6)
    x[2] = 0.0                                                                   # zero rows: l2_normalize keeps them zero
    y[5] = 0.0
    got = solution.CosineLogits()(x, y)
    want = 5.0 * (l2n(f64(x)) * l2n(f64(y))).sum(-1, keepdims=True)
    assert got.shape == (7, 1) and got[2].item() == 0.0 and got[5].item() == 0.0
    np.testing.assert_allclose(f64(got), want, rtol=1e-5, atol=1e-6)


def test_losses_against_float64():
    torch.manual_seed(2)
    labels, logits = (torch.rand(6, 3) > 0.5).float(), torch.randn(6, 3) * 4
    np.testing.assert_allclose(solution.sigmoid_loss(labels, logits).item(), _xent(f64(logits), f64(labels)).mean(), rtol=1e-6)
    pos, neg = torch.randn(4, 1, 2) * 3, torch.randn(4, 1, 5) * 3
    want = np.concatenate([_xent(f64(pos), 1.0).reshape(-1), _xent(f64(neg), 0.0).reshape(-1)]).mean()
    np.testing.assert_allclose(solution.xent_loss(pos, neg).item(), want, rtol=1e-6)
    empty = solution.xent_loss(pos, torch.zeros(4, 1, 0))                        # no negatives: the positives alone
    np.testing.assert_allclose(empty.item(), _xent(f64(pos), 1.0).mean(), rtol=1e-6)


def test_get_label_from_fea(cpu_ops):
    nodes = torch.as_tensor([5, 3, 99, 11])
    label = solution.GetLabelFromFea('f1', 3)(nodes)
    want = np.stack([DENSE['f1'][_row(n)] if _row(n) >= 0 else np.zeros(3, np.float32) for n in nodes.tolist()])
    np.testing.assert_array_equal(label.numpy(), want)


def test_acc_score():
    labels = torch.tensor([[1., 0.], [1., 1.], [0., 0.]])
    pred = torch.tensor([[0.9, 0.6], [0.2, 0.5], [0.49, 0.1]])                   # floor(p + 0.5): 0.5 rounds up
    assert solution.acc_score(labels, pred).item() == pytest.approx(4 / 6)
    assert solution.acc_score(labels, labels).item() == 1.0


# ---------------------------------------------------------------------------- the solutions
def _id_encoder(dim=6):
    return ShallowEncoder(max_id=12, embedding_dim=dim, fused=False)


@pytest.mark.parametrize("num_pos", (1, 3))
@pytest.mark.parametrize("num_negs", (0, 1, 5))
@pytest.mark.parametrize("metric", ('mrr', 'hit1', 'hit3', 'hit10', 'mr'))
def test_unsupervise_solution_shapes_and_tuple(cpu_ops, num_pos, num_negs, metric):
    torch.manual_seed(3)
    target, context = _id_encoder(), _id_encoder()
    sol = solution.UnsuperviseSolution(target, context, solution.SamplePosWithTypes([0], num_pos, max_id=11),
                                       solution.SampleNegWithTypes(0, num_negs), metric_name=metric)
    assert {id(p) for p in sol.parameters()} == {id(p) for p in list(target.parameters()) + list(context.parameters())}
    inputs = torch.as_tensor([3, 5, 8, 11, 2])
    src, pos, negs = sol.to_sample(inputs)
    assert src.shape == (5, 1) and pos.shape == (5, num_pos) and negs.shape == (5, num_negs)
    emb, loss, name, value = sol(inputs)
    assert emb.shape == (5, 1, 6) and loss.dim() == 0 and name == metric and value.dim() == 0
    # float64 restatement of base_unsupervise.__call__ on the stand-in's ids
    T, C = f64(target.embedding.embeddings), f64(context.embedding.embeddings)
    e, p, n = T[src.numpy()], C[pos.numpy()], C[negs.numpy()]
    logit, neg_logit = np.einsum('bid,bjd->bij', e, p), np.einsum('bid,bjd->bij', e, n)
    want = np.concatenate([_xent(logit, 1.0).reshape(-1), _xent(neg_logit, 0.0).reshape(-1)]).mean()
    np.testing.assert_allclose(loss.item(), want, rtol=1e-5)
    np.testing.assert_array_equal(f64(emb), T[inputs.numpy()][:, None])
    loss.backward()
    assert target.embedding.embeddings.grad is not None and context.embedding.embeddings.grad is not None


@pytest.mark.parametrize("metric", ('f1', 'acc'))
def test_supervise_solution_tuple_against_float64(cpu_ops, metric):
    torch.manual_seed(4)
    enc = ShallowEncoder(dim=6, feature_idx='f2', feature_dim=5, fused=False)
    sol = solution.SuperviseSolution(solution.GetLabelFromFea('f1', 3), enc, solution.DenseLogits(3, dim=6), metric_name=metric)
    inputs = torch.as_tensor([3, 5, 8, 11, 7])
    emb, loss, name, value = sol(inputs)
    assert emb.shape == (5, 6) and name == metric
    feat = _dense_feature(inputs, ['f2'], [5])[0].double().numpy()
    h = feat @ f64(enc.dense.kernel)
    logit = h @ f64(sol.logit_fn.out_fc.weight).T
    label = _dense_feature(inputs, ['f1'], [3])[0].double().numpy()
    np.testing.assert_allclose(f64(emb), h, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(loss.item(), _xent(logit, label).mean(), rtol=1e-5)
    fn = f1_score if metric == 'f1' else solution.acc_score
    np.testing.assert_allclose(value.item(), fn(torch.as_tensor(label), torch.sigmoid(torch.as_tensor(logit))).item(), rtol=1e-6)


def test_multi_type_negatives_are_refused(cpu_ops):
    negs = solution.SampleNegWithTypes([0, 1], 4)(torch.as_tensor([3, 5]))
    assert isinstance(negs, list) and len(negs) == 2 and all(n.shape == (2, 4) for n in negs)
    sol = solution.UnsuperviseSolution(_id_encoder(), _id_encoder(), solution.SamplePosWithTypes([0]),
                                       solution.SampleNegWithTypes([0, 1], 4))
    with pytest.raises(ValueError, match="list"):
        sol(torch.as_tensor([3, 5]))


def test_unknown_metrics_raise():
    enc = _id_encoder()
    for bad in ('precision', 'mrr'):
        with pytest.raises(ValueError, match="metric_name"):
            solution.SuperviseSolution(solution.GetLabelFromFea('f1', 3), enc, solution.DenseLogits(3, dim=6), metric_name=bad)
    for bad in ('precision', 'f1'):
        with pytest.raises(ValueError, match="metric_name"):
            solution.UnsuperviseSolution(enc, enc, solution.SamplePosWithTypes([0]), solution.SampleNegWithTypes(0),
                                         metric_name=bad)
    with pytest.raises(NotImplementedError, match="auc"):
        solution.SuperviseSolution(solution.GetLabelFromFea('f1', 3), enc, solution.DenseLogits(3, dim=6), metric_name='auc')
