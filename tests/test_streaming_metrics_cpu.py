"""CPU: the streaming metrics' numpy restatement (tests/metrics_reference.py) -- TF's literal [T, N] comparison against the
bucket-and-suffix-sum form, the threshold table, the double sigmoid, floor(p + 0.5) in float32, the AUC against sklearn --
and the streaming=True wiring of SuperviseModel, SuperviseSolution and the graph auto-encoders on CPU stand-ins, with the
metric ops patched to the restatement."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
import metrics_reference as ref
from euler_b200 import autoencoder as ae, metrics, ops, solution, supervised
from euler_b200.encoders import ShallowEncoder
from test_gae_cpu import TableEncoder, sampler  # noqa: F401  (fixture)
from test_shallow_encoder_cpu import _dense_feature

F32 = np.float32


# ---------------------------------------------------------------------------- the restatement
@pytest.mark.parametrize("T", [2, 3, 4, 200, 5000, 16384])
def test_threshold_table(T):
    t = ref.thresholds(T)
    assert t.dtype == F32 and t.size == T
    assert np.all(np.diff(t.astype(np.float64)) > 0)
    assert t[0] < 0 and t[-1] > 1
    assert t[0] == F32(-1e-7) and t[-1] == F32(1.0 + 1e-7)
    for i in (1, T // 2, T - 2):
        if 0 < i < T - 1:
            assert t[i] == F32(i / (T - 1))


def test_threshold_table_strictly_increasing_for_every_T():
    for T in list(range(2, 600)) + list(range(16000, 16385)):
        t = ref.thresholds(T)
        assert np.all(t[1:] > t[:-1]) and t[0] < F32(0) and t[-1] > F32(1), T


def _edge_predictions(T, rng):
    """every threshold in [0, 1] and its float32 neighbours, 0, -0, 1, subnormals and random values"""
    t = ref.thresholds(T)
    t = t[(t >= 0) & (t <= 1)]
    near = np.concatenate([t, np.nextafter(t, F32(-1)), np.nextafter(t, F32(2))])
    special = np.array([0.0, -0.0, 1.0, 1e-45, 1e-39, np.nextafter(F32(1), F32(0))], F32)
    p = np.concatenate([near, special, rng.rand(997).astype(F32)]).astype(F32)
    return p[(p >= 0) & (p <= 1)]


def _labels(n, rng):
    return rng.choice(np.array([0, 1, 2, -1, 0.5, np.nan, -0.0], F32), size=n)


@pytest.mark.parametrize("T", [2, 3, 200, 5000])
def test_literal_comparison_equals_bucket_counts(T):
    rng = np.random.RandomState(T)
    p = _edge_predictions(T, rng)
    lab = _labels(p.size, rng)
    np.testing.assert_array_equal(ref.literal_counts(lab, p, T), ref.bucket_counts(lab, p, T))
    for n in (0, 1, 31):
        np.testing.assert_array_equal(ref.literal_counts(lab[:n], p[:n], T), ref.bucket_counts(lab[:n], p[:n], T))


def test_label_casts():
    # nonzero is positive, NaN included; -0.0 is negative
    c = ref.literal_counts(np.array([0, -0.0, 1, 2, -1, 0.5, np.nan], F32), np.full(7, 0.6, F32), 3)
    assert c[0][0] == 5 and c[3][0] == 2


def test_streaming_auc_refuses_and_recovers():
    a = ref.Auc(200)
    v1 = a.update([1, 0, 1], [0.9, 0.2, 0.4])
    s1 = a.state.copy()
    assert np.isfinite(v1)
    assert np.isnan(a.update([1, 0], [0.5, 1.5]))
    assert np.isnan(a.update([1, 0], [np.nan, 0.5]))
    np.testing.assert_array_equal(a.state, s1)
    assert a.refused == 2
    a.update([0], [0.1])      # counted, but the value stays NaN until a reset
    assert np.isnan(a.value()) and a.state[2].sum() > s1[2].sum()


def test_auc_against_sklearn():
    from sklearn.metrics import roc_auc_score
    rng = np.random.RandomState(7)
    T = 200
    t = ref.thresholds(T).astype(np.float64)
    for _ in range(5):
        b = rng.randint(1, T - 1, size=2000)
        p = ((t[b - 1] + t[b]) / 2).clip(0, 1).astype(F32)           # strictly between two thresholds
        lab = (rng.rand(2000) < np.clip(p, 0.05, 0.95)).astype(F32)
        a = ref.Auc(T)
        v = a.update(lab, p)
        assert abs(float(v) - roc_auc_score(lab, p)) < 1e-5
        assert abs(float(v) - ref.auc_value_f64(*a.state)) < 1e-6


def test_double_sigmoid():
    # the models pass sigmoid(logit) and auc_score applies sigmoid again: every prediction lands in [0.5, 0.7311]
    x = torch.tensor([-1e30, -100.0, -1.0, 0.0, 1.0, 100.0, 1e30, float('-inf'), float('inf')])
    p = torch.sigmoid(torch.sigmoid(x))
    assert float(p.min()) >= 0.5 and float(p.max()) <= 0.7311
    assert float(p[0]) == 0.5 and float(p[-1]) == float(torch.sigmoid(torch.tensor(1.0)))


def test_streaming_auc_applies_sigmoid(monkeypatch):
    seen = []
    monkeypatch.setattr(ops, "metric_auc_update", lambda labels, predictions, *state: seen.append(predictions.clone()))
    m = metrics.StreamingAuc(200)
    x = torch.tensor([-3.0, 0.0, 2.0])
    m(torch.ones(3), x)
    torch.testing.assert_close(seen[0], torch.sigmoid(x), rtol=0, atol=0)


def test_floor_half_edges():
    p = np.array([0.49999997, 0.5, -0.5, 0.49999994, 1.5, -0.50000006, np.nan], F32)
    np.testing.assert_array_equal(ref.rounded(p)[:6], np.array([1, 1, 0, 0, 2, -1], F32))
    assert np.isnan(ref.rounded(p)[6])
    torch.testing.assert_close(torch.floor(torch.from_numpy(p) + 0.5), torch.from_numpy(ref.rounded(p)), equal_nan=True)
    f1 = ref.F1()
    f1.update(np.array([1, 0, 0], F32), np.array([0.49999997, np.nan, 0.2], F32))   # NaN predicts positive
    np.testing.assert_array_equal(f1.state, np.array([1, 0, 1], F32))
    acc = ref.Accuracy()
    assert acc.value() == 0
    acc.update(np.array([1, 0, 0], F32), np.array([0.49999997, np.nan, 0.2], F32))  # NaN is never correct
    np.testing.assert_array_equal(acc.state, np.array([2, 3], F32))


def test_f1_matches_the_batch_form_on_one_batch():
    rng = np.random.RandomState(3)
    lab, pred = (rng.rand(300) < 0.4).astype(F32), rng.rand(300).astype(F32)
    f1 = ref.F1()
    v = f1.update(lab, pred)
    assert v == supervised.f1_score(torch.from_numpy(lab), torch.from_numpy(pred)).item()


# ---------------------------------------------------------------------------- the wiring, on the restatement
class _Patched(object):
    """ops.metric_* restated on CPU tensors, in place, recording every call"""

    def __init__(self):
        self.calls = []

    def auc(self, labels, predictions, tp, fn, tn, fp, refused, value):
        self.calls.append(('auc', labels.clone(), predictions.clone()))
        T = tp.numel()
        r = ref.Auc(T)
        r.state = np.stack([t.numpy() for t in (tp, fn, tn, fp)])
        r.refused = int(refused)
        v = r.update(labels.numpy(), predictions.numpy())
        for t, s in zip((tp, fn, tn, fp), r.state):
            t.copy_(torch.from_numpy(s))
        refused.fill_(r.refused)
        value.fill_(float(v))
        return value

    def count(self, kind, state, value, labels=None, predictions=None, correct=None, total=None):
        self.calls.append((kind, None if labels is None else labels.clone(),
                           None if predictions is None else predictions.clone(), correct, total))
        r = ref.F1() if kind == 'f1' else ref.Accuracy()
        r.state = state.numpy().copy()
        v = r.add_counts(int(correct), total) if correct is not None else r.update(labels.numpy(), predictions.numpy())
        state.copy_(torch.from_numpy(r.state))
        value.fill_(float(v))
        return value


@pytest.fixture
def patched(monkeypatch):
    p = _Patched()
    monkeypatch.setattr(ops, "metric_auc_update", p.auc)
    monkeypatch.setattr(ops, "metric_count_update", p.count)
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    return p


class _Model(supervised.SuperviseModel):
    def __init__(self, metric_name, streaming):
        super().__init__('f1', 3, metric_name, dim=5, streaming=streaming)
        self.enc = ShallowEncoder(dim=5, feature_idx='f2', feature_dim=5, fused=False)

    def embed(self, n_id):
        return self.enc(n_id)


BATCHES = [torch.as_tensor([3, 5, 8, 11, 7]), torch.as_tensor([5, 5, 2]), torch.as_tensor([8, 3, 3, 11])]


def _restate(name, calls):
    """the restatement fed the labels and predictions the metric received, batch after batch: (values, final state)"""
    r = {'auc': lambda: ref.Auc(5000), 'f1': ref.F1, 'acc': ref.Accuracy}[name]()
    vals = []
    for c in calls:
        if c[0] == 'acc' and c[3] is not None:
            vals.append(r.add_counts(int(c[3]), c[4]))
        else:
            vals.append(r.update(c[1].numpy(), c[2].numpy()))
    return vals, r


def _states(m):
    return [b.clone() for b in m.buffers()]


@pytest.mark.parametrize("metric", ['f1', 'acc', 'auc'])
def test_supervise_model_streaming(patched, metric):
    torch.manual_seed(0)
    plain = _Model('f1', False)
    model = _Model(metric, True)
    assert set(model.state_dict()) == set(plain.state_dict())
    assert isinstance(model.metric, metrics.METRICS[metric])
    values = [model(b)[3] for b in BATCHES]
    assert len(patched.calls) == 3
    if metric == 'auc':   # sigmoid(sigmoid(logit))
        logit = model.out_fc(model.embed(BATCHES[2]))
        torch.testing.assert_close(patched.calls[2][2], torch.sigmoid(torch.sigmoid(logit.detach())))
    want, r = _restate(metric, patched.calls)
    np.testing.assert_array_equal(np.array([v.item() for v in values], F32), np.array(want, F32))
    assert model.metric.result().item() == values[-1].item()
    model.metric.reset()
    assert all(float(b.abs().sum()) == 0 for b in model.metric.buffers())
    assert model.metric.result().item() == 0.0


def test_supervise_model_refusals_unchanged():
    with pytest.raises(ValueError, match="f1"):
        _Model('auc', False)
    with pytest.raises(ValueError, match="metric_name"):
        _Model('mrr', True)


@pytest.mark.parametrize("metric", ['f1', 'acc', 'auc'])
def test_supervise_solution_streaming(patched, metric):
    torch.manual_seed(4)
    enc = ShallowEncoder(dim=6, feature_idx='f2', feature_dim=5, fused=False)
    plain = solution.SuperviseSolution(solution.GetLabelFromFea('f1', 3), enc, solution.DenseLogits(3, dim=6))
    sol = solution.SuperviseSolution(solution.GetLabelFromFea('f1', 3), enc, solution.DenseLogits(3, dim=6),
                                     metric_name=metric, streaming=True)
    assert set(sol.state_dict()) == set(plain.state_dict())
    values = []
    for b in BATCHES:
        emb, loss, name, v = sol(b)
        assert name == metric
        values.append(v.item())
    want, _ = _restate(metric, patched.calls)
    np.testing.assert_array_equal(np.array(values, F32), np.array(want, F32))
    sol.metric.reset()
    assert sol.metric.result().item() == 0.0
    with pytest.raises(NotImplementedError, match="auc"):
        solution.SuperviseSolution(solution.GetLabelFromFea('f1', 3), enc, solution.DenseLogits(3, dim=6), metric_name='auc')


@pytest.mark.parametrize("variational", [False, True])
def test_autoencoder_streaming_composed(patched, sampler, variational):
    """fused=False on the CPU: the streaming accuracy is fed the composed labels and predictions"""
    log = []
    enc = TableEncoder(1, log)
    kw = dict(node_type=0, edge_type=[0], max_id=40, num_negs=3, fused=False)
    if variational:
        model = ae.VariationalGraphAutoEncoder(1.0, enc, generator=torch.Generator().manual_seed(2), streaming=True, **kw)
        plain = ae.VariationalGraphAutoEncoder(1.0, TableEncoder(1, []), **kw)
    else:
        model = ae.GraphAutoEncoder(enc, streaming=True, **kw)
        plain = ae.GraphAutoEncoder(TableEncoder(1, []), **kw)
    assert set(model.state_dict()) == set(plain.state_dict())
    values = []
    for b in BATCHES:
        emb, loss, name, acc = model(b)
        assert name == 'acc'
        values.append(acc.item())
    assert [c[0] for c in patched.calls] == ['acc'] * 3
    assert [c[1].numel() for c in patched.calls] == [2 * 3 * b.numel() for b in BATCHES]
    want, r = _restate('acc', patched.calls)
    np.testing.assert_array_equal(np.array(values, F32), np.array(want, F32))
    np.testing.assert_array_equal(model.metric.state.numpy(), r.state)
    model.metric.reset()
    assert model.metric.result().item() == 0.0


def test_autoencoder_streaming_fused_counts(patched, monkeypatch):
    """the fused path adds gae_loss's correct count of 2BK predictions, with no labels or predictions"""
    model = ae.GraphAutoEncoder(TableEncoder(1, []), 0, [0], 40, num_negs=3, streaming=True)
    counts = iter([torch.tensor(7), torch.tensor(2), torch.tensor(11)])
    monkeypatch.setattr(ops, "gae_loss", lambda e, p, n: (torch.zeros(()), next(counts)))
    vals = [model.loss_and_acc(None, torch.zeros(b.numel(), 3, 6), None)[1].item() for b in BATCHES]
    assert [(c[0], c[3].item(), c[4]) for c in patched.calls] == [('acc', 7, 30), ('acc', 2, 18), ('acc', 11, 24)]
    assert vals[-1] == F32(20) / F32(72) and model.metric.state.tolist() == [20.0, 72.0]


def test_metrics_get():
    assert isinstance(metrics.get('auc'), metrics.StreamingAuc) and metrics.get('auc').num_thresholds == 5000
    assert isinstance(metrics.get('f1'), metrics.StreamingF1) and isinstance(metrics.get('acc'), metrics.StreamingAccuracy)
    assert metrics.get('f1') is not metrics.get('f1')
    with pytest.raises(ValueError):
        metrics.get('mrr')
    for bad in (1, 16385):
        with pytest.raises(ValueError):
            metrics.StreamingAuc(bad)
    m = metrics.StreamingAuc(7)
    assert m.state_dict() == {} and [b.shape for b in m.buffers()][:4] == [(7,)] * 4
