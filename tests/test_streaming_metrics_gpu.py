"""GPU: the streaming metrics on the device (ops.metric_auc_update, ops.metric_count_update, euler_b200/metrics.py) bit for
bit against the numpy float32 restatement of TF 1.x tf.metrics (tests/metrics_reference.py) over consecutive batches, at the
threshold edges and special values; refusals, determinism, CUDA-graph replay, and a supervised and a GAE training step with
streaming=True."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
import metrics_reference as ref

pytestmark = pytest.mark.gpu
F32 = np.float32


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


def _edge_predictions(T):
    """every threshold in [0, 1] and its float32 neighbours on both sides, 0, -0, 1 and subnormals"""
    t = ref.thresholds(T)
    near = np.concatenate([t, np.nextafter(t, F32(-1)), np.nextafter(t, F32(2))])
    special = np.array([0.0, -0.0, 1.0, 1e-45, 1e-40, 1.1754942e-38, np.nextafter(F32(1), F32(0))], F32)
    p = np.concatenate([near, special]).astype(F32)
    return p[(p >= 0) & (p <= 1)]


LABEL_VALUES = np.array([0, 1, 2, -1, 0.5, np.nan, -0.0], F32)


def _batches(T, rng):
    """(labels, predictions) numpy batches: the edge values, then N in {0, 1, 31, 1000, 2^20 + 7} of random predictions, some
    of them in the double sigmoid's range [0.5, 0.7311]"""
    out = []
    p = _edge_predictions(T)
    out.append((rng.choice(LABEL_VALUES, size=p.size), p))
    for n in (0, 1, 31, 1000, (1 << 20) + 7):
        p = rng.rand(n).astype(F32)
        if n > 31:
            p[::2] = (0.5 + 0.2311 * rng.rand(p[::2].size)).astype(F32)
        lab = rng.choice(LABEL_VALUES, size=n) if n <= 1000 else (rng.rand(n) < p).astype(F32)
        out.append((lab, p))
    return out


def _auc_state(m):
    return np.stack([b.cpu().numpy() for b in (m.tp, m.fn, m.tn, m.fp)])


def _dev(x):
    return torch.as_tensor(np.asarray(x, F32), device="cuda")


@pytest.mark.parametrize("T", [2, 3, 200, 5000, 16384])
def test_auc_state_and_value_bit_exact(eb, T):
    from euler_b200 import metrics, ops
    rng = np.random.RandomState(T)
    m = metrics.StreamingAuc(T, device="cuda")
    want = ref.Auc(T, counts=ref.bucket_counts)
    for k, (lab, p) in enumerate(_batches(T, rng)):
        if p.size <= 4096:   # TF's literal comparison where it is small, else the bucket form it equals
            np.testing.assert_array_equal(ref.literal_counts(lab, p, T), ref.bucket_counts(lab, p, T))
        v = ops.metric_auc_update(_dev(lab), _dev(p), m.tp, m.fn, m.tn, m.fp, m.refused, m.value)
        wv = want.update(lab, p)
        _assert_bits(_auc_state(m), want.state, "T=%d batch %d state" % (T, k))
        _assert_bits(v.item(), wv, "T=%d batch %d value" % (T, k))
        assert abs(v.item() - ref.auc_value_f64(*want.state)) < 1e-6
    assert int(m.refused) == 0


def test_auc_batch_above_2_24_follows_the_integer_count_rule(eb):
    from euler_b200 import ops
    T, n = 5000, (1 << 24) + 5
    g = torch.Generator(device="cuda").manual_seed(1)
    p = torch.rand(n, generator=g, device="cuda")
    lab = (torch.rand(n, generator=g, device="cuda") < p).float()
    st = [torch.zeros(T, device="cuda") for _ in range(4)]
    refused, value = torch.zeros((), dtype=torch.int64, device="cuda"), torch.zeros((), device="cuda")
    for rounds in (1, 2):
        ops.metric_auc_update(lab, p, *st, refused, value)
        counts = ref.bucket_counts(lab.cpu().numpy(), p.cpu().numpy(), T)
        want = counts.astype(F32)
        if rounds == 2:
            want = want + want
        _assert_bits(np.stack([s.cpu().numpy() for s in st]), want, "state after %d batches" % rounds)
        _assert_bits(value.item(), ref.auc_value(*want), "value")


def test_auc_refusals(eb):
    from euler_b200 import EulerError, metrics, ops
    T = 200
    m = metrics.StreamingAuc(T, device="cuda")
    want = ref.Auc(T)
    lab, p = np.array([1, 0, 1, 0], F32), np.array([0.9, 0.2, 0.6, 0.4], F32)
    ops.metric_auc_update(_dev(lab), _dev(p), m.tp, m.fn, m.tn, m.fp, m.refused, m.value)
    want.update(lab, p)
    before = _auc_state(m)
    for bad in ([0.5, 1.5, 0.2, 0.1], [0.5, -1e-30, 0.2, 0.1], [0.5, np.nan, 0.2, 0.1], [np.inf, 0.5, 0.5, 0.5]):
        v = ops.metric_auc_update(_dev(lab), _dev(bad), m.tp, m.fn, m.tn, m.fp, m.refused, m.value)
        assert np.isnan(v.item())
        _assert_bits(_auc_state(m), before, "a refused batch leaves the state")
    assert int(m.refused) == 4 and np.isnan(m.result().item())
    ops.metric_auc_update(_dev(lab), _dev(p), m.tp, m.fn, m.tn, m.fp, m.refused, m.value)   # counted, still NaN
    want.update(lab, p)
    _assert_bits(_auc_state(m), want.state, "counted after a refusal")
    assert np.isnan(m.value.item())
    m.reset()
    assert int(m.refused) == 0 and m.result().item() == 0.0 and not _auc_state(m).any()
    x = torch.logit(_dev(p))   # StreamingAuc applies sigmoid itself
    v = m(_dev(lab), x)
    w = ref.Auc(T)
    _assert_bits(v.item(), w.update(lab, torch.sigmoid(x).cpu().numpy()), "value after reset")
    # bad shapes, dtypes, devices and T raise on the host
    st = (m.tp, m.fn, m.tn, m.fp, m.refused, m.value)
    for args in ((_dev([1, 0]), _dev([0.5])), (_dev(lab).double(), _dev(p)), (torch.as_tensor(lab), torch.as_tensor(p)),
                 (_dev(lab), _dev(p).half())):
        with pytest.raises(EulerError):
            ops.metric_auc_update(*args, *st)
    with pytest.raises(EulerError):
        ops.metric_auc_update(_dev(lab), _dev(p), m.tp[:1], m.fn[:1], m.tn[:1], m.fp[:1], m.refused, m.value)
    with pytest.raises(EulerError):
        ops.metric_auc_update(_dev(lab), _dev(p), m.tp, m.fn[:5], m.tn, m.fp, m.refused, m.value)
    with pytest.raises(EulerError):
        ops.metric_auc_update(_dev(lab), _dev(p), m.tp, m.fn, m.tn, m.fp, m.refused.int(), m.value)
    for T_bad in (1, 16385, 0):
        big = torch.zeros(max(T_bad, 1), device="cuda")
        with pytest.raises(EulerError):   # the library's own check
            ops._call("eu_metric_auc_update", _dev(lab), _dev(p), 4, T_bad, big, big, big, big, m.refused, m.value)
    with pytest.raises(EulerError):
        ops._call("eu_metric_auc_update", _dev(lab), _dev(p), -1, T, *st)
    for bad in (1, 16385):
        with pytest.raises(ValueError):
            metrics.StreamingAuc(bad)


def _ibits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _capture(step):
    """step captured in a CUDA graph on a side stream, after one eager run there (which binds the ctx to that stream)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = step()
    torch.cuda.current_stream().wait_stream(s)
    return cg, out


@pytest.mark.parametrize("T", [200, 5000])
def test_repeat_bits_and_graph_replay(eb, T):
    from euler_b200 import metrics
    g = torch.Generator(device="cuda").manual_seed(T)
    batches = []
    for n in (61952, 20480, 7):
        x = torch.randn(n, generator=g, device="cuda")
        batches.append(((torch.rand(n, generator=g, device="cuda") < torch.sigmoid(x)).float(), torch.sigmoid(x)))
    mods = [metrics.StreamingAuc(T, device="cuda"), metrics.StreamingF1(device="cuda"), metrics.StreamingAccuracy(device="cuda")]

    def run():
        for m in mods:
            m.reset()
        vals = [[m(lab, p) for m in mods] for lab, p in batches]
        return vals, [[b.clone() for b in m.buffers()] for m in mods]

    v1, s1 = run()
    v2, s2 = run()
    for a, b in zip(sum(v1, []) + sum(s1, []), sum(v2, []) + sum(s2, [])):
        assert torch.equal(_ibits(a), _ibits(b))
    # one captured update of each metric, replayed three times from a reset state, against three eager updates
    lab0, p0 = batches[0]
    cg, out = _capture(lambda: [m(lab0, p0) for m in mods])
    for m in mods:
        m.reset()
    cg.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, v1[0]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    cg.replay()
    cg.replay()
    eager = [metrics.StreamingAuc(T, device="cuda"), metrics.StreamingF1(device="cuda"), metrics.StreamingAccuracy(device="cuda")]
    for _ in range(3):
        vals = [e(lab0, p0) for e in eager]
    torch.cuda.synchronize()
    for a, b in zip(out, vals):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for m, e in zip(mods, eager):
        for a, b in zip(m.buffers(), e.buffers()):
            assert torch.equal(_ibits(a), _ibits(b))


@pytest.mark.parametrize("kind", ["f1", "acc"])
def test_count_metrics_bit_exact(eb, kind):
    from euler_b200 import metrics
    rng = np.random.RandomState(11)
    m = metrics.get(kind, device="cuda")
    want = ref.F1() if kind == 'f1' else ref.Accuracy()
    edge = np.array([0.49999997, 0.5, -0.5, 0.49999994, 1.5, -0.50000006, np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45], F32)
    batches = [(rng.choice(LABEL_VALUES, size=edge.size), edge)]
    for n in (0, 1, 31, 1000, (1 << 20) + 7):
        p = (rng.rand(n) * 1.4 - 0.2).astype(F32)
        p[::7] = np.nan
        batches.append((rng.choice(LABEL_VALUES, size=n), p))
    for k, (lab, p) in enumerate(batches):
        v = m(_dev(lab), _dev(p))
        wv = want.update(lab, p)
        _assert_bits(m.state.cpu().numpy(), want.state, "%s batch %d state" % (kind, k))
        _assert_bits(v.item(), wv, "%s batch %d value" % (kind, k))
    m.reset()
    assert m.result().item() == 0.0 and not m.state.cpu().numpy().any()


def test_add_counts_equals_the_prediction_form(eb):
    from euler_b200 import EulerError, metrics, ops
    rng = np.random.RandomState(12)
    a, b = metrics.StreamingAccuracy(device="cuda"), metrics.StreamingAccuracy(device="cuda")
    for n in (20480, 0, 5, 61952):
        lab = (rng.rand(n) < 0.5).astype(F32)
        p = rng.rand(n).astype(F32)
        correct = torch.as_tensor(int((ref.rounded(p) == lab).sum()), device="cuda")
        va, vb = a(_dev(lab), _dev(p)), b.add_counts(correct, n)
        assert torch.equal(va.view(torch.int32), vb.view(torch.int32)) and torch.equal(a.state, b.state)
    with pytest.raises(EulerError):
        ops.metric_count_update('f1', b.state, b.value, correct=correct, total=5)
    with pytest.raises(EulerError):
        ops.metric_count_update('acc', b.state, b.value, correct=correct.int(), total=5)
    with pytest.raises(EulerError):
        ops.metric_count_update('auc', b.state, b.value, _dev([1.0]), _dev([1.0]))
    with pytest.raises(EulerError):
        ops.metric_count_update('f1', b.state, b.value, _dev([1.0]), _dev([1.0]))   # f1's state is f32[3]
    with pytest.raises(EulerError):
        ops._call("eu_metric_count_update", 7, _dev([1.0]), _dev([1.0]), 1, None, b.state, b.value)


# ---------------------------------------------------------------------------- whole training steps
MAX_ID, FEAT = 3000, 16


@pytest.fixture
def feature_graph():
    import euler_b200
    g = graphs.random_graph(seed=49, n=MAX_ID, T=1, avg_deg=5, feat_dim=FEAT)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    return euler_b200


@pytest.mark.parametrize("metric", ["auc", "f1", "acc"])
def test_supervise_model_steps(feature_graph, metric):
    from euler_b200 import encoders
    from euler_b200.supervised import SuperviseModel
    torch.manual_seed(2)
    enc = encoders.SageEncoder([[0], [0]], [5, 2], 8, 'mean', feature_idx=0, feature_dim=FEAT, max_id=MAX_ID, device="cuda")

    class Model(SuperviseModel):
        def __init__(self, streaming):
            super().__init__(0, 3, metric, dim=8, device="cuda", streaming=streaming)

        def embed(self, n_id):
            return enc(n_id)

    model = Model(True)
    assert 'metric' in dict(model.named_children()) and not any(k.startswith('metric') for k in model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    want = {'auc': lambda: ref.Auc(5000), 'f1': ref.F1, 'acc': ref.Accuracy}[metric]()
    rng = np.random.RandomState(5)
    for step in range(3):
        inputs = torch.as_tensor(rng.randint(1, MAX_ID + 1, size=512), device="cuda")
        feature_graph.seed(31 + step)
        label, = feature_graph.get_dense_feature(inputs, [0], [3])
        feature_graph.seed(31 + step)
        emb, loss, name, value = model(inputs)
        with torch.no_grad():
            logit = model.out_fc(emb)
        p = torch.sigmoid(logit)
        if metric == 'auc':
            p = torch.sigmoid(p)
        wv = want.update(label.cpu().numpy(), p.cpu().numpy())
        _assert_bits(value.item(), wv, "%s step %d" % (metric, step))
        opt.zero_grad()
        loss.backward()
        opt.step()
    state = _auc_state(model.metric) if metric == 'auc' else model.metric.state.cpu().numpy()
    _assert_bits(state, want.state, "state after three steps")


def test_gae_steps(feature_graph):
    from euler_b200 import autoencoder as ae, encoders
    torch.manual_seed(3)
    enc = encoders.SageEncoder([[0], [0]], [5, 5], 16, 'mean', feature_idx=0, feature_dim=FEAT, max_id=MAX_ID, device="cuda")
    model = ae.GraphAutoEncoder(enc, 0, [0], MAX_ID, num_negs=10, streaming=True)
    opt = torch.optim.Adam(model.parameters(), lr=0.01)
    want = ref.Accuracy()
    rng = np.random.RandomState(3)
    seen = []
    orig = model.fused_acc

    def record(correct, count):
        seen.append((int(correct), count))
        return orig(correct, count)
    model.fused_acc = record
    for step in range(3):
        inputs = torch.as_tensor(rng.randint(1, MAX_ID + 1, size=256), device="cuda")
        emb, loss, name, acc = model(inputs)
        _assert_bits(acc.item(), want.add_counts(*seen[-1]), "GAE step %d" % step)
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert [c for _, c in seen] == [2 * 256 * 10] * 3
    _assert_bits(model.metric.state.cpu().numpy(), want.state, "GAE state")
