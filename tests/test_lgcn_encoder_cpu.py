"""CPU: LGCEncoder's constructor and its literal composition (fused=False) on a deterministic CPU stand-in of sample_neighbor /
get_dense_feature, against a float64 numpy restatement of encoders.py:895-922 (a stable top_k, TF's channels-last 'valid'
conv1d, row 0); and one LGCN loss and f1 against the same restatement."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import ops
from euler_b200.encoders import LGCEncoder
from euler_b200.supervised import LGCN, f1_score

N_IDS = 12                                        # ids 1 .. 12 have rows; any other id is absent
_rng = np.random.RandomState(3)
FEAT = {'f': (_rng.randint(-4, 5, size=(N_IDS, 6)) / 4).astype(np.float32),       # quarters in [-1, 1]: many ties
        'lab': _rng.randint(0, 2, size=(N_IDS, 3)).astype(np.float32)}


def _dense_feature(nodes, names, dims, thread_num=1):
    """get_dense_feature's rule: the stored columns, zeros past them, a zero row for an absent id"""
    out = []
    for name, d in zip(names, dims):
        f = np.zeros((nodes.numel(), d), np.float32)
        for i, n in enumerate(nodes.reshape(-1).tolist()):
            if 1 <= n <= N_IDS:
                w = min(d, FEAT[name].shape[1])
                f[i, :w] = FEAT[name][n - 1, :w]
        out.append(torch.as_tensor(f))
    return out


def _sample_neighbor(nodes, edge_types, count, default_node=-1, condition=''):
    """a deterministic stand-in: neighbour j of node n is (5 n + 3 j) % 15, the absent id 13 kept, 14 replaced by
    default_node"""
    nodes = torch.as_tensor(nodes, dtype=torch.int64).reshape(-1)
    nb = (5 * nodes[:, None] + 3 * torch.arange(count)[None, :]) % 15
    return torch.where(nb == 14, torch.full_like(nb, default_node), nb), None, None


@pytest.fixture
def cpu_ops(monkeypatch):
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    monkeypatch.setattr(ops, "sample_neighbor", _sample_neighbor)


def f64(t):
    return t.detach().double().numpy()


def _top_k_rows_f64(nodes, nb_num, name, dim, k):
    """[B, k + 1, dim]: the node row, then tf.nn.top_k over each column of the neighbour rows (equal values: lower index
    first)"""
    nb = _sample_neighbor(nodes, [0], nb_num)[0]
    node = f64(_dense_feature(nodes, [name], [dim])[0])
    rows = f64(_dense_feature(nb.reshape(-1), [name], [dim])[0]).reshape(-1, nb_num, dim)
    order = np.argsort(-rows, axis=1, kind='stable')[:, :k]
    return np.concatenate([node[:, None], np.take_along_axis(rows, order, axis=1)], 1)


def _conv1d_valid(x, conv):
    """tf.layers.conv1d, channels last, 'valid': out[b, t, o] = sum_{w, i} x[b, t + w, i] kernel[w, i, o] + bias[o], with
    kernel[w, i, o] = conv.weight[o, i, w]"""
    kernel = f64(conv.weight).transpose(2, 1, 0)
    width = kernel.shape[0]
    T = x.shape[1] - width + 1
    return np.stack([np.einsum('bwi,wio->bo', x[:, t:t + width], kernel) for t in range(T)], 1) + f64(conv.bias)


def _lgc_f64(enc, inputs):
    nodes = torch.as_tensor(inputs).reshape(-1)
    x = _top_k_rows_f64(nodes, enc.nb_num, enc.feature_idx, enc.feature_dim, enc.k)
    return _conv1d_valid(_conv1d_valid(x, enc.conv1), enc.conv2)[:, 0]


def test_constructor_arguments_errors_and_widths():
    with pytest.raises(ValueError, match="feature_idx"):
        LGCEncoder([0])
    with pytest.raises(ValueError, match="nb_num"):
        LGCEncoder([0], 'f', 6, k=11, nb_num=10)
    with pytest.raises(ValueError, match="nb_num"):
        LGCEncoder([0], 'f', 6, k=0)
    enc = LGCEncoder([0], 'f', 6)
    assert (enc.k, enc.hidden_dim, enc.nb_num, enc.out_dim, enc.fused) == (3, 128, 10, 64, True)   # upstream's defaults
    for k in (1, 2, 3, 4, 5):
        enc = LGCEncoder([0], 'f', 6, k, 7, 10, 5)
        assert tuple(enc.conv1.weight.shape) == (7, 6, k // 2 + 1) and tuple(enc.conv2.weight.shape) == (5, 7, k // 2 + 1)
        assert not enc.conv1.bias.any() and not enc.conv2.bias.any()
        bound = (6.0 / ((6 + 7) * (k // 2 + 1))) ** 0.5                       # glorot-uniform over the kernel's fans
        assert enc.conv1.weight.abs().max() <= bound
        assert enc.conv1.padding == (0,) and enc.conv1.stride == (1,)


@pytest.mark.parametrize("same", (True, False))
@pytest.mark.parametrize("k", (1, 2, 3, 4))
def test_composition_against_float64(cpu_ops, k, same):
    nb_num = k if same else 10
    torch.manual_seed(k)
    enc = LGCEncoder([0], 'f', 8, k, 7, nb_num, 5, fused=False)          # 8 columns: two past the slot's stored 6
    inputs = torch.as_tensor([[3, 5, 11], [8, 1, 13], [2, 12, 6]], dtype=torch.int64)   # 13 is absent
    nodes = inputs.reshape(-1)
    x = enc.top_k_rows(nodes, _sample_neighbor(nodes, [0], nb_num)[0])
    assert x.shape == (9, k + 1, 8) and x.dtype == torch.float32
    np.testing.assert_array_equal(f64(x), _top_k_rows_f64(nodes, nb_num, 'f', 8, k))
    out = enc(inputs)
    assert out.shape == (9, 5) and out.dtype == torch.float32
    np.testing.assert_allclose(f64(out), _lgc_f64(enc, inputs), rtol=1e-5, atol=1e-6)


def test_odd_k_never_reads_the_kth_value(cpu_ops):
    """upstream's quirk: for odd k the two valid convolutions reach rows 0 .. 2 (k // 2) only"""
    torch.manual_seed(0)
    enc = LGCEncoder([0], 'f', 6, 3, 7, 10, 5, fused=False)
    nodes = torch.as_tensor([3, 5, 11], dtype=torch.int64)
    x = enc.top_k_rows(nodes, _sample_neighbor(nodes, [0], 10)[0])
    h = enc.conv2(enc.conv1(x.transpose(1, 2)))[:, :, 0]
    x[:, 3] = 1e3
    torch.testing.assert_close(enc.conv2(enc.conv1(x.transpose(1, 2)))[:, :, 0], h, rtol=0, atol=0)


def _xent(x, z):
    return np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))


def test_lgcn_loss_and_f1_against_float64(cpu_ops):
    torch.manual_seed(0)
    model = LGCN(7, [0], 'lab', 3, feature_idx='f', feature_dim=6, k=3, nb_num=10, out_dim=5, fused=False)
    assert tuple(model.out_fc.weight.shape) == (3, 5) and model.out_fc.bias is None     # out_fc reads out_dim columns
    enc = model._encoder
    assert (enc.hidden_dim, enc.out_dim, enc.edge_type) == (7, 5, [0])
    inputs = torch.as_tensor([3, 5, 11, 8, 2, 13, 9], dtype=torch.int64)
    emb, loss, name, metric = model(inputs)
    h = _lgc_f64(enc, inputs)
    logit = h @ f64(model.out_fc.weight).T
    label = f64(_dense_feature(inputs, ['lab'], [3])[0])
    assert name == 'f1' and emb.shape == (7, 5)
    np.testing.assert_allclose(f64(emb), h, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(loss.item(), _xent(logit, label).mean(), rtol=1e-5)
    want = f1_score(torch.as_tensor(label), torch.as_tensor(1 / (1 + np.exp(-logit))))
    np.testing.assert_allclose(float(metric), float(want), rtol=1e-6)
    loss.backward()
    assert all(p.grad is not None for p in model.parameters())
