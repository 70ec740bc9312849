"""CPU: ShallowEncoder's constructor (upstream's ValueErrors, output_dim and the sub-layers it builds for every combination
of inputs) and its literal composition (fused=False) on a CPU stand-in of the feature ops, against a float64 numpy
restatement of encoders.py:134-171."""
import itertools

import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
from euler_b200 import ops
from euler_b200.encoders import ShallowEncoder


def test_constructor_errors():
    with pytest.raises(ValueError, match="combiner"):
        ShallowEncoder(combiner='mean')
    with pytest.raises(ValueError, match="dim provided"):
        ShallowEncoder(combiner='add')
    with pytest.raises(ValueError, match="feature_dim"):
        ShallowEncoder(feature_idx=['a', 'b'], feature_dim=[3])
    with pytest.raises(ValueError, match="sparse_feature_idx"):
        ShallowEncoder(sparse_feature_idx=['a', 'b'], sparse_feature_max_id=[3])
    with pytest.raises(ValueError, match="embedding_num"):
        ShallowEncoder(max_id=5, sparse_feature_idx=['a'], sparse_feature_max_id=[3], embedding_dim=[4, 4, 4])
    with pytest.raises(ValueError, match="use_hash_embedding"):
        ShallowEncoder(max_id=5, use_hash_embedding=[False, False])
    with pytest.raises(NotImplementedError):
        ShallowEncoder(max_id=5, use_hash_embedding=True)
    ShallowEncoder(feature_idx=-1, use_hash_embedding=[True, False])   # no embeddings: the list is never read, as upstream


@pytest.mark.parametrize("use_id,use_feature,use_sparse,combiner,dim",
                         [c for c in itertools.product((False, True), (False, True), (False, True), ('concat', 'add'), (None, 6))
                          if not (c[3] == 'add' and c[4] is None)])
def test_output_dim_and_sub_layers(use_id, use_feature, use_sparse, combiner, dim):
    kw = dict(dim=dim, combiner=combiner, embedding_dim=[3, 5, 2][:use_id + 2 * use_sparse] if combiner == 'concat' else 16,
              feature_idx=['f1', 'f2'] if use_feature else -1, feature_dim=[4, 7] if use_feature else 0,
              max_id=9 if use_id else -1, sparse_feature_idx=['s1', 's2'] if use_sparse else -1,
              sparse_feature_max_id=[19, 29] if use_sparse else -1)
    enc = ShallowEncoder(**kw)
    emb = [] if not (use_id or use_sparse) else ([dim] * (use_id + 2 * use_sparse) if combiner == 'add' else kw['embedding_dim'])
    want = dim if dim is not None else (11 if use_feature else 0) + sum(emb)
    assert enc.output_dim == want
    assert hasattr(enc, 'embedding') == use_id and hasattr(enc, 'sparse_embeddings') == use_sparse and hasattr(enc, 'dense') == bool(dim)
    if use_id:
        assert tuple(enc.embedding.embeddings.shape) == (11, emb[0])                # Embedding(max_id + 1, d): max_id + 2 rows
    if use_sparse:
        shapes = [tuple(e.embeddings.shape) for e in enc.sparse_embeddings]
        assert shapes == [(21, emb[use_id]), (31, emb[use_id + 1])]
    if dim:
        in_dim = (11 if use_feature else 0) + (sum(emb) if combiner == 'concat' else 0)
        assert tuple(enc.dense.kernel.shape) == (in_dim, dim)
        assert (enc.dense.kernel.abs() <= 0.36 * (3.0 / max(in_dim, 1)) ** 0.5).all()


# ---------------------------------------------------------------------------- the composition on a CPU stand-in
IDS = np.array([3, 5, 8, 11], np.int64)              # the stand-in graph's nodes; other ids are absent
DENSE = {'f1': np.arange(4 * 3, dtype=np.float32).reshape(4, 3) / 7, 'f2': -np.arange(4 * 5, dtype=np.float32).reshape(4, 5) / 3}
SPARSE = {'s1': [[1, 4], [], [0, 0, 2], [7]], 's2': [[3], [1, 2], [], [0]]}


def _row(n):
    hit = np.flatnonzero(IDS == n)
    return int(hit[0]) if len(hit) else -1


def _dense_feature(nodes, names, dims, thread_num=1):
    out = []
    for name, d in zip(names, dims):
        f = np.zeros((nodes.numel(), d), np.float32)
        for i, n in enumerate(nodes.tolist()):
            r = _row(n)
            if r >= 0:
                k = min(d, DENSE[name].shape[1])
                f[i, :k] = DENSE[name][r, :k]
        out.append(torch.as_tensor(f))
    return out


def _sparse_feature(nodes, names, default_values=None, thread_num=1):
    out = []
    for name, dv in zip(names, default_values):
        rows, cols, vals = [], [], []
        for i, n in enumerate(nodes.tolist()):
            r = _row(n)
            bag = (SPARSE[name][r] if r >= 0 else []) or [dv]
            rows += [i] * len(bag)
            cols += list(range(len(bag)))
            vals += bag
        idx = torch.as_tensor(np.stack([rows, cols], 1), dtype=torch.int64)
        out.append((idx, torch.as_tensor(vals, dtype=torch.int64), (nodes.numel(), max(cols) + 1)))
    return out


def _restated(enc, nodes):
    """encoders.py:134-171 in float64 numpy, from the encoder's own parameters"""
    f64 = lambda t: t.detach().double().numpy()   # noqa: E731
    flat = nodes.reshape(-1)
    parts = []
    if enc.use_id:
        parts.append(f64(enc.embedding.embeddings)[flat])
    if enc.use_feature:
        feats = np.concatenate([d.numpy().astype(np.float64) for d in _dense_feature(torch.as_tensor(flat), enc.feature_idx, enc.feature_dim)], 1)
        parts.append(feats @ f64(enc.dense.kernel) if enc.combiner == 'add' else feats)
    if enc.use_sparse_feature:
        for name, m, e in zip(enc.sparse_feature_idx, enc.sparse_feature_max_id, enc.sparse_embeddings):
            t = f64(e.embeddings)
            parts.append(np.stack([t[(SPARSE[name][_row(n)] if _row(n) >= 0 else []) or [m + 1]].sum(0) for n in flat]))
    if enc.combiner == 'add':
        out = sum(parts)
    else:
        out = np.concatenate(parts, 1)
        if enc.dim:
            out = out @ f64(enc.dense.kernel)
    return out.reshape(nodes.shape + (enc.output_dim,))


@pytest.mark.parametrize("combiner,dim", [('concat', None), ('concat', 6), ('add', 4)])
def test_composition_against_float64(monkeypatch, combiner, dim):
    monkeypatch.setattr(ops, "get_dense_feature", _dense_feature)
    monkeypatch.setattr(ops, "get_sparse_feature", _sparse_feature)
    torch.manual_seed(0)
    enc = ShallowEncoder(dim=dim, feature_idx=['f1', 'f2'], feature_dim=[4, 2], max_id=12, sparse_feature_idx=['s1', 's2'],
                         sparse_feature_max_id=[9, 4], embedding_dim=[3, 2, 5], combiner=combiner, fused=False)
    nodes = torch.as_tensor([[3, 5, 2], [11, 8, 0], [12, 3, 3]], dtype=torch.int64)   # 2, 0 and 12: absent nodes
    out = enc(nodes)
    assert out.shape == (3, 3, enc.output_dim) and out.dtype == torch.float32
    np.testing.assert_allclose(out.detach().double().numpy(), _restated(enc, nodes.numpy()), rtol=1e-6, atol=1e-6)
