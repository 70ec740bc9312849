"""Graph-level minibatches on the CPU (no device): the label list of eu_graph_labels_inspect against the reference's own
Graph::GetGraphLabel on the tiny fixture and the multi-graph one, the SparseTensor packing rule of get_graph_by_label, and Set2SetPool's TF LSTMCell restated in numpy."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from euler_b200 import graph_pool, ops  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

LABELS_SO = os.path.join(ROOT, "oracle", "_ref", "libeuler_ref_labels.so")
MULTI = os.path.join(ROOT, "tests", "golden", "multigraph_euler")


def ref_graph_labels(directory):
    """Graph::GetGraphLabel of the reference's own load of `directory`"""
    po.RefGraph.load(directory, "all", "all")
    R = C.CDLL(LABELS_SO)
    R.ref_graph_labels.restype = C.c_int64
    R.ref_graph_labels.argtypes = [C.c_int64, C.c_char_p, C.c_void_p, C.c_int64]
    n = R.ref_graph_labels(0, None, None, 0)
    ends = np.zeros(max(n, 1), np.int64)
    R.ref_graph_labels(0, None, ends.ctypes.data, n)
    total = int(ends[n - 1]) if n else 0
    buf = C.create_string_buffer(max(total, 1))
    R.ref_graph_labels(total, buf, ends.ctypes.data, n)
    raw = buf.raw[:total]
    starts = [0] + [int(e) for e in ends[:n - 1]]
    return [raw[s:int(e)] for s, e in zip(starts, ends[:n])]


@pytest.mark.parametrize("fixture", ["tiny_euler", "multigraph_euler"])
def test_inspect_lists_the_reference_labels_in_its_order(fixture):
    if not os.path.exists(LABELS_SO):
        pytest.skip("the reference shim oracle/_ref/libeuler_ref_labels.so is not built (no reference sources)")
    directory = os.path.join(ROOT, "tests", "golden", fixture)
    got = ops.inspect_graph_labels(directory)
    assert got == ref_graph_labels(directory)
    if fixture == "multigraph_euler":     # 40 graphs and the "" of the nodes without a graph_label
        assert len(got) == 41 and b"" in got


def pack(node_lists):
    """tf_euler/kernels/get_graph_by_label_op.cc's SparseTensorBuilder: row i lists graph i's ids at (i, j); a graph without
    ids gets the single entry (i, 0) = 0"""
    idx, val = [], []
    for i, ids in enumerate(node_lists):
        if len(ids) == 0:
            idx.append((i, 0)); val.append(0)
        for j, v in enumerate(ids):
            idx.append((i, j)); val.append(v)
    shape = (len(node_lists), max([max(len(x), 1) for x in node_lists], default=0))
    return np.asarray(idx, np.int64).reshape(-1, 2), np.asarray(val, np.int64), shape


def test_packing_rule_of_empty_and_unknown_labels():
    idx, val, shape = pack([[5, 7, 9], [], [3], []])
    assert idx.tolist() == [[0, 0], [0, 1], [0, 2], [1, 0], [2, 0], [3, 0]]
    assert val.tolist() == [5, 7, 9, 0, 3, 0]
    assert shape == (4, 3)
    idx, val, shape = pack([])
    assert idx.shape == (0, 2) and val.shape == (0,) and shape == (0, 0)


def np_lstm_cell(x, c, h, kernel, bias, forget_bias=1.0):
    """TF 1.x LSTMCell (no peepholes, no projection): i, j, f, o = split(concat([x, h]) W + b, 4);
    c' = sigmoid(f + forget_bias) c + sigmoid(i) tanh(j); h' = sigmoid(o) tanh(c')"""
    sig = lambda z: 1.0 / (1.0 + np.exp(-z))  # noqa: E731
    z = np.concatenate([x, h], axis=1) @ kernel + bias
    i, j, f, o = np.split(z, 4, axis=1)
    c2 = sig(f + forget_bias) * c + sig(i) * np.tanh(j)
    return sig(o) * np.tanh(c2), c2


@pytest.mark.parametrize("layers", [1, 2, 3])
def test_lstm_is_tf_multi_rnn_cell_of_lstm_cells(layers):
    torch.manual_seed(layers)
    dim, B = 6, 5
    cell = graph_pool.MultiRNNCell([graph_pool.LSTMCell(2 * dim if k == 0 else dim, dim) for k in range(layers)]).double()
    with torch.no_grad():
        for cl in cell.cells:
            cl.bias.uniform_(-0.5, 0.5)
    rs = np.random.RandomState(layers)
    x = rs.randn(B, 2 * dim)
    state = [(rs.randn(B, dim), rs.randn(B, dim)) for _ in range(layers)]
    out, new = cell(torch.from_numpy(x), [(torch.from_numpy(c), torch.from_numpy(h)) for c, h in state])
    inp = x
    for k, cl in enumerate(cell.cells):     # MultiRNNCell: each cell fed the previous one's output
        h, c = np_lstm_cell(inp, state[k][0], state[k][1], cl.kernel.detach().numpy(), cl.bias.detach().numpy())
        np.testing.assert_allclose(new[k][0].detach().numpy(), c, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(new[k][1].detach().numpy(), h, rtol=1e-12, atol=1e-12)
        inp = h
    np.testing.assert_allclose(out.detach().numpy(), inp, rtol=1e-12, atol=1e-12)
