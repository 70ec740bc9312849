"""Graph-level minibatches on the GPU: sample_graph_label against the reference's engine loop, get_graph_by_label against a
numpy restatement, and the fused attention readout of AttentionPool / Set2SetPool (eu_graph_attention_readout, forward and
backward) against the composition of the mp ops and a float64 restatement.

Readout forward: on dyadic inputs (entries k/8) every product and partial sum is exact, so for graphs of at most 256 rows the
op equals scatter_softmax -> multiply -> scatter_add bit for bit; on random inputs it is within 1e-5 of float64.  An unsorted
index gives the bits of the stably sorted rows.  Backward: within 1e-5 of float64 autograd, identical from run to run."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import euler_b200  # noqa: E402
from euler_b200 import graph_pool, ops  # noqa: E402
from euler_b200._lib import EulerError  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

pytestmark = pytest.mark.gpu
LABELS_SO = os.path.join(ROOT, "oracle", "_ref", "libeuler_ref_labels.so")
DIMS = (1, 3, 4, 64, 128, 200)


def cuda(a, dtype=np.float32):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


# ------------------------------------------------------------------------------------------------ graphs with labels
def labelled_graph(rs, n_graphs, sizes=None, unlabelled=5, name="graph_label"):
    """a disjoint union of path graphs with a binary slot `name`: graph k's nodes carry the label b'g<k>', `unlabelled` nodes
    carry none; ids are shuffled so that a label's rows are not in id order.  Returns (Graph, ids, per-node label bytes)."""
    sizes = rs.randint(1, 40, size=n_graphs) if sizes is None else np.asarray(sizes)
    n = int(sizes.sum()) + unlabelled
    ids = rs.permutation(np.arange(1, n + 1)).astype(np.uint64)
    vals = [b"g%d" % k for k, s in enumerate(sizes) for _ in range(s)] + [b""] * unlabelled
    grp_ptr = np.zeros(n + 1, np.int64)
    bin_ptr = np.zeros(n + 1, np.int64)
    bin_ptr[1:] = np.cumsum([len(v) for v in vals])
    g = euler_b200.Graph.from_csr(ids, grp_ptr, np.zeros(0, np.uint64), w=np.zeros(0, np.float32), bin_ptr=bin_ptr,
                                  bin_val=np.frombuffer(b"".join(vals), np.uint8) if bin_ptr[-1] else np.zeros(0, np.uint8),
                                  n_bin_slots=1, binary_feature_names=[name])
    return g, ids, vals


def restated_by_label(ids, vals, labels):
    """get_graph_by_label restated from the node arrays: row i = the ids of label i ascending, (i, 0) = 0 when there are none"""
    idx, out = [], []
    for i, lab in enumerate(labels):
        mine = sorted(int(x) for x, v in zip(ids, vals) if v == lab and lab != b"")
        if not mine:
            idx.append((i, 0)); out.append(0)
        for j, x in enumerate(mine):
            idx.append((i, j)); out.append(x)
    return np.asarray(idx, np.int64).reshape(-1, 2), np.asarray(out, np.int64)


def ref_labels_lib():
    R = C.CDLL(LABELS_SO)
    R.ref_sample_graph_label.argtypes = [C.c_int32, C.c_int64, C.c_void_p]
    return R


@pytest.mark.parametrize("seed", [1, 7, 12345])
def test_sample_graph_label_is_the_reference_stream(tiny_dir, seed):
    gr = euler_b200.Graph.load(tiny_dir)
    euler_b200.set_graph(gr, rng="minstd", seed=seed)
    L = len(ops.graph_labels())
    got = ops.sample_graph_label(300).cpu().numpy()
    after = ops.sample_node(50, "-1").cpu().numpy()
    po.RefGraph.load(tiny_dir)
    po.ref().ref_seed(seed)
    want = np.zeros(300, np.int32)
    ref_labels_lib().ref_sample_graph_label(300, L, want.ctypes.data)
    want_after = np.zeros(50, np.uint64)
    po.ref().ref_sample_node(np.asarray([-1], np.int32), 1, 50, want_after)
    assert np.array_equal(got, want)
    assert np.array_equal(after.astype(np.uint64), want_after), "the stream position after the label draws"
    assert ops.sample_graph_label(0).numel() == 0


def test_graph_without_labels_is_a_state_error():
    rs = np.random.RandomState(0)
    g, _, _ = labelled_graph(rs, 3, name="not_a_label")
    euler_b200.set_graph(g)
    for call in (lambda: ops.sample_graph_label(4), ops.graph_labels, lambda: ops.get_graph_by_label(["g0"])):
        with pytest.raises(EulerError, match="graph label set is empty"):
            call()


def test_philox_draws_every_label_uniformly():
    from scipy.stats import chisquare
    rs = np.random.RandomState(1)
    g, _, _ = labelled_graph(rs, 37, unlabelled=0)
    euler_b200.set_graph(g, rng="philox", seed=3)
    L = len(ops.graph_labels())
    draws = torch.cat([ops.sample_graph_label(20000) for _ in range(5)]).cpu().numpy()
    counts = np.bincount(draws, minlength=L)
    assert counts.shape == (L,) and counts.min() > 0
    assert chisquare(counts).pvalue > 1e-4


def test_get_graph_by_label_matches_the_restatement():
    rs = np.random.RandomState(2)
    g, ids, vals = labelled_graph(rs, 40, sizes=list(rs.randint(1, 60, size=39)) + [300])
    euler_b200.set_graph(g)
    labels = ops.graph_labels()
    assert sorted(labels) == sorted(set(vals))
    pick = [labels.index(b"g3"), labels.index(b"g3"), labels.index(b"g39"), labels.index(b""), -1, labels.index(b"g0")]
    idx, val, shape = ops.get_graph_by_label(torch.tensor(pick, dtype=torch.int32, device="cuda"))
    want_idx, want_val = restated_by_label(ids, vals, [labels[p] if p >= 0 else b"?" for p in pick])
    assert np.array_equal(idx.cpu().numpy(), want_idx) and np.array_equal(val.cpu().numpy(), want_val)
    assert shape == (len(pick), 300)
    idx2, val2, shape2 = ops.get_graph_by_label(["g3", "g3", "g39", "", "no such label", b"g0"])
    assert torch.equal(idx, idx2) and torch.equal(val, val2) and shape2 == shape
    idx0, val0, shape0 = ops.get_graph_by_label(torch.zeros(0, dtype=torch.int32, device="cuda"))
    assert idx0.shape == (0, 2) and val0.numel() == 0 and shape0 == (0, 0)
    drawn = ops.sample_graph_label(64)
    idx3, val3, _ = ops.get_graph_by_label(drawn)
    want_idx, want_val = restated_by_label(ids, vals, [labels[p] for p in drawn.cpu().tolist()])
    assert np.array_equal(idx3.cpu().numpy(), want_idx) and np.array_equal(val3.cpu().numpy(), want_val)


# ------------------------------------------------------------------------------------------------ readout
def batch_index(sizes):
    return torch.from_numpy(np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)).cuda()


def composition(x, index, B, logits=None, q=None):
    """attention_pool.py / set2set_pool.py composed from the mp ops"""
    e = logits.view(-1, 1) if q is None else (x * ops.gather(q, index)).sum(-1, keepdim=True)
    a = ops.scatter_softmax(e, index, B)
    return ops.scatter_add(a * x, index, B), a.view(-1)


def readout64(x, index, B, logits=None, q=None):
    """the readout in float64 torch: max from -1e9, exp, sum, alpha, weighted sum"""
    x, idx = x.double(), index.long()
    lg = logits.double().view(-1) if q is None else (x * q.double()[idx]).sum(1)
    m = torch.full((B,), -1e9, dtype=torch.float64, device=x.device).scatter_reduce(0, idx, lg, "amax", include_self=True)
    ex = torch.exp(lg - m[idx])
    s = torch.zeros(B, dtype=torch.float64, device=x.device).index_add(0, idx, ex)
    a = ex / s[idx]
    return torch.zeros(B, x.shape[1], dtype=torch.float64, device=x.device).index_add(0, idx, a[:, None] * x), a


SIZES = [0, 1, 255, 256, 257, 3, 0, 1300, 40]


def unaligned(t):
    """the same values at a row start that is 4 bytes past a 16-byte boundary"""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("mode", ["logits", "q"])
def test_forward_is_bit_exact_on_dyadic_inputs(dim, mode):
    euler_b200.set_graph(labelled_graph(np.random.RandomState(0), 2)[0])
    rs = np.random.RandomState(dim)
    small = [0, 1, 255, 256, 3, 0, 17]
    B, index = len(small), batch_index(small)
    N = int(index.numel())
    x = cuda(rs.randint(-4, 5, size=(N, dim)) / 8.0)
    lg = cuda(rs.randint(-4, 5, size=N) / 8.0)
    q = cuda(rs.randint(-4, 5, size=(B, dim)) / 8.0) if mode == "q" else None
    for xx in (x, unaligned(x)):
        out = ops.graph_attention_readout(xx, index, B, logits=None if q is not None else lg, q=q)
        want, _ = composition(xx, index, B, logits=None if q is not None else lg, q=q)
        assert torch.equal(out, want), "dim=%d aligned=%s" % (dim, xx.data_ptr() % 16 == 0)
        assert torch.equal(out[0], torch.zeros(dim, device="cuda")) and torch.equal(out[5], out[0])


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("mode", ["logits", "q"])
def test_forward_matches_float64_and_unsorted_index_gives_sorted_bits(dim, mode):
    euler_b200.set_graph(labelled_graph(np.random.RandomState(0), 2)[0])
    rs = np.random.RandomState(100 + dim)
    B, index = len(SIZES), batch_index(SIZES)
    N = int(index.numel())
    x = cuda(rs.randn(N, dim))
    lg = cuda(rs.randn(N) * 3)
    q = cuda(rs.randn(B, dim) / np.sqrt(dim)) if mode == "q" else None
    kw = dict(logits=lg) if q is None else dict(q=q)
    out = ops.graph_attention_readout(x, index, B, **kw)
    want, _ = readout64(x, index, B, **kw)
    torch.testing.assert_close(out.double(), want, rtol=1e-5, atol=1e-5)
    perm = torch.from_numpy(rs.permutation(N)).cuda()
    kw2 = dict(logits=lg[perm]) if q is None else dict(q=q)
    out2 = ops.graph_attention_readout(x[perm], index[perm], B, **kw2)
    # the permuted rows against the same rows stably sorted by graph
    order = torch.sort(index[perm].long(), stable=True).indices
    kw3 = dict(logits=lg[perm][order]) if q is None else dict(q=q)
    out3 = ops.graph_attention_readout(x[perm][order], index[perm][order], B, **kw3)
    assert torch.equal(out2, out3)


@pytest.mark.parametrize("dim", (3, 64, 200))
@pytest.mark.parametrize("mode", ["logits", "q"])
def test_backward_matches_float64_autograd_and_is_deterministic(dim, mode):
    euler_b200.set_graph(labelled_graph(np.random.RandomState(0), 2)[0])
    rs = np.random.RandomState(200 + dim)
    B, index = len(SIZES), batch_index(SIZES)
    N = int(index.numel())
    x0, lg0 = rs.randn(N, dim), rs.randn(N) * 2
    q0 = rs.randn(B, dim) / np.sqrt(dim)
    g0 = rs.randn(B, dim)
    g0[2] = 0.0                                          # a graph that gets no gradient: its rows get exact zeros
    w0 = q0 if mode == "q" else lg0

    def run():
        x, w = cuda(x0).requires_grad_(), cuda(w0).requires_grad_()
        kw = dict(q=w) if mode == "q" else dict(logits=w)
        ops.graph_attention_readout(x, index, B, **kw).backward(cuda(g0))
        return x.grad, w.grad

    gx, gw = run()
    gx2, gw2 = run()
    assert torch.equal(gx, gx2) and torch.equal(gw, gw2)
    x, w = cuda(x0, np.float64).requires_grad_(), cuda(w0, np.float64).requires_grad_()
    kw = dict(q=w) if mode == "q" else dict(logits=w)
    readout64(x, index, B, **kw)[0].backward(cuda(g0, np.float64))
    torch.testing.assert_close(gx.double(), x.grad, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(gw.double(), w.grad, rtol=1e-5, atol=1e-5)
    rows2 = index == 2
    assert torch.count_nonzero(gx[rows2]) == 0
    if mode == "logits":
        assert torch.count_nonzero(gw[rows2]) == 0
    # autograd through the float32 composition agrees too
    x, w = cuda(x0).requires_grad_(), cuda(w0).requires_grad_()
    kw = dict(q=w) if mode == "q" else dict(logits=w)
    composition(x, index, B, **kw)[0].backward(cuda(g0))
    torch.testing.assert_close(gx, x.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gw, w.grad, rtol=1e-4, atol=1e-4)


def test_pools_match_float64_restatements():
    euler_b200.set_graph(labelled_graph(np.random.RandomState(0), 2)[0])
    torch.manual_seed(0)
    rs = np.random.RandomState(6)
    sizes = [5, 1, 30, 300, 12]
    B, index = len(sizes), batch_index(sizes)
    N = int(index.numel())
    x = cuda(rs.randn(N, 16))
    ap = graph_pool.AttentionPool()
    out = ap(x, index, B)
    gate = ap.gate_nn(x)
    want, _ = readout64(x, index, B, logits=gate.detach())
    torch.testing.assert_close(out.double(), want, rtol=1e-5, atol=1e-5)
    for aggr in ("mean", "max"):
        o2 = graph_pool.AttentionPool(gate_nn=ap.gate_nn, aggr=aggr)(x, index, B)
        assert o2.shape == (B, 16)
    s2s = graph_pool.Set2SetPool(16, processing_steps=3, num_layers=2)
    got = s2s(x, index, B)
    comp = graph_pool.Set2SetPool(16, processing_steps=3, num_layers=2)
    comp.lstm.load_state_dict(s2s.lstm.state_dict())
    lstm64 = comp.lstm.double().cuda()
    cell_in = torch.zeros(B, 32, dtype=torch.float64, device="cuda")
    state = lstm64.zero_state(B, "cuda")
    state = [(c.double(), h.double()) for c, h in state]
    for _ in range(3):
        q, state = lstm64(cell_in, state)
        r, _ = readout64(x, index, B, q=q)
        cell_in = torch.cat([q, r], dim=-1)
    torch.testing.assert_close(got.double(), cell_in, rtol=1e-5, atol=1e-5)
    assert graph_pool.Pooling("add")(x, index, B).shape == (B, 16)


# ------------------------------------------------------------------------------------------------ the multi-graph fixture
MULTI = os.path.join(ROOT, "tests", "golden", "multigraph_euler")


def fixture_json():
    """the fixture's nodes and edges, from the committed generator the fixture was converted from"""
    import json
    import subprocess
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "g.json")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "tools", "make_multigraph_json.py"), out])
        with open(out) as f:
            return json.load(f)


def node_table(js):
    """id -> (graph_label bytes (b'' when absent), f1 value, dense label)"""
    t = {}
    for nd in js["nodes"]:
        f = {x["name"]: x["value"] for x in nd["features"]}
        t[nd["id"]] = (f.get("graph_label", "").encode(), f["f1"][0], f["label"][0])
    return t


@pytest.mark.parametrize("fixture", ["tiny_euler", "multigraph_euler"])
def test_device_label_list_equals_the_inspected_one(fixture):
    d = os.path.join(ROOT, "tests", "golden", fixture)
    euler_b200.set_graph(euler_b200.Graph.load(d))
    assert ops.graph_labels() == ops.inspect_graph_labels(d)


def test_get_graph_by_label_on_the_fixture_files():
    js = fixture_json()
    table = node_table(js)
    ids = np.asarray(list(table), np.uint64)
    vals = [table[i][0] for i in table]
    euler_b200.set_graph(euler_b200.Graph.load(MULTI))
    labels = ops.graph_labels()
    big = max(set(vals) - {b""}, key=vals.count)              # the graph of 300 nodes
    want_labels = [big, b"7", b"7", b"", b"nope", b"0"]
    idx, val, shape = ops.get_graph_by_label(want_labels)
    want_idx, want_val = restated_by_label(ids, vals, want_labels)
    assert np.array_equal(idx.cpu().numpy(), want_idx) and np.array_equal(val.cpu().numpy(), want_val)
    assert shape == (6, vals.count(big)) and vals.count(big) == 300
    t = torch.tensor([labels.index(x) if x in labels else -1 for x in want_labels], dtype=torch.int32, device="cuda")
    idx2, val2, _ = ops.get_graph_by_label(t)
    assert torch.equal(idx, idx2) and torch.equal(val, val2)
    idx0, val0, shape0 = ops.get_graph_by_label([])
    assert idx0.shape == (0, 2) and val0.numel() == 0 and shape0 == (0, 0)


@pytest.mark.parametrize("mode", ["logits", "q"])
def test_backward_with_an_unsorted_index_gives_the_sorted_rows_bits(mode):
    euler_b200.set_graph(labelled_graph(np.random.RandomState(0), 2)[0])
    rs = np.random.RandomState(300)
    B, index = len(SIZES), batch_index(SIZES)
    N, dim = int(index.numel()), 64
    perm = torch.from_numpy(rs.permutation(N)).cuda()
    order = torch.sort(index[perm].long(), stable=True).indices
    x0, lg0 = cuda(rs.randn(N, dim)), cuda(rs.randn(N))
    q0, g0 = cuda(rs.randn(B, dim) / 8), cuda(rs.randn(B, dim))

    def grads(rows):
        x = x0[rows].clone().requires_grad_()
        w = (q0 if mode == "q" else lg0[rows]).clone().requires_grad_()
        ops.graph_attention_readout(x, index[rows], B, **{mode: w}).backward(g0)
        return x.grad, w.grad

    gx_u, gw_u = grads(perm)                  # unsorted index: walked through the stable sort
    gx_s, gw_s = grads(perm[order])           # the same rows stably sorted by graph
    assert torch.equal(gx_u[order], gx_s)
    assert torch.equal(gw_u[order] if mode == "logits" else gw_u, gw_s)


def test_gin_step_on_the_fixture_matches_a_float64_restatement():
    """One GIN training step as examples/gin/gin.py builds it through euler_estimator's graph_estimator.py, with an
    AttentionPool readout and a Set2SetPool head: sample_graph_label -> get_graph_by_label (node_idx = values, node_graph_idx =
    indices[:, 0], the one-hot label from the column-0 node's dense `label`) -> 2-hop GCNDataFlow without self loops ->
    SparseEmbedding(f1) -> two GINConv layers (scatter_add, mlp((1 + eps) x + aggr), relu) -> fc -> pools -> out_fc ->
    sigmoid cross entropy (base_graph.GraphModel).  Everything in float32 on the device, against float64 on the CPU over
    the same parameters; the blocks are checked against the fixture's edges."""
    from euler_b200.dataflow import GCNDataFlow
    from euler_b200.encoders import SparseEmbedding
    js = fixture_json()
    table = node_table(js)
    adj = {}
    for e in js["edges"]:
        adj.setdefault(e["src"], []).append(e["dst"])
    euler_b200.set_graph(euler_b200.Graph.load(MULTI), rng="minstd", seed=9)
    torch.manual_seed(0)
    B, dims, n_cls = 8, [16, 16, 8], 2
    # ---- graph_estimator.get_train_from_input
    labels = ops.sample_graph_label(B)
    indices, node_idx, _ = ops.get_graph_by_label(labels)
    graph_index = indices[:, 0].to(torch.int32)
    names = ops.graph_labels()
    lab = [names[i] for i in labels.cpu().tolist()]
    want_idx, want_val = restated_by_label(np.asarray(list(table), np.uint64), [table[i][0] for i in table], lab)
    assert np.array_equal(indices.cpu().numpy(), want_idx) and np.array_equal(node_idx.cpu().numpy(), want_val)
    first = node_idx[indices[:, 1] == 0]
    y = ops.get_dense_feature(first, ["label"], [1])[0].view(-1).to(torch.int64)
    assert y.cpu().tolist() == [int(table[int(i)][2]) if int(i) in table else 0 for i in first.cpu().tolist()]
    onehot = torch.nn.functional.one_hot(y, n_cls).to(torch.float32)
    # ---- the model (float32, device)
    flow = GCNDataFlow([[0], [0]], add_self_loops=False)(node_idx)
    emb = SparseEmbedding(3, dims[0], device="cuda")
    with torch.no_grad():
        emb.embeddings.normal_(0, 1)                       # larger than the 2e-4 default, so the comparison means something
    mlps = [graph_pool._glorot_uniform(dims[0], dims[0], "cuda"), graph_pool._glorot_uniform(dims[0], dims[1], "cuda")]
    fc_w, fc_b = graph_pool._glorot_uniform(dims[1], dims[2], "cuda"), torch.full((dims[2],), 0.1, device="cuda")
    ap = graph_pool.AttentionPool()
    s2s = graph_pool.Set2SetPool(dims[2], processing_steps=2, num_layers=1)
    out_fc = graph_pool._glorot_uniform(dims[2], n_cls, "cuda")
    out_fc2 = graph_pool._glorot_uniform(2 * dims[2], n_cls, "cuda")
    eps = 0.0
    x = emb.lookup(flow[0].n_id, "f1", 0)
    for mlp, blk in zip(mlps, flow):
        x_t = ops.gather(x, blk.res_n_id)
        aggr = ops.scatter_add(ops.gather(x, blk.edge_index[1]), blk.edge_index[0], blk.size[0])
        x = torch.relu(((1 + eps) * x_t + aggr) @ mlp)
    node_emb = x @ fc_w + fc_b
    g_att = ap(node_emb, graph_index, B)
    g_s2s = s2s(node_emb, graph_index, B)
    logit, logit2 = g_att @ out_fc, g_s2s @ out_fc2
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    loss = bce(logit, onehot) + bce(logit2, onehot)
    # ---- the blocks list exactly the fixture's out-edges of their targets
    for blk in flow:
        src_ids, tgt_ids = blk.n_id.cpu().numpy(), blk.n_id[blk.res_n_id.long()].cpu().numpy()
        ei = blk.edge_index.cpu().numpy()
        got = sorted(zip(tgt_ids[ei[0]].tolist(), src_ids[ei[1]].tolist()))
        want = sorted((int(t), d) for t in tgt_ids for d in adj.get(int(t), []))
        assert got == want
    # ---- float64 restatement on the CPU
    D = lambda t: t.detach().double().cpu()  # noqa: E731
    x64 = D(emb.embeddings)[torch.tensor([table[i][1] if i in table else 0 for i in flow[0].n_id.cpu().tolist()])]   # absent: default 0
    for mlp, blk in zip(mlps, flow):
        ei = blk.edge_index.long().cpu()
        aggr = torch.zeros(blk.size[0], x64.shape[1], dtype=torch.float64).index_add(0, ei[0], x64[ei[1]])
        x64 = torch.relu(((1 + eps) * x64[blk.res_n_id.long().cpu()] + aggr) @ D(mlp))
    ne64 = x64 @ D(fc_w) + D(fc_b)
    gi = graph_index.cpu()
    att64, _ = readout64(ne64, gi, B, logits=ne64 @ D(ap.gate_nn.kernel))
    lstm = graph_pool.MultiRNNCell([graph_pool.LSTMCell(2 * dims[2], dims[2])]).double()
    lstm.load_state_dict({k: v.double().cpu() for k, v in s2s.lstm.state_dict().items()})
    cell_in, state = torch.zeros(B, 2 * dims[2], dtype=torch.float64), lstm.zero_state(B, "cpu")
    state = [(c.double(), h.double()) for c, h in state]
    for _ in range(2):
        q, state = lstm(cell_in, state)
        r, _ = readout64(ne64, gi, B, q=q)
        cell_in = torch.cat([q, r], dim=-1)
    l64 = bce(att64 @ D(out_fc), D(onehot)) + bce(cell_in @ D(out_fc2), D(onehot))
    torch.testing.assert_close(D(node_emb), ne64, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(D(g_att), att64, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(D(g_s2s), cell_in.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(D(loss), l64.detach(), rtol=1e-5, atol=1e-5)
    loss.backward()                                       # the whole step differentiates through the fused ops
    assert torch.isfinite(emb.embeddings.grad).all() and torch.count_nonzero(ap.gate_nn.kernel.grad) > 0
