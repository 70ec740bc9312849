"""GPU: eu_sample_n_with_types against the reference engine's per-row loop (bit for bit, with the stream continuing into the next
sample_node), its Philox draws, its refusals, sample_node_with_src, and the solution package against float64 replays of the
same ids."""
import copy
import json
import os

import numpy as np
import pytest
import torch

import cases
import graphs
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
INT32_MIN = -2 ** 31
REF_RECORD = os.path.join(graphs.GOLDEN, "sample_n_with_types_ref.json")


class RefOutputs(cases.RefOutputs):
    """cases.RefOutputs over this module's own record, tests/golden/sample_n_with_types_ref.json: the reference's outputs,
    checked live where oracle/_ref is built (EU_RECORD_REF=1 writes them instead), their digests elsewhere"""

    def __init__(self, name):
        self.name, self.live = name, po.have_ref()
        self.rec = json.load(open(REF_RECORD)).get(name, {}) if os.path.exists(REF_RECORD) else {}

    def want(self, key, fn, values=False):
        if not self.live:
            assert key in self.rec, "no recorded reference output %s/%s" % (self.name, key)
            r = self.rec[key]
            return np.asarray(r["values"], r["dtype"]) if values else cases._recorded(r)
        out = fn()
        r = {"values": np.asarray(out).tolist(), "dtype": np.asarray(out).dtype.str} if values else cases._digests(out)
        if os.environ.get("EU_RECORD_REF"):
            allrec = json.load(open(REF_RECORD)) if os.path.exists(REF_RECORD) else {}
            allrec.setdefault(self.name, {})[key] = r
            with open(REF_RECORD, "w") as f:
                json.dump(allrec, f, indent=0, sort_keys=True)
        else:
            assert self.rec.get(key) == r, "the reference's %s/%s differs from %s" % (self.name, key, REF_RECORD)
        return out


def _eb():
    import euler_b200
    return euler_b200


def _ref_rows(sample, types, count, next_type, next_count):
    """the reference engine's loop (euler/core/kernels/sample_n_with_types_op.cc): SampleNode({t}, count) row by row, then
    the next SampleNode({next_type}, next_count) on the same stream; `sample(types, count)` is one SampleNode call"""
    rows = np.stack([np.asarray(sample([int(t)], count), np.uint64) for t in types]).astype(np.int64)
    return rows.reshape(len(types), count), np.asarray(sample([next_type], next_count), np.uint64).astype(np.int64)


def _device(types, count, next_type, next_count):
    eb = _eb()
    got = eb.sample_n_with_types(count, torch.as_tensor(types, dtype=torch.int32, device="cuda"))
    return got.cpu().numpy(), eb.sample_node(next_count, [next_type]).cpu().numpy()


# ---------------------------------------------------------------------------- bit-exact draws
GRID = [(n, count, s) for n in (1, 7, 4097) for count in (1, 5, 64) for s in (1, 77, 2024)]


def _grid_types(n):
    return np.random.RandomState(n).randint(0, 3, size=n).astype(np.int32)


def ref_random_graph_rows():
    """the reference on a 3-type random graph (CPU only: EU_RECORD_REF=1 records it without a GPU): its node-map order and,
    for every case of GRID, the rows and the next SampleNode({1}, 40)"""
    ref = RefOutputs("sample_n_with_types_random_graph")
    g = graphs.random_graph(seed=41, n=3000, T=2, avg_deg=4, n_node_types=3)
    rg = graphs.ref_graph(g) if ref.live else None
    order = ref.want("map_order", lambda: rg.node_ids_in_map_order(), values=True)
    wants = {(n, count, s): ref.want("n%d_count%d_seed%d" % (n, count, s),
                                     lambda: (rg.seed(s), _ref_rows(rg.sample_node, _grid_types(n), count, 1, 40))[1])
             for n, count, s in GRID}
    return g, order, wants


def test_rows_equal_the_reference_loop_on_a_three_type_graph():
    """a 3-type random graph built into the reference and onto the device (the reference's node-map order as sampler order):
    n in {1, 7, 4097} x count in {1, 5, 64} x three seeds, and the sample_node after each call"""
    g, order, wants = ref_random_graph_rows()
    cases.CudaBackend(g, order)
    eb = _eb()
    for n, count, s in GRID:
        eb.seed(s)
        got, nxt = _device(_grid_types(n), count, 1, 40)
        key = "n=%d count=%d seed=%d" % (n, count, s)
        cases.eq(got, wants[(n, count, s)][0], "rows " + key)
        cases.eq(nxt, wants[(n, count, s)][1], "next sample_node " + key)
        assert eb.context().draws() == 2 * n * count + 2 * 40


def test_rows_equal_the_oracle_loop_on_the_heterogeneous_rmat():
    """the device R-MAT with 3 node types against the C restatement's SampleNode (pinned to the reference by
    test_oracle_vs_ref), row by row on one engine"""
    eb = _eb()
    n_nodes, E, T, NT = 30000, 240000, 5, 3
    gr = eb.Graph.rmat_hetero(n_nodes, E, T, NT)
    ex = gr.export()
    og = po.OracleGraph(ex["ids"], ex["node_type"], ex["node_w"], T, ex["grp_ptr"], ex["nbr"], ex["cum_w"], ex["grp_cum"], None)
    og.build_node_sampler(np.arange(n_nodes), NT)
    eb.set_graph(gr)
    for n, count in ((1, 64), (7, 5), (4097, 1), (4097, 64)):
        types = np.random.RandomState(count).randint(0, NT, size=n).astype(np.int32)
        for s in (3, 5, 8):
            rng = po.Rng(s)
            want = _ref_rows(lambda t, c: og.sample_node(t, c, rng), types, count, 2, 33)
            eb.seed(s)
            got, nxt = _device(types, count, 2, 33)
            cases.eq(got, want[0], "rmat rows n=%d count=%d seed=%d" % (n, count, s))
            cases.eq(nxt, want[1], "rmat next sample_node n=%d count=%d seed=%d" % (n, count, s))


FIXTURE_CASES = [(n, count, s) for n, count in ((1, 64), (7, 5), (7, 64), (4097, 1)) for s in (11, 12345, 99)]
FIXTURES = {"tiny_euler": 2, "multigraph_euler": 3}


def _fixture_types(fixture, n, count):
    return np.random.RandomState(n + count).randint(0, FIXTURES[fixture], size=n).astype(np.int32)


def ref_fixture_rows(fixture):
    """the reference's loop on its own load of a committed fixture (CPU only, like ref_random_graph_rows), keyed by the order
    in which this machine lists the partitions; only the cases recorded for that order (EU_RECORD_REF=1 records them)"""
    d = os.path.join(graphs.GOLDEN, fixture)
    ref = RefOutputs("sample_n_with_types_" + fixture)
    order = cases.partition_order(d)
    rg = po.RefGraph.load(d) if ref.live else None
    wants = {}
    for n, count, s in FIXTURE_CASES:
        key = "%s n%d_count%d_seed%d" % (order, n, count, s)
        if key in ref.rec or (ref.live and os.environ.get("EU_RECORD_REF")):
            wants[(n, count, s)] = ref.want(key, lambda: (rg.seed(s), _ref_rows(rg.sample_node, _fixture_types(fixture, n, count),
                                                                               count, 0, 21))[1])
    return wants


@pytest.mark.parametrize("fixture", sorted(FIXTURES))
def test_rows_equal_the_reference_loop_on_loaded_fixtures(fixture):
    """Graph.load of the committed fixtures: always against sample_node row by row (which
    test_sample_node_on_a_loaded_graph_follows_the_reference_map_order pins to the reference on these directories), and
    against the reference's own load of the same directory where its output is recorded for this listing order"""
    wants = ref_fixture_rows(fixture)
    eb = _eb()
    eb.set_graph(eb.Graph.load(os.path.join(graphs.GOLDEN, fixture)), rng="minstd", seed=1)
    for n, count, s in FIXTURE_CASES:
        types, key = _fixture_types(fixture, n, count), "n=%d count=%d seed=%d" % (n, count, s)
        eb.seed(s)
        got, nxt = _device(types, count, 0, 21)
        eb.seed(s)
        loop = _ref_rows(lambda t, c: eb.sample_node(c, t).cpu().numpy(), types, count, 0, 21)
        cases.eq(got, loop[0], "%s rows vs sample_node %s" % (fixture, key))
        cases.eq(nxt, loop[1], "%s next vs sample_node %s" % (fixture, key))
        if (n, count, s) in wants:
            cases.eq(got, wants[(n, count, s)][0], "%s rows %s" % (fixture, key))
            cases.eq(nxt, wants[(n, count, s)][1], "%s next sample_node %s" % (fixture, key))


# ---------------------------------------------------------------------------- philox
def test_philox_draws_follow_the_node_weights():
    from scipy import stats
    eb = _eb()
    g = graphs.random_graph(seed=43, n=240, T=1, n_node_types=3)
    eb.set_graph(graphs.cuda_graph(g), rng="philox", seed=9)
    types = torch.as_tensor(np.random.RandomState(1).randint(0, 3, size=6000), dtype=torch.int32, device="cuda")
    a = eb.sample_n_with_types(64, types)
    b = eb.sample_n_with_types(64, types)
    assert not torch.equal(a, b), "the call counter keys each call's draws"
    draws, tt = a.cpu().numpy(), types.cpu().numpy()
    for t in range(3):
        ids, w = g["ids"][g["node_type"] == t].astype(np.int64), g["node_w"][g["node_type"] == t].astype(np.float64)
        d = draws[tt == t].reshape(-1)
        assert np.isin(d, ids).all(), "type %d: a draw of another type" % t
        obs = np.array([(d == i).sum() for i in ids], np.float64)
        p = stats.chisquare(obs, w / w.sum() * d.size).pvalue
        assert p > 1e-4, "type %d: chi-square p = %g" % (t, p)


# ---------------------------------------------------------------------------- refusals
def test_refusals_leave_out_and_the_engine_untouched():
    eb = _eb()
    from euler_b200 import ops
    g = graphs.random_graph(seed=45, n=500, T=1, n_node_types=3)
    g["node_w"][g["node_type"] == 2] = 0.0                                       # type 2 has total weight 0
    eb.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    eb.seed(5)
    want_next = eb.sample_node(30, [1]).cpu().numpy()
    absent = int(eb.get_node_type(torch.as_tensor([10 ** 12], device="cuda"))[0])
    assert absent == INT32_MIN
    for bad, what in (([0, absent, 1], "not a node"), ([0, 2, 1], "total weight 0"), ([0, 3], "outside"), ([-1, 0], "outside")):
        types = torch.as_tensor(bad, dtype=torch.int32, device="cuda")
        out = torch.full((len(bad), 6), -7, dtype=torch.int64, device="cuda")
        eb.seed(5)
        with pytest.raises(eb.EulerError, match=what):
            ops._call("eu_sample_n_with_types", types, types.numel(), 6, out)
        assert (out == -7).all(), "a refused call wrote out (%s)" % what
        assert eb.context().draws() == 0
        cases.eq(eb.sample_node(30, [1]).cpu().numpy(), want_next, "sample_node after a refusal (%s)" % what)
    with pytest.raises(eb.EulerError, match="not a node"):
        eb.sample_node_with_src([g["ids"][0], 10 ** 12], 3)
    for n, count in ((0, 5), (4, 0)):
        eb.seed(5)
        out = eb.sample_n_with_types(count, torch.zeros(n, dtype=torch.int32, device="cuda"))
        assert out.shape == (n, count) and eb.context().draws() == 0
        cases.eq(eb.sample_node(30, [1]).cpu().numpy(), want_next, "sample_node after n=%d count=%d" % (n, count))


def test_sample_node_with_src():
    eb = _eb()
    g = graphs.random_graph(seed=47, n=2000, T=1, n_node_types=3, id_stride=7)
    eb.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    src = torch.as_tensor(g["ids"][np.random.RandomState(2).randint(0, 2000, size=513)].astype(np.int64), device="cuda")
    eb.seed(8)
    got = eb.sample_node_with_src(src, 5)
    eb.seed(8)
    want = eb.sample_n_with_types(5, eb.get_node_type(src))
    assert got.shape == (513, 5) and torch.equal(got, want)
    src_t = eb.get_node_type(src)
    cases.eq(eb.get_node_type(got.reshape(-1)).reshape(513, 5).cpu().numpy(), src_t[:, None].expand(-1, 5).cpu().numpy(),
             "every draw has its source's type")
    cases.eq(src_t.cpu().numpy(), g["node_type"][(src.cpu().numpy() - 1) // 7], "get_node_type")


# ---------------------------------------------------------------------------- the solutions against float64
MAX_ID, FEAT = 3000, 16


@pytest.fixture
def feature_graph():
    eb = _eb()
    g = graphs.random_graph(seed=49, n=MAX_ID, T=1, avg_deg=5, feat_dim=FEAT)
    eb.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    return g


class _Table(torch.nn.Module):
    """float64 node-encoder rows looked up by id (the dense slot of every id the replay reads)"""

    def __init__(self, ids):
        super().__init__()
        from euler_b200 import ops
        self.ids = torch.unique(torch.cat([i.reshape(-1).cuda() for i in ids])).cpu()
        self.rows = ops.get_dense_feature(self.ids, [0], [FEAT])[0].double().cpu()

    def forward(self, x):
        return self.rows[torch.searchsorted(self.ids, x.reshape(-1).cpu())].reshape(tuple(x.shape) + (FEAT,))


class _Recorder:
    """wraps a callable and keeps what each call returned"""

    def __init__(self, fn):
        self.fn, self.out = fn, []

    def __call__(self, *a):
        r = self.fn(*a)
        self.out.append(r)
        return r


def _record_sage(enc):
    """records every sample tree enc draws in the float32 pass"""
    enc.sample = _Recorder(enc.sample)
    return enc


def _sage64(enc, trees, table):
    """enc in float64 on the CPU: each call aggregates the next recorded tree, rows from the table"""
    rec = enc.__dict__.pop('sample')
    e64 = copy.deepcopy(enc).double().cpu()
    enc.sample = rec
    e64.fused, e64._node_encoder = False, table
    queue = [[s.cpu() for s in t] for t in trees]

    class Replay(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.enc = e64

        def forward(self, ids):
            return self.enc.agg(ids.cpu(), queue.pop(0))
    return Replay(), e64


def _gcn64(enc, table):
    """enc in float64 on the CPU over the same (deterministic) get_multi_hop_neighbor"""
    from euler_b200 import encoders, ops
    e64 = encoders.GCNEncoder(enc.metapath, enc.dims[-1], 'gcn', feature_idx=0, feature_dim=FEAT, fused=False).double()
    e64.load_state_dict({k: v.double().cpu() for k, v in enc.state_dict().items()})
    e64._node_encoder = table

    class Replay(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.enc = e64

        def forward(self, ids):
            nodes, adjs = ops.get_multi_hop_neighbor(ids.cuda(), self.enc.metapath)
            out = self.enc._layers([table(n) for n in nodes], [tuple(a.cpu() for a in adj) for adj in adjs])
            return out.reshape(tuple(ids.shape) + (self.enc.dims[-1],))
    return Replay(), e64


def _close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(np.abs(b).max() if b.size else 0.0, 1e-30)
    assert np.abs(a - b).max() <= 1e-5 * scale, "%s: max error %g, largest entry %g" % (what, np.abs(a - b).max(), scale)


def _grads_close(pairs):
    for name, p32, p64 in pairs:
        assert p32.grad is not None and p64.grad is not None, name
        _close(p32.grad.cpu().numpy(), p64.grad.numpy(), "grad " + name)


def _cosine_pos_neg(e, p, n):
    from euler_b200 import solution
    cos = solution.CosineLogits()
    return cos(e, p).transpose(1, 2), cos(e, n).transpose(1, 2)


@pytest.mark.parametrize("kind", ("sage", "gcn", "sage_cosine"))
def test_unsupervise_solution_against_float64(feature_graph, kind):
    from euler_b200 import encoders, solution
    torch.manual_seed(0)
    if kind == "gcn":
        mk = lambda: encoders.GCNEncoder([[0], [0]], 8, 'gcn', feature_idx=0, feature_dim=FEAT, device="cuda")  # noqa: E731
    else:
        mk = lambda: _record_sage(encoders.SageEncoder([[0], [0]], [4, 3], 8, 'mean', feature_idx=0, feature_dim=FEAT,  # noqa: E731
                                                       max_id=MAX_ID, device="cuda"))
    target, context = mk(), mk()
    pos_fn = _Recorder(solution.SamplePosWithTypes([0], 2, max_id=MAX_ID))
    neg_fn = _Recorder(solution.SampleNegWithTypes(0, 5))
    kw = dict(logit_fn=_cosine_pos_neg) if kind == "sage_cosine" else {}
    sol = solution.UnsuperviseSolution(target, context, pos_fn, neg_fn, metric_name='mrr', **kw)
    inputs = torch.as_tensor(np.random.RandomState(3).randint(1, MAX_ID + 1, size=256), device="cuda")
    _eb().seed(21)
    emb, loss, _, metric = sol(inputs)
    loss.backward()
    pos, negs = pos_fn.out[0], neg_fn.out[0]
    if kind == "gcn":
        nodes = [n for ids in (inputs, pos, negs) for n in _eb().get_multi_hop_neighbor(ids, [[0], [0]])[0]]
        table = _Table(nodes)
        (t64, te), (c64, ce) = _gcn64(target, table), _gcn64(context, table)
    else:
        table = _Table([s for e in (target, context) for t in e.sample.out for s in t])
        (t64, te), (c64, ce) = _sage64(target, target.sample.out, table), _sage64(context, context.sample.out, table)
    sol64 = solution.UnsuperviseSolution(t64, c64, lambda _: pos.cpu(), lambda _: negs.cpu(), metric_name='mrr', **kw)
    emb64, loss64, _, metric64 = sol64(inputs.cpu())
    loss64.backward()
    _close(loss.item(), loss64.item(), "loss")
    _close(metric.item(), metric64.item(), "metric")
    _close(emb.detach().cpu().numpy(), emb64.detach().numpy(), "embedding")
    _grads_close([("target." + k, p, dict(te.named_parameters())[k]) for k, p in target.named_parameters()] +
                 [("context." + k, p, dict(ce.named_parameters())[k]) for k, p in context.named_parameters()])


def test_supervise_solution_against_float64(feature_graph):
    from euler_b200 import encoders, solution
    torch.manual_seed(1)
    enc = _record_sage(encoders.SageEncoder([[0], [0]], [4, 3], 8, 'mean', feature_idx=0, feature_dim=FEAT, max_id=MAX_ID,
                                            device="cuda"))
    logits = solution.DenseLogits(3, dim=8, device="cuda")
    sol = solution.SuperviseSolution(solution.GetLabelFromFea(0, 3), enc, logits)
    inputs = torch.as_tensor(np.random.RandomState(4).randint(1, MAX_ID + 1, size=300), device="cuda")
    emb, loss, name, metric = sol(inputs)
    loss.backward()
    table = _Table([s for t in enc.sample.out for s in t])
    e64, ee = _sage64(enc, enc.sample.out, table)
    l64 = copy.deepcopy(logits).double().cpu()
    sol64 = solution.SuperviseSolution(lambda x: solution.GetLabelFromFea(0, 3)(x.cuda()).double().cpu(), e64, l64)
    emb64, loss64, _, metric64 = sol64(inputs.cpu())
    loss64.backward()
    assert name == 'f1'
    _close(loss.item(), loss64.item(), "loss")
    _close(metric.item(), metric64.item(), "f1")
    _close(emb.detach().cpu().numpy(), emb64.detach().numpy(), "embedding")
    _grads_close([("enc." + k, p, dict(ee.named_parameters())[k]) for k, p in enc.named_parameters()] +
                 [("logits.out_fc.weight", logits.out_fc.weight, l64.out_fc.weight)])


def test_supervise_solution_equals_supervise_model(feature_graph):
    """SuperviseSolution(GetLabelFromFea, encoder, DenseLogits) and supervised.SuperviseModel give the same loss bits"""
    from euler_b200 import encoders, solution
    from euler_b200.supervised import SuperviseModel
    torch.manual_seed(2)
    enc = encoders.SageEncoder([[0], [0]], [5, 2], 8, 'mean', feature_idx=0, feature_dim=FEAT, max_id=MAX_ID, device="cuda")

    class Model(SuperviseModel):
        def __init__(self):
            super().__init__(0, 3, dim=8, device="cuda")

        def embed(self, n_id):
            return enc(n_id)

    model = Model()
    logits = solution.DenseLogits(3, dim=8, device="cuda")
    with torch.no_grad():
        logits.out_fc.weight.copy_(model.out_fc.weight)
    sol = solution.SuperviseSolution(solution.GetLabelFromFea(0, 3), enc, logits)
    inputs = torch.as_tensor(np.random.RandomState(5).randint(1, MAX_ID + 1, size=512), device="cuda")
    _eb().seed(31)
    a = model(inputs)
    _eb().seed(31)
    b = sol(inputs)
    assert torch.equal(a[0], b[0]) and a[2] == b[2]
    cases.eq(a[1].detach().cpu().numpy(), b[1].detach().cpu().numpy(), "loss bits")
    cases.eq(a[3].cpu().numpy(), b[3].cpu().numpy(), "f1 bits")
