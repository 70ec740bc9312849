"""GPU: the whole-graph adjacency (ops.graph_adjacency, eu_graph_adjacency) row by row against get_full_neighbor's listing
with ids mapped to engine rows, graph_node_ids / graph_node_rows, and GCNEncoder.infer / GenieEncoder.infer against
forward on the same ids."""
import numpy as np
import pytest
import torch

import graphs

pytestmark = pytest.mark.gpu

N = 500
FEAT = 8
ABSENT = 10 ** 9        # ids from here on are not nodes


def _graph(seed=3, T=3, id_stride=1, hub=0, absent=0):
    """graphs.random_graph with T edge types, rows without entries and multi-edges; absent > 0 replaces every 7th listed
    id by one of `absent` ids that are not nodes"""
    g = graphs.random_graph(seed=seed, n=N, T=T, avg_deg=4, id_stride=id_stride, hub=hub, empty_frac=0.2, feat_dim=FEAT)
    if absent:
        rng = np.random.RandomState(seed)
        g["nbr"][::7] = (ABSENT + rng.randint(0, absent, size=len(g["nbr"][::7]))).astype(np.uint64)
    return g


def _install(g):
    import euler_b200
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], grp_cum=g["grp_cum"] if g["T"] > 1 else None,
                                   feat=g["feat"], feat_slot_dims=[FEAT])
    euler_b200.set_graph(gr, rng="minstd", seed=1)
    return gr


def _check_rows(types, rows):
    """graph_adjacency(types, rows) against get_full_neighbor of the rows' nodes, bit for bit; returns its outputs"""
    import euler_b200
    node_ids = euler_b200.graph_node_ids()
    n = node_ids.numel()
    indptr, cols, w, extra = euler_b200.graph_adjacency(types, rows=rows, weights=True)
    sel = torch.arange(rows.start, rows.stop, device="cuda") if isinstance(rows, range) else torch.as_tensor(rows, device="cuda")
    inside = (sel >= 0) & (sel < n)
    listed = torch.where(inside, node_ids[sel.clamp(0, max(n - 1, 0))], ABSENT - 1)   # a row outside the graph lists nothing
    fp, fids, fw, _ = euler_b200.get_full_neighbor(listed, types)
    assert torch.equal(indptr, fp)
    row_of = {int(v): r for r, v in enumerate(node_ids.tolist())}
    firsts = {}
    want = [row_of[v] if v in row_of else n + firsts.setdefault(v, len(firsts)) for v in fids.tolist()]
    assert cols.tolist() == want
    assert extra.tolist() == list(firsts)
    assert w.cpu().numpy().tobytes() == fw.cpu().numpy().tobytes()
    return indptr, cols, w, extra


@pytest.mark.parametrize("types", ([0], [2, 0], [1, 1, 0], [0, 1, 2], [5]))
@pytest.mark.parametrize("id_stride", (1, 3))
def test_adjacency_equals_the_listing(types, id_stride):
    g = _graph(id_stride=id_stride)
    _install(g)
    indptr, cols, _, extra = _check_rows(types, range(N))
    lens = np.diff(indptr.cpu().numpy())
    assert extra.numel() == 0 and (types == [5] or ((lens == 0).any() and lens.max() > 0))
    import euler_b200
    assert torch.equal(euler_b200.graph_node_ids().cpu(), torch.as_tensor(g["ids"].astype(np.int64)))


def test_hub_row_and_absent_ids():
    import euler_b200
    g = _graph(hub=20000, absent=40)
    _install(g)
    indptr, cols, _, extra = _check_rows([0, 1, 2], range(N))
    assert np.diff(indptr.cpu().numpy()).max() >= 20000
    assert 0 < extra.numel() <= 40 and (extra >= ABSENT).all()
    ids = torch.as_tensor(np.r_[g["ids"][[5, 0, 99]].astype(np.int64), ABSENT - 3], device="cuda")
    assert euler_b200.graph_node_rows(ids).tolist() == [5, 0, 99, -1]
    _check_rows([2, 0], torch.as_tensor([7, -1, 3, 7, N + 4, 0], device="cuda"))      # a row list, rows outside the graph
    _check_rows([1], torch.zeros(0, dtype=torch.int64, device="cuda"))


def test_loaded_graph_uses_the_id_table(tiny_dir):
    import euler_b200
    gr = euler_b200.Graph.load(tiny_dir)
    euler_b200.set_graph(gr, rng="minstd", seed=1)
    for types in ([0], [1, 0], [0, 1]):
        _check_rows(types, range(gr.num_nodes))


def test_chunked_builds_concatenate_to_the_one_shot_build():
    import euler_b200
    _install(_graph(absent=25))
    n = N
    indptr, cols, w, extra = euler_b200.graph_adjacency([1, 0], weights=True)
    ip, ids, ws, off = [torch.zeros(1, dtype=torch.int64, device="cuda")], [], [], 0
    for r0, r1 in ((0, 130), (130, 131), (131, 131), (131, 400), (400, n)):
        p, c, cw, x = _check_rows([1, 0], range(r0, r1))
        ip.append(p[1:] + off)
        off += int(p[-1])
        ids.append(torch.where(c < n, c, -1 - x[(c - n).clamp(min=0)]) if x.numel() else c)   # absent: the id, by its chunk's numbering
        ws.append(cw)
    assert extra.numel() > 0
    one = torch.where(cols < n, cols, -1 - extra[(cols - n).clamp(min=0)])
    assert torch.equal(torch.cat(ip), indptr) and torch.equal(torch.cat(ids), one) and torch.equal(torch.cat(ws), w)


def test_argument_errors():
    import euler_b200
    _install(_graph())
    for rows in (range(-1, 3), range(0, N + 1), range(0, 10, 2), range(5, 3)):
        with pytest.raises(euler_b200.EulerError):
            euler_b200.graph_adjacency([0], rows=rows)


# ---------------------------------------------------------------------------- inference against forward
def _encoder(cls, metapath, aggregator, use_residual):
    torch.manual_seed(0)
    return cls(metapath, 8, aggregator, feature_idx="feat0", feature_dim=FEAT, use_residual=use_residual, head_num=2,
               device="cuda")


def _close(a, b, what):
    assert a.shape == b.shape, what
    assert (a.double() - b.double()).abs().max() <= 1e-5 * b.abs().max().clamp(min=1e-3), what


def _ids(g):
    """every node once in a shuffled order, a repeat, an isolated node and two ids that are not nodes"""
    lens = np.diff(g["grp_ptr"]).reshape(N, g["T"]).sum(1)
    rng = np.random.RandomState(1)
    ids = g["ids"][rng.permutation(N)].astype(np.int64)
    return torch.as_tensor(np.r_[ids, ids[:3], g["ids"][np.argmin(lens)], ABSENT + 1, ABSENT - 5], device="cuda")


@pytest.mark.parametrize("use_residual", (False, True))
@pytest.mark.parametrize("metapath", ([[0], [0]], [[0], [1]], [[0, 1], [1]], [[2]], [[0], [1], [0]]))
@pytest.mark.parametrize("aggregator", ("gcn", "mean", "attention"))
def test_gcn_infer_equals_forward(aggregator, metapath, use_residual):
    from euler_b200.encoders import GCNEncoder
    g = _graph(absent=30)
    _install(g)
    enc = _encoder(GCNEncoder, metapath, aggregator, use_residual)
    ids = _ids(g)
    with torch.no_grad():
        want = torch.cat([enc(ids[a:a + 128]) for a in range(0, ids.numel(), 128)])
    got = enc.infer(ids)
    _close(got, want, "infer(ids)")
    every = enc.infer(chunk_rows=97)
    order = torch.as_tensor(g["ids"].astype(np.int64), device="cuda")
    with torch.no_grad():
        _close(every, torch.cat([enc(order[a:a + 128]) for a in range(0, N, 128)]), "infer()")


def test_infer_bits_do_not_depend_on_chunk_rows():
    from euler_b200.encoders import GCNEncoder, GenieEncoder
    g = _graph(absent=30)
    _install(g)
    ids = _ids(g)
    for cls, agg in ((GCNEncoder, "gcn"), (GCNEncoder, "mean"), (GCNEncoder, "attention"), (GenieEncoder, "attention")):
        enc = _encoder(cls, [[0], [1]], agg, True)
        a, b = enc.infer(ids, chunk_rows=1 << 20), enc.infer(ids, chunk_rows=61)
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), (cls.__name__, agg)


@pytest.mark.parametrize("use_residual", (False, True))
@pytest.mark.parametrize("aggregator", ("gcn", "attention"))
def test_genie_infer_equals_forward(aggregator, use_residual):
    from euler_b200.encoders import GenieEncoder
    g = _graph(absent=30)
    _install(g)
    enc = _encoder(GenieEncoder, [[0], [1]], aggregator, use_residual)
    ids = _ids(g)
    with torch.no_grad():
        want = torch.cat([enc(ids[a:a + 128]) for a in range(0, ids.numel(), 128)])
    _close(enc.infer(ids), want, "genie infer(ids)")
    assert enc.infer().shape == (N, 8)


def test_absent_ids_are_encoded_as_forward_encodes_them():
    """forward on an id that is not a node: its node-encoder row (zero features), then every layer with no neighbours"""
    from euler_b200.encoders import GCNEncoder
    g = _graph(absent=30)
    _install(g)
    enc = _encoder(GCNEncoder, [[0], [0]], "gcn", True)
    ids = torch.as_tensor([ABSENT + 1, ABSENT - 5, ABSENT + 1], device="cuda")
    with torch.no_grad():
        want = enc(ids)
        h = enc.node_encoder(ids)
        assert not h.any()                       # no features, no id embedding: the row is zero
        for a in enc.aggregators:
            empty = (torch.zeros(4, dtype=torch.int64, device="cuda"), torch.zeros(0, dtype=torch.int64, device="cuda"))
            h = h + a((h, h, empty))
    _close(want, h, "forward's own meaning")
    _close(enc.infer(ids), want, "infer")
