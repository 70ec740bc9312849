"""GPU: the fused knowledge-graph step (ops.kg_margin_loss: eu_kg_loss and its backward passes) against the float64 torch
composition of upstream's models (knowledge.composed_kg_loss), and through whole training steps of the five models."""
import numpy as np
import pytest
import torch

import kg_reference as kr

pytestmark = pytest.mark.gpu

MODELS = ('transe', 'transh', 'transr', 'transd', 'distmult')
DIMS = (1, 3, 4, 32, 50, 100, 128, 200)
KS = (1, 5, 64, 4097)
CORRUPTS = ('front', 'tail', 'both')
# TransR's (ent_dim, rel_dim) for each dim: within ent_dim * rel_dim <= 16384, unequal dims included
TRANSR_DIMS = {1: (1, 1), 3: (4, 3), 4: (3, 4), 32: (32, 32), 50: (100, 50), 100: (100, 100), 128: (128, 128), 200: (64, 200)}


@pytest.fixture(scope="module")
def graph():
    import euler_b200
    g = euler_b200.Graph.rmat(1024, 8000, seed=5)
    euler_b200.set_graph(g, rng="minstd", seed=1)
    return g


def _dims(model, dim):
    return TRANSR_DIMS[dim] if model == 'transr' else (dim, dim)


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("corrupt", CORRUPTS)
@pytest.mark.parametrize("l1", (True, False))
@pytest.mark.parametrize("model", MODELS)
def test_against_float64(graph, model, l1, corrupt, dim):
    """scores and loss within 1e-6 of float64; ranks exact; every table's gradient within 1e-5 of float64 autograd, bit-identical
    run to run, zero on untouched rows, and the sparse COO equal to the dense rows"""
    di = DIMS.index(dim)
    K = KS[(di + CORRUPTS.index(corrupt)) % len(KS)]
    ent_dim, rel_dim = _dims(model, dim)
    rng = np.random.RandomState(1000 * di + 10 * MODELS.index(model) + CORRUPTS.index(corrupt) + 5 * l1)
    n_ent, n_rel, B = 60, 8, 7 if K == 4097 else 33
    tabs = kr.tables(model, n_ent, n_rel, ent_dim, rel_dim, rng, offset=di % 2)
    src, dst, neg, rel = kr.ids(rng, B, K, n_ent, n_rel)
    margin = 5.0    # every row active: the gate itself is covered by test_hinge_gate
    kr.check_against_float64(model, tabs, src, dst, neg, rel, l1, corrupt, margin, absolute=dim == 1)


@pytest.mark.parametrize("model", MODELS)
def test_hinge_gate(graph, model):
    """rows with a negative hinge argument get no gradient; a margin that closes every row gives loss 0 and zero gradients"""
    from euler_b200 import ops
    rng = np.random.RandomState(3)
    ent_dim, rel_dim = _dims(model, 32)
    tabs = kr.tables(model, 40, 6, ent_dim, rel_dim, rng)
    src, dst, neg, rel = kr.ids(rng, 50, 5, 40, 6)
    scores = kr.raw(model, tabs, src, dst, neg, rel, True, 'both', 0.0)[0].cpu()
    h = (scores[:, 1:].mean(1) - scores[:, 0]).double()
    margin = float(-h.median()) + 1e-3   # about half the rows active, none at the boundary
    t = [tb.clone().requires_grad_(True) for tb in tabs]
    l, _ = ops.kg_margin_loss(src, dst, neg, rel, t, model, corrupt='both', margin=margin)
    l.backward()
    _, _, loss64, g64, _ = kr.ref64(model, tabs, src, dst, neg, rel, True, 'both', margin)
    assert abs(float(l) - float(loss64)) <= 1e-6 * abs(float(loss64))
    for x, g in zip(t, g64):
        assert kr.rel_err(x.grad, g) <= 1e-5
    t = [tb.clone().requires_grad_(True) for tb in tabs]
    l, _ = ops.kg_margin_loss(src, dst, neg, rel, t, model, corrupt='both', margin=-1000.0)
    l.backward()
    assert float(l) == 0.0 and all(not x.grad.any() for x in t)


def test_hub_negative_exact_on_integer_gradients(graph):
    """a negative repeated 3000 times (1500 per triple, front and tail): one-hot unit rows keep every entry's gradient an
    integer, so the fixed-order sums must equal float64 exactly"""
    from euler_b200 import ops
    dim, n_ent, K, B = 8, 12, 1500, 2
    ent = torch.zeros(n_ent, dim)
    for i in range(n_ent):
        ent[i, i % dim] = 1.0
    relt = torch.zeros(3, dim)
    relt[:, 1] = 1.0
    src, dst = torch.tensor([0, 2]).cuda(), torch.tensor([3, 4]).cuda()
    rel = torch.tensor([0, 1]).cuda()
    neg = torch.full((B, K), 5, dtype=torch.int64).cuda()
    t = [ent.cuda().requires_grad_(True), relt.cuda().requires_grad_(True)]
    l, _ = ops.kg_margin_loss(src, dst, neg, rel, t, 'transe', l1=True, corrupt='both', margin=10.0)
    (l * float(B * 2 * K)).backward()    # cn = 1, cp = -2K: integer entries
    _, _, _, g64, _ = kr.ref64('transe', [ent, relt], src.cpu(), dst.cpu(), neg.cpu(), rel.cpu(), True, 'both', 10.0)
    for x, g in zip(t, g64):
        want = (g * float(B * 2 * K)).numpy()
        assert np.array_equal(x.grad.cpu().numpy(), want.astype(np.float32))
        assert np.abs(want).max() >= 1000


def test_l2_zero_difference_has_zero_gradient(graph):
    """TransH (its rows are not normalised) with s + r - d = 0 exactly: the L2 term's gradient is 0, never NaN"""
    from euler_b200 import ops
    dim = 4
    ent = torch.tensor([[0.5, 0, 0, 0], [1.5, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]])
    relt = torch.tensor([[1.0, 0, 0, 0]])
    hyper = torch.tensor([[0, 0, 0, 1.0]])
    src, dst, rel = torch.tensor([0]).cuda(), torch.tensor([1]).cuda(), torch.tensor([0]).cuda()
    neg = torch.tensor([[2, 3]]).cuda()
    scores = kr.raw('transh', [x.cuda() for x in (ent, relt, hyper)], src, dst, neg, rel, False, 'both', 1.0)[0]
    assert float(scores[0, 0]) == 0.0
    t = [x.cuda().requires_grad_(True) for x in (ent, relt, hyper)]
    l, _ = ops.kg_margin_loss(src, dst, neg, rel, t, 'transh', l1=False, corrupt='both', margin=1.0)
    l.backward()
    _, _, _, g64, _ = kr.ref64('transh', [ent, relt, hyper], src.cpu(), dst.cpu(), neg.cpu(), rel.cpu(), False, 'both', 1.0)
    for x, g in zip(t, g64):
        assert torch.isfinite(x.grad).all()
        assert kr.rel_err(x.grad, g) <= 1e-5
    assert dim == ent.shape[1]


def test_bad_arguments_raise(graph):
    import euler_b200
    from euler_b200 import ops
    rng = np.random.RandomState(9)
    tabs = kr.tables('transe', 20, 4, 8, 8, rng)
    src, dst, neg, rel = kr.ids(rng, 6, 3, 20, 4)
    bad = neg.clone()
    bad[2, 1] = 20
    with pytest.raises(euler_b200.EulerError):
        ops.kg_margin_loss(src, dst, bad, rel, tabs, 'transe')
    with pytest.raises(euler_b200.EulerError):
        ops.kg_margin_loss(src, dst, neg, rel + 4, tabs, 'transe')
    with pytest.raises(euler_b200.EulerError):
        ops.kg_margin_loss(src, dst, neg[:, :0], rel, tabs, 'transe')
    big = kr.tables('transr', 20, 4, 256, 128, rng)
    with pytest.raises(euler_b200.EulerError, match="not supported"):
        ops.kg_margin_loss(src, dst, neg, rel, big, 'transr')
    with pytest.raises(euler_b200.EulerError):
        ops.kg_margin_loss(src, dst, neg, rel, tabs[:1], 'transe')


@pytest.mark.parametrize("model", MODELS)
def test_empty_batch(graph, model):
    from euler_b200 import ops
    rng = np.random.RandomState(2)
    ent_dim, rel_dim = _dims(model, 4)
    t = [x.clone().requires_grad_(True) for x in kr.tables(model, 10, 3, ent_dim, rel_dim, rng)]
    e = torch.zeros(0, dtype=torch.int64).cuda()
    l, m = ops.kg_margin_loss(e, e, e.reshape(0, 2), e, t, model)
    assert torch.isnan(l)
    l.backward()
    assert all(not x.grad.any() for x in t)


def _kg_graph(n_ent=200, n_rel=6, n_edges=3000, seed=0):
    """a synthetic knowledge graph: entities of node type 0, triples of edge type 0 with the relation id in the slot 'id'"""
    import euler_b200
    rng = np.random.RandomState(seed)
    src = rng.randint(0, n_ent, n_edges)
    dst = rng.randint(0, n_ent, n_edges)
    rel = rng.randint(0, n_rel, n_edges)
    order = np.lexsort((dst, src))
    src, dst, rel = src[order], dst[order], rel[order]
    ptr = np.zeros(n_ent + 1, np.int64)
    np.add.at(ptr, src + 1, 1)
    ptr = np.cumsum(ptr)
    g = euler_b200.Graph.from_csr(np.arange(n_ent), ptr, dst, w=np.ones(n_edges, np.float32))
    g.set_edges(src, dst, np.zeros(n_edges, np.int32), dense=rel.reshape(-1, 1).astype(np.float32), dense_names=['id'])
    return g


@pytest.mark.parametrize("cls", ['TransE', 'TransH', 'TransR', 'TransD', 'DistMult'])
def test_training_step_matches_composed(cls):
    """sample_edge -> 'id' -> sample_node -> loss -> backward -> SGD, fused against fused=False within 1e-5"""
    import euler_b200
    from euler_b200 import knowledge
    g = _kg_graph()
    euler_b200.set_graph(g, rng="minstd", seed=3)
    kw = dict(num_negs=4, margin=1.0, corrupt='both', device='cuda')
    dims = (16, 12) if cls == 'TransR' else (16, 16)
    torch.manual_seed(0)
    fused = getattr(knowledge, cls)(0, 0, 199, 5, *dims, **kw)
    composed = getattr(knowledge, cls)(0, 0, 199, 5, *dims, fused=False, **kw)
    composed.load_state_dict(fused.state_dict())
    edges = euler_b200.sample_edge(64, 0)
    rel = euler_b200.get_edge_dense_feature(edges, ['id'], [1])[0]
    assert torch.equal(rel.cpu(), rel.cpu().round()) and float(rel.max()) < 6
    outs = []
    for mdl in (fused, composed):
        euler_b200.seed(77)
        opt = torch.optim.SGD(mdl.parameters(), lr=0.5)
        out = mdl(edges)
        opt.zero_grad()
        out.loss.backward()
        opt.step()
        outs.append(out)
    assert abs(float(outs[0].loss) - float(outs[1].loss)) <= 1e-5 * max(1.0, abs(float(outs[1].loss)))
    assert abs(float(outs[0].metric) - float(outs[1].metric)) <= 1e-5 * max(1.0, abs(float(outs[1].metric)))
    for a, b in zip(outs[0].embedding, outs[1].embedding):
        assert a.shape == b.shape and kr.rel_err(a, b) <= 1e-5
    for (n, p), (_, q) in zip(fused.named_parameters(), composed.named_parameters()):
        assert kr.rel_err(p, q) <= 1e-5, n
