"""GPU: the knowledge-graph step over bfloat16 tables.  For every model, L1 / L2, corruption and width, aligned and offset
tables, the forward (scores, rank, loss, embeddings) and the dense and sparse gradients of bf16 tables are the f32 op's bits
on the widened tables; the sparse gradient is the dense one on the touched rows and repeats run to run.  Refusals write
nothing.  One bf16 train_step equals the f32 step on widened tables (on a synthetic graph and on the converted fixture
tests/golden/kg_euler), and 300 Adam steps of bf16 training track f32 training."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import bf16_reference as bf
import graphs  # noqa: F401  (sys.path)

pytestmark = pytest.mark.gpu
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ['transe', 'transh', 'transr', 'transd', 'distmult']
DIMS = [1, 3, 4, 16, 128, 200, 256, 509, 512]
TRANSR_DIMS = [(1, 1), (3, 3), (4, 4), (16, 16), (128, 128), (512, 32), (32, 512), (257, 63)]
CASES = [(m, d, d) for m in MODELS if m != 'transr' for d in DIMS] + [('transr', e, r) for e, r in TRANSR_DIMS]
N_ENT, N_REL, B = 40, 6, 7


@pytest.fixture(scope="module")
def graph():
    import euler_b200
    g = euler_b200.Graph.rmat(1024, 8000, seed=11)
    euler_b200.set_graph(g, rng="minstd", seed=1)
    return euler_b200


def _bf16(bits, offset=0):
    """uint16 bf16 bits [N, D] on the device; offset puts the data `offset` elements past an 8-byte boundary"""
    bits = np.ascontiguousarray(bits, np.uint16)
    buf = torch.zeros(bits.size + offset, dtype=torch.int16, device="cuda")
    buf[offset:] = torch.from_numpy(bits.reshape(-1).view(np.int16)).cuda()
    return buf.view(torch.bfloat16)[offset:].view(bits.shape)


def _bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _tables(model, ent_dim, rel_dim, rng, offset):
    """(bf16 tables, the same tables widened to f32 and contiguous) in the model's table order"""
    shapes = [(N_ENT, ent_dim), (N_REL, rel_dim)]
    shapes += {'transh': [(N_REL, ent_dim)], 'transr': [(N_REL, ent_dim * rel_dim)],
               'transd': [(N_ENT, ent_dim), (N_REL, rel_dim)]}.get(model, [])
    t16 = [_bf16(bf.round_bits(rng.randn(*s).astype(F32) * F32(0.3)), offset) for s in shapes]
    return t16, [t.float() for t in t16]


def _ids(rng, K):
    d = lambda a: torch.as_tensor(a, dtype=torch.int64).cuda()   # noqa: E731
    return (d(rng.randint(0, N_ENT - 4, size=B)), d(rng.randint(0, N_ENT - 4, size=B)),
            d(rng.randint(0, N_ENT - 4, size=(B, K))), d(rng.randint(0, N_REL - 1, size=B)))   # the last rows untouched


def _slots(model, tabs):
    from euler_b200 import ops
    slots = [None] * 4
    for t, tb in zip(ops._KG_SLOTS[ops.KG_MODELS[model]], tabs):
        slots[t] = tb
    return slots


def _cfg(model, tabs, l1, corrupt, with_emb=True):
    from euler_b200 import ops
    return (ops.KG_MODELS[model], l1, ops.KG_CORRUPT[corrupt], 1.0, tabs[0].shape[1], tabs[1].shape[1], True, with_emb)


def _dense(model, tabs, ids, cfg, scores, g):
    """eu_kg_loss_backward(_dtype): the dense f32 gradient of each table, in the model's order (prefilled with 7s)"""
    from euler_b200 import ops
    src, dst, neg, rel = ids
    slots = _slots(model, tabs)
    p = ops._kg_problem(cfg[0], cfg[1], cfg[2], cfg[3], src, dst, rel, neg, slots, cfg[4], cfg[5])
    grads = [None if t is None else torch.full(tuple(t.shape), 7.0, device="cuda") for t in slots]
    if tabs[0].dtype == torch.bfloat16:
        ops._call("eu_kg_loss_backward_dtype", C.byref(p), 1, g, scores, grads)
    else:
        ops._call("eu_kg_loss_backward", C.byref(p), g, scores, grads)
    return [x for x in grads if x is not None]


def _sparse(model, tabs, ids, cfg, scores, g):
    from euler_b200 import ops
    src, dst, neg, rel = ids
    slots = _slots(model, tabs)
    bufs, counts = ops._raw_kg_sparse_grads(slots, src, dst, rel, neg, cfg, scores, g)
    return [(bufs[t][0][:counts[t]].clone(), bufs[t][1][:counts[t]].clone()) for t in range(4) if slots[t] is not None]


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    x, y = (a.view(torch.int32), b.view(torch.int32)) if a.dtype == torch.float32 else (a, b)
    assert torch.equal(x, y), what


# ------------------------------------------------------------------------------------------------ forward and backward
@pytest.mark.parametrize("model,ent_dim,rel_dim", CASES)
def test_bf16_step_is_the_f32_step_on_widened_tables(graph, model, ent_dim, rel_dim):
    """every l1 x corrupt x offset x K: forward, dense and sparse gradients bit-equal to the f32 op's; sparse = dense on the
    touched rows, zero elsewhere; a second run gives the same bits"""
    from euler_b200 import ops
    for offset in (0, 1, 4):   # 16-byte aligned; scalar path; 8-byte aligned only (bf16's 4-wide path, f32's scalar one)
        rng = np.random.RandomState(ent_dim * 13 + rel_dim + offset + MODELS.index(model) * 1000)
        t16, t32 = _tables(model, ent_dim, rel_dim, rng, offset)
        for K in (1, 5, 300):
            ids = _ids(rng, K)
            src, dst, neg, rel = ids
            for l1 in ((True, False) if model != 'distmult' else (True,)):
                for corrupt in ('front', 'tail', 'both'):
                    what = (model, ent_dim, rel_dim, offset, K, l1, corrupt)
                    cfg = _cfg(model, t16, l1, corrupt)
                    f16 = ops._raw_kg(*_slots(model, t16), src, dst, rel, neg, cfg)
                    f32 = ops._raw_kg(*_slots(model, t32), src, dst, rel, neg, cfg)
                    _same(f16[0], f32[0], what + ("scores",))
                    assert torch.equal(f16[1], f32[1]), what + ("rank",)
                    _same(f16[2], f32[2], what + ("loss",))
                    for e16, e32 in zip(f16[3], f32[3]):
                        _same(e16, e32, what + ("embedding",))
                    g = torch.tensor([0.75], dtype=torch.float32, device="cuda")
                    d16 = _dense(model, t16, ids, cfg, f16[0], g)
                    d32 = _dense(model, t32, ids, cfg, f16[0], g)
                    for k, (a, b) in enumerate(zip(d16, d32)):
                        _same(a, b, what + ("dense", k))
                    s16 = _sparse(model, t16, ids, cfg, f16[0], g)
                    s32 = _sparse(model, t32, ids, cfg, f16[0], g)
                    again = _sparse(model, t16, ids, cfg, f16[0], g)
                    for k, ((r16, v16), (r32, v32), (ra, va), d) in enumerate(zip(s16, s32, again, d16)):
                        assert torch.equal(r16, r32) and torch.equal(r16, ra), what + ("rows", k)
                        _same(v16, v32, what + ("sparse", k))
                        _same(v16, va, what + ("repeat", k))
                        _same(v16, d[r16], what + ("sparse = dense", k))
                        rest = torch.ones(d.shape[0], dtype=torch.bool, device="cuda")
                        rest[r16] = False
                        assert not d[rest].any(), what + ("untouched", k)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_write_nothing(graph):
    from euler_b200 import EulerError, ops
    rng = np.random.RandomState(3)
    for model, e, r in (('transe', 513, 513), ('transr', 129, 128), ('transe', 8, 8)):
        t16, _ = _tables(model, e, r, rng, 0)
        before = [_bits(t) for t in t16]
        src, dst, neg, rel = _ids(rng, 3)
        slots = _slots(model, t16)
        p = ops._kg_problem(ops.KG_MODELS[model], 1, 3, 1.0, src, dst, rel, neg, slots, e, r)
        scores = torch.full((B, 7), 7.0, device="cuda")
        rank = torch.full((B,), 7, dtype=torch.int32, device="cuda")
        loss = torch.full((), 7.0, device="cuda")
        g = torch.ones(1, device="cuda")
        grads = [None if t is None else torch.full(tuple(t.shape), 7.0, device="cuda") for t in slots]
        rows = [None if t is None else torch.full((B * 5,), 7, dtype=torch.int64, device="cuda") for t in slots]
        vals = [None if t is None else torch.full((B * 5, t.shape[1]), 7.0, device="cuda") for t in slots]
        counts = (C.c_int64 * 4)(7, 7, 7, 7)
        # a width past the bounds: EU_ERR_UNSUPPORTED (4); an unknown dtype: EU_ERR_INVALID (1)
        for dt, code in (((1, 4) if e != 8 else (2, 1)), (5, 1), (-1, 1)):
            with pytest.raises(EulerError, match="error %d:" % code):
                ops._call("eu_kg_loss_dtype", C.byref(p), dt, scores, rank, loss, None, None, None)
            with pytest.raises(EulerError, match="error %d:" % code):
                ops._call("eu_kg_loss_backward_dtype", C.byref(p), dt, g, scores, grads)
            with pytest.raises(EulerError, match="error %d:" % code):
                ops._call("eu_kg_loss_backward_sparse_dtype", C.byref(p), dt, g, scores, rows, vals, counts)
        torch.cuda.synchronize()
        assert bool((scores == 7).all()) and bool((rank == 7).all()) and float(loss) == 7.0
        assert all(bool((x == 7).all()) for x in grads + rows + vals if x is not None)
        assert list(counts) == [7, 7, 7, 7]
        for t, b in zip(t16, before):
            np.testing.assert_array_equal(_bits(t), b)
    t16, _ = _tables('transe', 8, 8, rng, 0)
    leaf = [t16[0].clone().requires_grad_(True), t16[1]]
    with pytest.raises(EulerError, match="autograd"):
        ops.kg_margin_loss(*_ids(rng, 3)[:2], _ids(rng, 3)[2], _ids(rng, 3)[3], leaf, 'transe')
    with pytest.raises(EulerError, match="one dtype"):
        ops.kg_margin_loss(*_ids(rng, 3)[:2], _ids(rng, 3)[2], _ids(rng, 3)[3], [t16[0], t16[1].float()], 'transe')


# ------------------------------------------------------------------------------------------------ models
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


@pytest.fixture(scope="module")
def kg_graph():
    import euler_b200
    g = _kg_graph()
    euler_b200.set_graph(g, rng="minstd", seed=3)
    return g


def _pair(cls, node_type=0, edge_type=0, node_max_id=199, edge_max_id=5, dims=None, **kw):
    """(a bf16 model, an f32 model holding its widened tables)"""
    from euler_b200 import knowledge
    dims = dims or ((16, 12) if cls == 'TransR' else (16, 16))
    out = []
    for dt in (torch.bfloat16, torch.float32):
        torch.manual_seed(0)
        out.append(getattr(knowledge, cls)(node_type, edge_type, node_max_id, edge_max_id, *dims, device='cuda',
                                           table_dtype=dt, **kw))
    with torch.no_grad():
        for p16, p32 in zip(out[0].tables(), out[1].tables()):
            p32.copy_(p16.float())
    return out


class _Recorder:
    """wraps an optimizer's apply_sparse to keep copies of the rows and values handed to it"""

    def __init__(self, opt):
        self.opt, self.seen = opt, []
        self.apply_sparse = self._apply

    def _apply(self, params, rows, values):
        self.seen.append(([r.clone() for r in rows], [v.clone() for v in values]))
        return self.opt.apply_sparse(params, rows, values)


def _one_step_equal(m16, m32, edges, seed):
    import euler_b200
    from euler_b200 import optimizers
    o16 = _Recorder(optimizers.get('adam')(m16.tables(), 0.01, seed=9))
    o32 = _Recorder(optimizers.get('adam')(m32.tables(), 0.01))
    outs = []
    for m, o in ((m16, o16), (m32, o32)):
        euler_b200.seed(seed)
        outs.append(m.train_step(edges, o))
    _same(outs[0].loss, outs[1].loss, "loss")
    _same(outs[0].metric, outs[1].metric, "metric")
    for a, b in zip(outs[0].embedding, outs[1].embedding):
        _same(a, b, "embedding")
    (r16, v16), (r32, v32) = o16.seen[0], o32.seen[0]
    assert len(r16) == len(m16.tables())
    for k, (a, b, x, y) in enumerate(zip(r16, r32, v16, v32)):
        assert torch.equal(a, b), k
        _same(x, y, ("values", k))
    for t in m16.tables():
        assert t.dtype == torch.bfloat16 and not t.requires_grad
    return outs


@pytest.mark.parametrize("cls", ['TransE', 'TransH', 'TransR', 'TransD', 'DistMult'])
def test_train_step_bf16_equals_f32_on_widened_tables(kg_graph, cls):
    import euler_b200
    m16, m32 = _pair(cls, num_negs=4, corrupt='both')
    edges = euler_b200.sample_edge(64, 0)
    _one_step_equal(m16, m32, edges, 77)
    # forward of a bf16 model (evaluation): the f32 model's loss, metric and embeddings on the widened tables, no gradient
    with torch.no_grad():
        for p16, p32 in zip(m16.tables(), m32.tables()):
            p32.copy_(p16.float())
    euler_b200.seed(5)
    a = m16(edges)
    euler_b200.seed(5)
    b = m32(edges)
    _same(a.loss, b.loss.detach(), "forward loss")
    _same(a.metric, b.metric, "forward metric")
    assert not a.loss.requires_grad


def test_out_of_range_id_leaves_tables_and_slots_untouched(kg_graph):
    import euler_b200
    from euler_b200 import EulerError, optimizers
    m16, _ = _pair('TransD', num_negs=4)
    opt = optimizers.get('adam')(m16.tables(), 0.01, seed=9)
    euler_b200.seed(1)
    edges = euler_b200.sample_edge(32, 0)
    m16.train_step(edges, opt)   # slots exist from here
    torch.cuda.synchronize()
    before = [_bits(t) for t in m16.tables()] + [_bits(s) for t in m16.tables() for s in opt.state[t].values()
                                                 if torch.is_tensor(s) and s.dim() == 2]
    step = int(opt.sr_step)
    bad = edges.clone()
    bad[3, 0] = 10 ** 6
    with pytest.raises(EulerError, match="outside"):
        m16.train_step(bad, opt)
    torch.cuda.synchronize()
    after = [_bits(t) for t in m16.tables()] + [_bits(s) for t in m16.tables() for s in opt.state[t].values()
                                                if torch.is_tensor(s) and s.dim() == 2]
    assert len(after) == len(before) == 3 * 4
    for a, b in zip(after, before):
        np.testing.assert_array_equal(a, b)
    assert int(opt.sr_step) == step


@pytest.mark.parametrize("cls,lr", [('TransE', 1e-3), ('TransD', 1e-4), ('TransR', 1e-3), ('DistMult', 1e-3)])
def test_training_tracks_f32(kg_graph, cls, lr):
    """300 Adam steps of 512 triples from the same tables and draws: the mean loss of the last 50 bf16 steps lies within 2 %
    of f32 training's.  At lr 1e-3 both learn; TransD runs at upstream's lr 1e-4, whose early updates are a fraction of a
    bf16 ulp, and its bf16 tables still move"""
    import euler_b200
    from euler_b200 import optimizers
    m16, m32 = _pair(cls, num_negs=8, corrupt='both', dims=(32, 16) if cls == 'TransR' else (32, 32))
    o16 = optimizers.get('adam')(m16.tables(), lr, seed=5)
    o32 = optimizers.get('adam')(m32.tables(), lr)
    start = [t.float().clone() for t in m16.tables()]
    l16, l32 = [], []
    for s in range(300):
        euler_b200.seed(2000 + s)
        edges = euler_b200.sample_edge(512, 0)
        for m, o, out in ((m16, o16, l16), (m32, o32, l32)):
            euler_b200.seed(1000 + s)
            out.append(m.train_step(edges, o).loss)
    a = np.array([float(x) for x in l16])
    b = np.array([float(x) for x in l32])
    assert abs(a[-50:].mean() - b[-50:].mean()) <= 0.02 * b[-50:].mean(), (a[-50:].mean(), b[-50:].mean())
    if lr >= 1e-3:
        assert b[:10].mean() - b[-50:].mean() > 0.02, (b[:10].mean(), b[-50:].mean())
        assert a[:10].mean() - a[-50:].mean() > 0.02, (a[:10].mean(), a[-50:].mean())
    moved = np.mean([float((t.float() != s).float().mean()) for t, s in zip(m16.tables(), start)])
    assert moved > 0.2, moved   # the bf16 tables take the small updates


# ------------------------------------------------------------------------------------------------ the converted fixture
def test_fixture_transe_step_bf16_equals_f32():
    """tests/golden/kg_euler through Graph.load: one bf16 TransE train_step equals the f32 step on widened tables"""
    import euler_b200
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "kg.json")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "tools", "make_kg_json.py"), out])
        with open(out) as f:
            js = json.load(f)
    g = euler_b200.Graph.load(os.path.join(ROOT, "tests", "golden", "kg_euler"))
    euler_b200.set_graph(g, rng="minstd", seed=5)
    node_max_id = max(n["id"] for n in js["nodes"])
    edge_max_id = int(max(e["features"][0]["value"][0] for e in js["edges"]))
    m16, m32 = _pair('TransE', 'train', 'train', node_max_id, edge_max_id, dims=(16, 16), num_negs=3, corrupt='both')
    edges = euler_b200.sample_edge(48, 'train')
    outs = _one_step_equal(m16, m32, edges, 11)
    assert np.isfinite(float(outs[0].loss))
