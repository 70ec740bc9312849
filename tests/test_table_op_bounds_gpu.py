"""GPU: the fused id-table ops at the top of the ranges they accept, where code that narrower shapes never reach runs:
  - the KG step (ops.kg_margin_loss) at dims 256 .. 512, a lane's float4 chunks 2 and 3, and TransR at the edges of
    ent_dim * rel_dim <= 16384; dims of 513 and larger matrices are refused;
  - the skip-gram step (ops.skipgram_xent_loss) across k_sg_fwd's split between the target chunks kept in registers and
    those read again from memory (dim > 512);
  - ShallowEncoder (ops.shallow_encode) with all 8 dense and 8 sparse slots, 9 tables through one backward pass, and a row of
    exactly EU_SHALLOW_MAX_WIDTH columns; a wider row or a 9th slot is refused;
  - the pooled op (ops.shallow_encode_pool) on narrow rows and long segments, where the launcher widens the lane groups
    until a block's cached graph rows fit in 48 KB, up to count 512, on f32 and bfloat16 graphs.
Each against float64, or against a float32 restatement of the op's defined order where the result is bit-exact."""
import ctypes as C

import numpy as np
import pytest
import torch

import embedding_reference as er
import kg_reference as kr
import skipgram_reference as sr

pytestmark = pytest.mark.gpu

UNSUPPORTED = 4   # EU_ERR_UNSUPPORTED


def _status(sym, *args):
    """the status of one raw library call on this thread's Context (tensors passed as their data pointers)"""
    from euler_b200 import _lib, ops
    return getattr(_lib.load(), sym)(ops._ctx_on_stream()._h, *[ops._arg(a) for a in args])


@pytest.fixture(scope="module")
def rmat_graph():
    import euler_b200
    return euler_b200.Graph.rmat(1024, 8000, seed=5)


@pytest.fixture
def rmat(rmat_graph):
    import euler_b200
    euler_b200.set_graph(rmat_graph, rng="minstd", seed=1)


# ---------------------------------------------------------------------------- the KG step, dims 129 .. 512
KG_MODELS = ('transe', 'transh', 'transr', 'transd', 'distmult')
KG_DIMS = (256, 257, 384, 509, 512)
# TransR's (ent_dim, rel_dim) in place of each dim: the edges of ent_dim * rel_dim <= 16384 with rows up to 512 wide
KG_TRANSR = {256: (128, 128), 257: (257, 63), 384: (32, 512), 509: (509, 32), 512: (512, 32)}


def _margin_all_active(model, tabs, src, dst, neg, rel, l1):
    """a margin at which every triple's hinge argument is at least the largest |score|: every row reaches the gradient, and
    the loss is not a small difference of large scores (wide L1 rows score in the hundreds)"""
    scores = kr.raw(model, tabs, src, dst, neg, rel, l1, 'both', 0.0)[0].double()
    h = scores[:, 1:].mean(1) - scores[:, 0]
    return max(0.0, float(-h.min())) + float(scores.abs().max())


@pytest.mark.parametrize("dim", KG_DIMS)
@pytest.mark.parametrize("l1", (True, False))
@pytest.mark.parametrize("model", KG_MODELS)
def test_kg_wide_rows_against_float64(rmat, model, l1, dim):
    """test_kg_gpu.test_against_float64's checks at dims whose rows fill a lane's chunks 2 and 3 (columns 256 .. 511)"""
    di = KG_DIMS.index(dim)
    offset = (di + l1) % 2              # each dim aligned under one norm, one float off (scalar loads) under the other
    K = (1, 300)[(di // 2 + l1) % 2]    # 300 negatives span two blocks of kKgTile
    ent_dim, rel_dim = KG_TRANSR[dim] if model == 'transr' else (dim, dim)
    rng = np.random.RandomState(100 * di + 10 * KG_MODELS.index(model) + l1)
    n_ent, n_rel = 60, 8
    B = 16 if K == 1 else 2 if model == 'transr' else 4   # TransR's float64 side holds a matrix per negative
    tabs = kr.tables(model, n_ent, n_rel, ent_dim, rel_dim, rng, offset=offset)
    if l1 and model != 'distmult':
        # sign() jumps at 0, where f32 and f64 may round a difference (a + r) - c to opposite sides: with ~10^5 differences
        # per case some land within an ulp of 0 on random rows.  Relation rows of +-1 and entity rows near one row (TransH's
        # scaled to unit length, as the other models' mapped rows are) keep every difference near +-r_j: for these seeds
        # none lies within 1e-6 of 0, far above the rounding of either side.  (Rows much closer than this make the
        # relation-side gradients a cancellation of f32 terms and cost them their 1e-5.)
        tabs[1].copy_(tabs[1].sign())
        for t in [tabs[0]] + ([tabs[2]] if model == 'transd' else []):
            t.copy_(t[:1] + 0.15 * t)
        if model == 'transh':
            tabs[0].copy_(tabs[0] / tabs[0][0].norm())
    src, dst, neg, rel = kr.ids(rng, B, K, n_ent, n_rel)
    margin = _margin_all_active(model, tabs, src, dst, neg, rel, l1)
    kr.check_against_float64(model, tabs, src, dst, neg, rel, l1, 'both', margin)


def _unit_rows(rng, n, dim):
    """rows of 64 or 256 entries +-1 and zeros elsewhere: the norm is 8 or 16, so every normalised entry is exact"""
    t = np.zeros((n, dim), np.float32)
    for i in range(n):
        k = (64, 256)[i % 2]
        t[i, rng.choice(dim, k, replace=False)] = rng.choice([-1.0, 1.0], k)
    return t


@pytest.mark.parametrize("model", ('transe', 'distmult'))
def test_kg_dyadic_scores_equal_float64_at_512(rmat, model):
    """L1 TransE and DistMult scores over normalised rows of +-1/8 and +-1/16: every term and partial sum is exact, so the
    scores equal float64's bit for bit"""
    dim, n_ent, n_rel, B, K = 512, 60, 8, 4, 300
    rng = np.random.RandomState(17 + len(model))
    src, dst, neg, rel = kr.ids(rng, B, K, n_ent, n_rel)
    for offset in (0, 1):
        tabs = []
        for rows in (_unit_rows(rng, n_ent, dim), _unit_rows(rng, n_rel, dim)):
            v = torch.zeros(rows.size + offset)
            v[offset:] = torch.from_numpy(rows.reshape(-1))
            tabs.append(v.cuda()[offset:].view(rows.shape))
        scores = kr.raw(model, tabs, src, dst, neg, rel, True, 'both', 1.0)[0]
        host = [x.cpu() for x in tabs + [src, dst, neg, rel]]
        pos64, neg64 = kr.ref64(model, host[:2], *host[2:], True, 'both', 1.0)[:2]
        want = torch.cat([pos64, neg64], 1).detach().float().numpy()
        assert scores.cpu().numpy().tobytes() == want.tobytes(), (model, offset)
        assert np.abs(want).max() > 0


@pytest.mark.parametrize("model,ent_dim,rel_dim", [('transe', 513, 513), ('distmult', 513, 513), ('transr', 513, 8),
                                                   ('transr', 8, 513), ('transr', 129, 128)])
def test_kg_refuses_dims_past_its_bounds(rmat, model, ent_dim, rel_dim):
    """a dim of 513, or a TransR matrix of more than 16384 entries: EU_ERR_UNSUPPORTED from every entry point before it
    writes anything"""
    import euler_b200
    from euler_b200 import ops
    rng = np.random.RandomState(ent_dim + rel_dim)
    B, K = 6, 3
    tabs = kr.tables(model, 20, 4, ent_dim, rel_dim, rng)
    src, dst, neg, rel = kr.ids(rng, B, K, 20, 4)
    leaves = [t.clone().requires_grad_(True) for t in tabs]
    with pytest.raises(euler_b200.EulerError, match="not supported"):
        ops.kg_margin_loss(src, dst, neg, rel, leaves, model)
    assert all(x.grad is None and torch.equal(x, t) for x, t in zip(leaves, tabs))
    slots = [None] * 4
    for t, tb in zip(ops._KG_SLOTS[ops.KG_MODELS[model]], tabs):
        slots[t] = tb
    p = ops._kg_problem(ops.KG_MODELS[model], 1, ops.KG_CORRUPT['both'], 1.0, src, dst, rel, neg, slots, ent_dim, rel_dim)
    scores = torch.full((B, 1 + 2 * K), 7.0, device="cuda")
    rank = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    loss = torch.full((), 7.0, device="cuda")
    embs = [torch.full((B, rel_dim), 7.0, device="cuda") for _ in range(3)]
    grads = [None if t is None else torch.full_like(t, 7.0) for t in slots]
    rows = [None if t is None else torch.full((B * (K + 2),), 7, dtype=torch.int64, device="cuda") for t in slots]
    counts = (C.c_int64 * 4)(7, 7, 7, 7)
    g = torch.ones(1, device="cuda")
    assert _status("eu_kg_loss", C.byref(p), scores, rank, loss, *embs) == UNSUPPORTED
    assert _status("eu_kg_loss_backward", C.byref(p), g, scores, grads) == UNSUPPORTED
    assert _status("eu_kg_loss_backward_sparse", C.byref(p), g, scores, rows, grads, counts) == UNSUPPORTED
    torch.cuda.synchronize()
    for out in [scores, rank, loss] + embs + [x for x in grads + rows if x is not None]:
        assert (out == 7).all()
    assert list(counts) == [7, 7, 7, 7]


# ---------------------------------------------------------------------------- the skip-gram step across its register split
# k_sg_fwd keeps a lane's first 4 target chunks in registers and reads chunks 4 .. from memory: with 32 lanes, dim > 512
SG_DIMS = (255, 256, 257, 384, 509, 512, 513, 1024, 1031, 2048)
SG_PK = ((1, 5), (3, 20))


@pytest.mark.parametrize("P,K", SG_PK)
@pytest.mark.parametrize("dim", SG_DIMS)
def test_skipgram_forward_dyadic_bit_exact(rmat, dim, P, K):
    """dyadic tables: the logits equal skipgram_reference.logits_f32's fixed order (and float64, every partial sum being
    exact), the ranks top_k's, the loss float64's within 1e-6"""
    rng = np.random.RandomState(dim * 31 + P * 7 + K)
    n_rows, B = 300, 65
    src, pos, negs = sr.pair_ids(rng, B, P, K, n_rows)
    ctx = sr.context_ids(pos, negs)
    for off in (0, 1):   # both tables aligned (float4 loads when dim % 4 == 0), or both one float off
        target, context = sr.device_table(n_rows, dim, rng, off), sr.device_table(n_rows, dim, rng, off)
        logits, rank, loss = sr.device_forward(src, pos, negs, target, context)
        tn, cn = target.cpu().numpy(), context.cpu().numpy()
        x = logits.cpu().numpy()
        head = sr.logits_f32(tn, cn, src[:4], ctx[:4])   # the literal order on the first rows (it is slow in Python)
        assert x[:4].tobytes() == head.tobytes(), (dim, P, K, off)
        x64 = sr.forward64(tn, cn, src, ctx, P)[0]
        assert x.tobytes() == x64.astype(np.float32).tobytes(), (dim, P, K, off)
        assert np.array_equal(rank.cpu().numpy(), sr.rank_top_k_literal(x[:, :P], x[:, P:]))
        ref = sr.loss64(x64, P)
        assert abs(float(loss) - ref) <= 1e-6 * abs(ref)


@pytest.mark.parametrize("P,K", SG_PK)
@pytest.mark.parametrize("dim", SG_DIMS)
def test_skipgram_gradients_across_the_register_split(rmat, dim, P, K):
    """separate and shared tables: loss within 1e-6 and gradients within 1e-5 of float64, bit-identical run to run, zero
    on untouched rows, and the sparse gradient equal to the dense one"""
    rng = np.random.RandomState(dim + 10 * K + P)
    n_rows, B = 500, 200
    src, pos, negs = sr.pair_ids(rng, B, P, K, n_rows)
    negs[:, 0] = 7                                   # a hub negative
    ctx = sr.context_ids(pos, negs)
    for off in (0, 1):
        target = sr.device_table(n_rows, dim, rng, off, dyadic=False)
        context = sr.device_table(n_rows, dim, rng, off, dyadic=False)
        for shared in (False, True):
            what = (dim, P, K, off, shared)
            tn = target.cpu().numpy()
            cn = tn if shared else context.cpu().numpy()
            wt, wc = sr.grads64(tn, cn, src, ctx, P)
            want = [wt + wc] if shared else [wt, wc]
            loss64 = sr.forward64(tn, cn, src, ctx, P)[1]
            a = sr.device_grads(src, pos, negs, target, context, shared)
            b = sr.device_grads(src, pos, negs, target, context, shared)
            s = sr.device_grads(src, pos, negs, target, context, shared, sparse=True)
            assert abs(float(a[0].detach()) - loss64) <= 1e-6 * abs(loss64), what
            for k, w in enumerate(want):
                got, again, sp = a[1 + k], b[1 + k], s[1 + k]
                assert got.cpu().numpy().tobytes() == again.cpu().numpy().tobytes(), what + (k,)
                g = got.cpu().numpy()
                assert np.abs(g - w).max() <= 1e-5 * np.abs(w).max(), what + (k,)
                assert (g[np.abs(w).sum(1) == 0] == 0).all(), what + (k,)
                assert sp.is_sparse and sp.to_dense().cpu().numpy().tobytes() == g.tobytes(), what + (k,)


# ---------------------------------------------------------------------------- ShallowEncoder at its slot and width bounds
N_NODES, N_ID = 600, 1000                      # graph ids 1 .. 600; an id table of N_ID rows
DENSE_DIMS = (1, 3, 3, 4, 5, 8, 12, 16)        # the dense slots feat0 .. feat7
SLOT_ROWS = (1000, 60, 300, 20, 5000, 100, 40, 2000)   # the table rows of uint64 slots u64_0 .. u64_7; the last is the default
ABSENT = (0, 650, 999)                         # ids the graph does not hold, all inside the id table


def _lens_mixed(rng, n):   # 0 (the default), 1, ordinary, and a few bags of more than 256 values
    k = rng.choice([0, 1, 2, 3, 5, 9], size=n, p=[0.3, 0.2, 0.2, 0.15, 0.1, 0.05])
    k[rng.choice(n, size=3, replace=False)] = [257, 300, 700]
    return k


def _slot_graph(g, feat_dtype="float32", feat=None):
    import euler_b200
    return euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                     node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"] if feat is None else feat,
                                     feat_slot_dims=list(DENSE_DIMS), u64_ptr=g["u64_ptr"], u64_val=g["u64_val"],
                                     n_u64_slots=g["S"], feat_dtype=feat_dtype)


@pytest.fixture(scope="module")
def slots():
    """one graph with 8 dense and 8 uint64 slots (slot 0 with bags past 256 values, slot 3 mostly empty)"""
    lens = [_lens_mixed] + [lambda rng, n, s=s: rng.randint(0, 2 + s % 4, size=n) for s in range(1, 8)]
    lens[3] = lambda rng, n: (rng.rand(n) < 0.2).astype(np.int64)
    vals = [lambda rng, k, m=m: rng.randint(0, m - 1, size=k) for m in SLOT_ROWS]
    g = er.slot_graph(21, N_NODES, lens, vals, feat_dim=sum(DENSE_DIMS))
    rng = np.random.RandomState(6)
    nodes = np.concatenate([g["ids"][rng.randint(0, N_NODES, size=700)], ABSENT, g["ids"][:5], g["ids"][:5]]).astype(np.int64)
    return dict(g=g, gr=_slot_graph(g), nodes=nodes)


@pytest.fixture
def slot_env(slots):
    import euler_b200
    euler_b200.set_graph(slots["gr"], rng="minstd", seed=1)
    return slots


def _table(n_rows, dim, seed, offset=0):
    """a random f32 table on the device whose data pointer is `offset` floats past a 16-byte boundary"""
    t = torch.randn(n_rows * dim + offset, generator=torch.Generator().manual_seed(seed)).cuda()
    return t[offset:].view(n_rows, dim)


COMBS = ("sum", "mean", "sqrtn")
# every dense slot, padded (feat0, feat1, feat3, feat6, feat7), clipped (feat2, feat5) or as stored (feat4)
DENSE8 = [("feat0", 1), ("feat1", 4), ("feat2", 2), ("feat3", 6), ("feat4", 5), ("feat5", 7), ("feat6", 20), ("feat7", 16)]


def _sparse8(dims, unknown):
    """8 sparse slots of the given dims, combiners mixed, some tables one float off; unknown: the last one names no slot"""
    out = [("u64_%d" % s, _table(SLOT_ROWS[s], d, 10 + s, offset=int(s % 3 == 2)), SLOT_ROWS[s] - 1, COMBS[s % 3])
           for s, d in enumerate(dims)]
    if unknown:
        out[7] = ("no_such_slot", _table(20, dims[7], 30), 7, "sqrtn")
    return out


def _grads_f64(env, nodes, gn, id_table, id_cols, sparse, cols):
    """float64 gradients of the id table (grad_out gn's columns id_cols) and of each sparse slot (columns cols[k]) and the
    sums of their terms' magnitudes, from the graph's bags"""
    import euler_b200
    g = env["g"]
    w, m = np.zeros(id_table.shape), np.zeros(id_table.shape)
    np.add.at(w, nodes, gn[:, id_cols])
    np.add.at(m, nodes, np.abs(gn[:, id_cols]))
    want, mag, touched = [w], [m], [np.unique(nodes)]
    for (n, t, dv, c), col in zip(sparse, cols):
        bl = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, euler_b200.get_graph().sparse_feature_id(n), dv)
        want.append(er.grad_f64(gn[:, col], bl, t.shape[0], c))
        mag.append(er.grad_f64(np.abs(gn[:, col]), bl, t.shape[0], c))
        touched.append(np.unique(np.concatenate([np.asarray(b, np.int64) for b in bl])))
    return want, mag, touched


def _check_grads(run, want, mag, touched):
    """run(sparse_grad) -> the tables' gradients: dense within 1e-5 of float64 and bit-identical run to run; sparse coalesced,
    one entry per distinct row the table's entries touch (the count the backward reads back), equal to the dense rows"""
    g1, g2, gs = run(False), run(False), run(True)
    assert len(g1) == len(want)
    for t in range(len(g1)):
        assert torch.equal(g1[t], g2[t]), t
        got = g1[t].cpu().numpy()
        err = np.abs(got - want[t])
        assert (err <= 1e-5 * mag[t] + 1e-7).all(), (t, float((err / (mag[t] + 1e-30)).max()))
        assert not got[mag[t].sum(1) == 0].any(), t
        s = gs[t]
        assert s.is_sparse and s.is_coalesced() and s._nnz() == len(touched[t]), (t, s._nnz(), len(touched[t]))
        assert np.array_equal(s.indices()[0].cpu().numpy(), touched[t]), t
        assert torch.equal(s.to_dense(), g1[t]), t


def _leaves(id_table, sparse):
    leaves = [id_table.detach().clone().requires_grad_(True)] + [t.detach().clone().requires_grad_(True) for _, t, _, _ in sparse]
    return leaves, [(n, leaf, dv, c) for (n, _, dv, c), leaf in zip(sparse, leaves[1:])]


def test_shallow_concat_eight_dense_and_eight_sparse_slots(slot_env):
    """an id table, 8 dense and 8 sparse slots (one unknown): the forward equals the composition's bits; the 9 tables'
    gradients through one backward pass"""
    import euler_b200
    nodes = slot_env["nodes"]
    id_table = _table(N_ID, 16, 1)
    sparse = _sparse8((4, 3, 16, 1, 8, 5, 12, 2), unknown=True)
    out = euler_b200.shallow_encode(nodes, id_table, DENSE8, sparse, "concat")
    idp, dp, sp = er.composed_parts(nodes, id_table, DENSE8, sparse)
    want = torch.cat(idp + dp + sp, 1)
    assert out.shape == want.shape == (len(nodes), 16 + 61 + 51)
    assert out.cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
    grad = torch.randn(out.shape, generator=torch.Generator().manual_seed(9)).cuda()
    cols, c0 = [], 16 + sum(d for _, d in DENSE8)
    for _, t, _, _ in sparse:
        cols.append(slice(c0, c0 + t.shape[1]))
        c0 += t.shape[1]
    want, mag, touched = _grads_f64(slot_env, nodes, grad.cpu().double().numpy(), id_table, slice(0, 16), sparse, cols)

    def run(sparse_grad):
        leaves, sp = _leaves(id_table, sparse)
        res = euler_b200.shallow_encode(nodes, leaves[0], DENSE8, sp, "concat", sparse_grad=sparse_grad)
        return torch.autograd.grad(res, leaves, grad)
    _check_grads(run, want, mag, touched)


def test_shallow_add_eight_sparse_slots(slot_env):
    """'add' over an id table and 8 sparse slots of one dim, with 8 dense slots beside: the sum and the dense part equal
    the composition's bits (id + sparse_0 + .. + sparse_7, left to right); the 9 tables' gradients"""
    import euler_b200
    nodes, dim = slot_env["nodes"], 12
    id_table = _table(N_ID, dim, 2, offset=1)
    sparse = _sparse8((dim,) * 8, unknown=False)
    emb, feats = euler_b200.shallow_encode(nodes, id_table, DENSE8, sparse, "add")
    idp, dp, sp = er.composed_parts(nodes, id_table, DENSE8, sparse)
    want = idp[0]
    for x in sp:
        want = want + x
    assert emb.cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
    assert feats.cpu().numpy().tobytes() == torch.cat(dp, 1).cpu().numpy().tobytes()
    grad = torch.randn(emb.shape, generator=torch.Generator().manual_seed(8)).cuda()
    cols = [slice(0, dim)] * 8
    want, mag, touched = _grads_f64(slot_env, nodes, grad.cpu().double().numpy(), id_table, slice(0, dim), sparse, cols)

    def run(sparse_grad):
        leaves, sp = _leaves(id_table, sparse)
        res = euler_b200.shallow_encode(nodes, leaves[0], DENSE8, sp, "add", sparse_grad=sparse_grad)
        return torch.autograd.grad(res[0], leaves, grad)
    _check_grads(run, want, mag, touched)


def test_shallow_row_of_16384_columns_and_the_refusals(slot_env):
    """a concat row of exactly EU_SHALLOW_MAX_WIDTH = 16384 columns (an id table and three sparse slots of 4096) equals the
    composition's bits; 16385 columns, or a 9th dense or sparse slot, are refused before the output is written"""
    import euler_b200
    from euler_b200 import _lib
    nodes = slot_env["nodes"][-40:]
    id_table = _table(N_ID, 4096, 3)
    sparse = [("u64_%d" % s, _table(SLOT_ROWS[s], 4096, 20 + s), SLOT_ROWS[s] - 1, COMBS[s % 3]) for s in (1, 3, 6)]
    assert _lib.SHALLOW_MAX_WIDTH == 16384
    out = euler_b200.shallow_encode(nodes, id_table, [], sparse, "concat")
    idp, _, sp = er.composed_parts(nodes, id_table, [], sparse)
    assert out.shape == (40, 16384)
    assert out.cpu().numpy().tobytes() == torch.cat(idp + sp, 1).cpu().numpy().tobytes()

    nd = torch.as_tensor(nodes, device="cuda")
    buf = torch.full((40 * 16385,), 7.0, device="cuda")
    with pytest.raises(euler_b200.EulerError, match="columns"):
        euler_b200.shallow_encode(nodes, id_table, [("feat0", 1)], sparse, "concat")
    p = er.shallow_problem(nd, id_table, [("feat0", 1)], sparse)
    assert _status("eu_shallow_encode", C.byref(p), buf, None) == UNSUPPORTED
    small = [("u64_1", _table(SLOT_ROWS[1], 2, 5), SLOT_ROWS[1] - 1, "sum")]
    with pytest.raises(euler_b200.EulerError, match="at most"):
        euler_b200.shallow_encode(nodes, None, DENSE8 + [("feat0", 1)], small, "concat")
    with pytest.raises(euler_b200.EulerError, match="at most"):
        euler_b200.shallow_encode(nodes, None, [], small * 9, "concat")
    for field in ("n_dense", "n_sparse"):
        p = er.shallow_problem(nd, None, DENSE8, small * 8)
        setattr(p, field, 9)
        assert _status("eu_shallow_encode", C.byref(p), buf, None) == UNSUPPORTED, field
    torch.cuda.synchronize()
    assert (buf == 7.0).all()


# ---------------------------------------------------------------------------- the pooled op with widened lane groups
POOL_M = 12800   # divisible by every count below
# (id dim, count): narrow rows (every part at most 3 wide: one lane per group) whose segments' graph rows overflow 48 KB per
# block, so the launcher widens the groups to 2 (count 25), 4 (64), 16 (200) and 32 lanes (512); and count 512 at dim 128
POOL_CASES = [(1, 25), (3, 64), (1, 200), (3, 512), (128, 512)]


@pytest.fixture(scope="module")
def pool_nodes(slots):
    g = slots["g"]
    rng = np.random.RandomState(12)
    nodes = g["ids"][rng.randint(0, N_NODES, size=POOL_M)].astype(np.int64)
    nodes[rng.choice(POOL_M, size=400, replace=False)] = rng.choice(ABSENT, size=400)
    nodes[:N_NODES] = g["ids"]                       # every node, the long bags included
    return nodes


def _pool_inputs(id_dim):
    dim = 3 if id_dim < 8 else id_dim
    return _table(N_ID, id_dim, 4, offset=1), [("feat1", 3)], [("u64_2", _table(SLOT_ROWS[2], dim, 5), SLOT_ROWS[2] - 1, "mean")]


@pytest.mark.parametrize("id_dim,count", POOL_CASES)
def test_pool_widened_groups_bit_exact_and_gradients(slot_env, pool_nodes, id_dim, count):
    """the forward equals embedding_reference.pool_f32 (each column added left to right from the segment's first row, mean
    divided once by fl(count)) over shallow_encode's rows, sum and mean; the gradients within 1e-5 of float64 and
    bit-identical run to run"""
    import euler_b200
    nodes = pool_nodes
    id_table, dense, sparse = _pool_inputs(id_dim)
    rows = euler_b200.shallow_encode(nodes, id_table, dense, sparse, "concat")
    W = rows.shape[1]
    for pool in ("sum", "mean"):
        out = euler_b200.shallow_encode_pool(nodes, count, id_table, dense, sparse, pool)
        want = er.pool_f32(rows, count, pool)
        assert out.shape == want.shape and out.cpu().numpy().tobytes() == want.tobytes(), (id_dim, count, pool)
        grad = torch.randn(POOL_M // count, W, generator=torch.Generator().manual_seed(count)).cuda()
        gn = np.repeat(grad.cpu().double().numpy(), count, axis=0) / (count if pool == "mean" else 1)
        w, m, touched = _grads_f64(slot_env, nodes, gn, id_table, slice(0, id_dim), sparse, [slice(id_dim + 3, W)])

        def run(sparse_grad):
            leaves, sp = _leaves(id_table, sparse)
            res = euler_b200.shallow_encode_pool(nodes, count, leaves[0], dense, sp, pool, sparse_grad=sparse_grad)
            return torch.autograd.grad(res, leaves, grad)
        _check_grads(run, w, m, touched)


def test_pool_widened_groups_on_a_bfloat16_graph(slots, pool_nodes):
    """k_shallow_pool<__nv_bfloat16> with widened groups: the bits of the f32 graph of the bf16 graph's exported table"""
    import euler_b200
    gb = _slot_graph(slots["g"], "bfloat16")
    gf = _slot_graph(slots["g"], "float32", gb.export()["feat"])
    id_table, dense, sparse = _pool_inputs(1)
    dense = [("feat1", 3), ("feat5", 7), ("feat6", 20)]   # bf16 rows read as stored, clipped and padded
    for count in (200, 512):
        for pool in ("sum", "mean"):
            outs = []
            for graph in (gb, gf):
                euler_b200.set_graph(graph, rng="minstd", seed=1)
                outs.append(euler_b200.shallow_encode_pool(pool_nodes, count, id_table, dense, sparse, pool))
            assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), (count, pool)
    assert not np.array_equal(gb.export()["feat"], slots["g"]["feat"])   # the bf16 table is rounded: the two graphs differ from the input
