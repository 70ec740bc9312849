"""gather, scatter_add / scatter_max / scatter_mean, get_dense_feature and the fused SAGE mean / add (mp_ops.cu) against the
float32 restatements of tests/mp_ops_reference.py, at every launch choice, on inputs with ±0.0, ±inf, NaN, subnormals, values
below scatter_max's -1e9 floor and exact ties.

Bit for bit wherever the kernel fixes the order of its arithmetic (NaN compared by position: a NaN made on the GPU and one made
on the CPU differ in bits).  The unsorted scatter path adds with atomics in no fixed order: add and mean are compared with
float64 within RTOL * sum|u| (plus what the atomics' flush of subnormals loses), with inf and NaN at the same places; max is
exact there too, but order-free among equal zeros.

Which case reaches each instantiation:
  k_gather / k_scatter_sorted / k_scatter_atomic  VEC: D % 4 == 0, "aligned" layout (G = 1 at D = 4 up to 32 at D >= 128);
                                                  scalar: every other D, and every D in the "in+4" / "out+4" layouts
  k_feature       VEC: test_dense_feature on [64] (dim 64, 68), [4, 128] (slot 0 dim 4, 8; slot 1 dim 128, 132), unknown slots
                  scalar: every other dim, every slot of [3, 8, 130] (offsets 3 and 11), every "out+4" call
  k_sage_mean     <1,true> 128; <2,true> 256; <1,false> 4, 64, 100; <2,false> 132, 200; <4,false> 260, 512;
                  <8,false> 516, 1024 (test_fused_sage_widths, dim == feat_dim on one slot)
  k_sage_mean_generic  3, 130, 1028 (test_fused_sage_widths); dim != feat_dim, "out+4", multi-slot graphs
                  (test_fused_sage_generic_cases); count 0 (test_fused_sage_count_zero)
  k_sage_classify / k_sage_broadcast<true|false>  test_fused_sage_dedup_rows (2^17 rows: dims 64 and 128 aligned for VEC, dim 3
                  and dim 64 "out+4" for the scalar broadcast)"""
import numpy as np
import pytest
import torch

import cases
import graphs
import mp_ops_reference as ref

pytestmark = pytest.mark.gpu
RTOL = 1e-5   # the unsorted atomic path: relative to sum|u| of the entry
WIDTHS = (1, 2, 3, 4, 5, 31, 32, 33, 64, 127, 128, 129, 256, 1024, 1030)
LAYOUTS = ("aligned", "in+4", "out+4")
SIZE = 64     # scatter output rows: 0-2, 10, 11, 30 and 50-63 get no edge; row 20 about half of them
HUB, EMPTY = 20, (0, 1, 2, 10, 11, 30)
ONLY_NEG0, NEG0_AMONG_NEG, BOTH_ZEROS = 5, 6, 7   # rows whose every column is: all -0.0; -0.0 and negatives; -0.0, +0.0, negatives
SPECIALS = np.asarray([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1e-40, -1e-40, -2e9, -1e9, -1e10, 3.5, -3.5],
                      np.float32)


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def eb():
    import euler_b200
    g = graphs.random_graph(seed=51, n=10, T=1)
    euler_b200.set_graph(graphs.cuda_graph(g))
    return euler_b200


def _call(name, *args):
    from euler_b200 import _lib, ops
    _lib.check(getattr(_lib.load(), name)(ops._ctx_on_stream()._h, *args))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _shifted(a):
    """a device copy of f32 array a starting 4 bytes past a 16-byte boundary: (the buffer to keep alive, the pointer)"""
    a = np.ascontiguousarray(a, np.float32).reshape(-1)
    buf = torch.full((a.size + 1,), float("nan"), dtype=torch.float32, device="cuda")
    buf[1:] = _dev(a)
    return buf, buf.data_ptr() + 4


def _raw(name, shape, layout, ins, *args):
    """entry point `name`(*args) with the f32 input array ins, if any, (its device pointer spliced where args holds None) and
    an output f32[shape] appended, both placed per layout ("aligned"; "in+4": the input 4 bytes past a 16-byte boundary;
    "out+4": the output so)"""
    keep, p_in = _shifted(ins) if layout == "in+4" else (None, None)
    if p_in is None and ins is not None:
        keep = _dev(np.asarray(ins, np.float32))
        p_in = keep.data_ptr()
    n = int(np.prod(shape))
    out, p_out = _shifted(np.full(n, np.nan, np.float32)) if layout == "out+4" else (None, None)
    if p_out is None:
        out = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
        p_out = out.data_ptr()
    _call(name, *[p_in if a is None else a for a in args], p_out)
    return (out[1:] if layout == "out+4" else out).cpu().numpy().reshape(shape)


def eq_nan(got, want, what):
    """bits everywhere, except that a NaN only has to be a NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), "%s: NaN at %s, want %s" % (what, np.argwhere(np.isnan(got))[:4], np.argwhere(nan)[:4])
    cases.eq(np.where(nan, np.float32(0), got), np.where(nan, np.float32(0), want), what)


def atomic_tol(u, idx, size):
    """what an order-free float32 sum may miss per entry: RTOL * sum|u|, plus 2^-126 for each update and each partial sum the
    atomics flush from a subnormal to zero"""
    n = ref.counts(idx, size).astype(np.float64)
    return RTOL * ref.sum_abs64(u, idx, size) + 2 * n * 2.0 ** -126


def close64(got, want64, tol, what):
    """inf and NaN where the float64 result has them, every finite entry within tol of it, or within the least subnormal
    (the rounding of a result that underflows)"""
    got = np.asarray(got, np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(want64)), what + ": NaN positions"
    inf = np.isinf(want64)
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], want64[inf]), what + ": inf positions"
    fin = np.isfinite(want64)
    err = np.abs(got[fin].astype(np.float64) - want64[fin])
    tol = tol[fin] + 2.0 ** -149
    k = (err - tol).argmax()
    assert (err <= tol).all(), "%s: error %g > %g at %s" % (what, err[k], tol[k], np.argwhere(fin)[k])


# ------------------------------------------------------------------ inputs
def _sorted_index(rs, E):
    rows = np.setdiff1d(np.arange(3, 50), EMPTY)
    fixed = np.repeat([ONLY_NEG0, NEG0_AMONG_NEG, BOTH_ZEROS], 3)
    return np.sort(np.r_[np.full(E // 2, HUB), fixed, rs.choice(rows, E - E // 2 - len(fixed))]).astype(np.int32)


def _updates(rs, idx, D):
    """randn over 20 binades, 30% quantised to halves (exact ties), 6% special values outside the hub row; rows ONLY_NEG0,
    NEG0_AMONG_NEG and BOTH_ZEROS as named (their first edge -0.0 and BOTH_ZEROS's second +0.0, in every column)"""
    E = len(idx)
    u = (rs.randn(E, D) * np.exp2(rs.randint(-10, 10, size=(E, D)))).astype(np.float32)
    q = rs.rand(E, D) < 0.3
    u[q] = rs.randint(-3, 4, size=q.sum()) * np.float32(0.5)
    m = (rs.rand(E, D) < 0.06) & (idx != HUB)[:, None]
    u[m] = rs.choice(SPECIALS, m.sum())
    for r in (ONLY_NEG0, NEG0_AMONG_NEG, BOTH_ZEROS):
        e = np.flatnonzero(idx == r)
        if len(e):
            u[e] = -np.abs(u[e])
            u[e[0]] = -0.0
            u[e[1]] = 0.0 if r == BOTH_ZEROS else u[e[1]]
    u[idx == ONLY_NEG0] = -0.0
    return u


def _scatter(eb, op, upd, idx, size, layout):
    if layout == "aligned":
        return getattr(eb, "scatter_" + op)(upd, idx, size).cpu().numpy()
    d_idx = _dev(np.asarray(idx, np.int32))
    E, D = upd.shape
    return _raw("eu_scatter_" + op, (size, D), layout, upd, None, D, d_idx.data_ptr(), E, size)


def _sorted_cases(rs, D):
    idx = _sorted_index(rs, 400)
    yield "sorted", idx, _updates(rs, idx, D)
    yield "E=0", np.zeros(0, np.int32), np.zeros((0, D), np.float32)
    yield "E=1", np.asarray([37], np.int32), rs.choice(SPECIALS, (1, D))
    const = np.full(300, 9, np.int32)
    u = _updates(rs, const, D)
    u[::7] = rs.choice(SPECIALS, (len(u[::7]), D))
    yield "constant", const, u


def _unsorted_cases(rs, D):
    idx = _sorted_index(rs, 400)
    u = _updates(rs, idx, D)
    p = rs.permutation(len(idx))
    yield "permuted", idx[p], u[p]
    last = idx.copy()
    last[-1] = 4   # sorted but for the last element
    yield "sorted but the last", last, u
    yield "descending", idx[::-1].copy(), u[::-1].copy()


# ------------------------------------------------------------------ gather
@pytest.mark.parametrize("D", WIDTHS)
def test_gather(eb, D):
    rs = np.random.RandomState(D)
    N = 300
    params = rs.randn(N, D).astype(np.float32)
    m = rs.rand(N, D) < 0.1
    params[m] = rs.choice(SPECIALS, m.sum())
    idx = rs.randint(0, N, size=700).astype(np.int32)
    idx[:4] = [N - 1, 0, N - 1, 0]
    for name, ix in (("random", idx), ("E=1", idx[:1]), ("E=0", idx[:0])):
        want = ref.gather(params, ix)   # a copy: NaN payloads too
        for layout in LAYOUTS:
            if layout == "aligned":
                got = eb.gather(params, ix).cpu().numpy()
            else:
                d_ix = _dev(ix)
                got = _raw("eu_gather", (len(ix), D), layout, params, None, N, D, d_ix.data_ptr(), len(ix))
            cases.eq(got, want, "gather %s D=%d %s" % (name, D, layout))


# ------------------------------------------------------------------ scatter
@pytest.mark.parametrize("D", WIDTHS)
def test_scatter_sorted_bit_exact(eb, D):
    rs = np.random.RandomState(100 + D)
    for name, idx, u in _sorted_cases(rs, D):
        with np.errstate(invalid="ignore"):
            want = {op: getattr(ref, "scatter_" + op)(u, idx, SIZE) for op in ("add", "max", "mean")}
        for layout in LAYOUTS:
            got = {op: _scatter(eb, op, u, idx, SIZE, layout) for op in ("add", "max", "mean")}
            for op in ("add", "max", "mean"):
                eq_nan(got[op], want[op], "scatter_%s %s D=%d %s" % (op, name, D, layout))
            if name == "sorted":   # in index order the first of -0.0 / +0.0 stays, and -0.0 beats negatives and -1e9
                assert (got["max"][[ONLY_NEG0, NEG0_AMONG_NEG, BOTH_ZEROS]].view(np.uint32) == 0x80000000).all()


@pytest.mark.parametrize("D", WIDTHS)
def test_scatter_unsorted(eb, D):
    rs = np.random.RandomState(200 + D)
    for name, idx, u in _unsorted_cases(rs, D):
        with np.errstate(invalid="ignore"):
            add64, tol = ref.scatter_add64(u, idx, SIZE), atomic_tol(u, idx, SIZE)
        den = ref.counts(idx, SIZE).astype(np.float64) + 1e-7
        want_max = ref.scatter_max_order_free(u, idx, SIZE)
        for layout in LAYOUTS:
            what = "%s D=%d %s" % (name, D, layout)
            close64(_scatter(eb, "add", u, idx, SIZE, layout), add64, tol, "scatter_add " + what)
            close64(_scatter(eb, "mean", u, idx, SIZE, layout), add64 / den, tol / den, "scatter_mean " + what)
            got = _scatter(eb, "max", u, idx, SIZE, layout)
            cases.eq(got, want_max, "scatter_max " + what)
            # the one departure from index order: +0.0 wins among equal zeros; -0.0 alone, or among negatives, stays
            assert (got[BOTH_ZEROS].view(np.uint32) == 0).all(), "scatter_max +0.0 among zeros " + what
            assert (got[[ONLY_NEG0, NEG0_AMONG_NEG]].view(np.uint32) == 0x80000000).all(), "scatter_max -0.0 " + what
            assert (got[list(EMPTY)] == np.float32(-1e9)).all()


# ------------------------------------------------------------------ autograd
def _grad(fn, x, g):
    x = torch.tensor(x, device="cuda", requires_grad=True)
    fn(x).backward(torch.as_tensor(g, device="cuda"))
    return x.grad.cpu().numpy()


@pytest.mark.parametrize("D", (1, 3, 4, 33, 128))
@pytest.mark.parametrize("order", ("sorted", "unsorted"))
def test_gradients(eb, D, order):
    rs = np.random.RandomState(300 + D)
    idx = _sorted_index(rs, 400)
    if order == "unsorted":
        idx = idx[rs.permutation(len(idx))]
    E, N = len(idx), SIZE
    gy = rs.randn(SIZE, D).astype(np.float32)
    # scatter_add: gather(grad, idx), a copy
    u = rs.randn(E, D).astype(np.float32)
    cases.eq(_grad(lambda x: eb.scatter_add(x, idx, SIZE), u, gy), ref.scatter_add_grad64(gy, idx).astype(np.float32),
             "scatter_add grad")
    # gather: scatter_add(grad, idx, N), in index order on a sorted index
    ge = rs.randn(E, D).astype(np.float32)
    got = _grad(lambda x: eb.gather(x, idx), rs.randn(N, D).astype(np.float32), ge)
    if order == "sorted":
        cases.eq(got, ref.scatter_add(ge, idx, N), "gather grad")
    close64(got, ref.gather_grad64(ge, idx, N), atomic_tol(ge, idx, N), "gather grad")
    # scatter_mean: the composition add / (count + 1e-7)
    got = _grad(lambda x: eb.scatter_mean(x, idx, SIZE), u, gy)
    want = ref.scatter_mean_grad64(gy, idx, SIZE)
    assert np.allclose(got, want, rtol=1e-6, atol=0), "scatter_mean grad"
    # scatter_max over halves in [-3, 3]: many ties, the gradient split evenly among them
    t = (rs.randint(-6, 7, size=(E, D)) * np.float32(0.5)).astype(np.float32)
    x = torch.tensor(t, device="cuda", requires_grad=True)
    out = eb.scatter_max(x, idx, SIZE)
    cases.eq(out.detach().cpu().numpy(), ref.scatter_max(t, idx, SIZE), "scatter_max forward")
    out.backward(torch.as_tensor(gy, device="cuda"))
    want = ref.scatter_max_grad64(t, idx, ref.scatter_max(t, idx, SIZE), gy)
    assert np.allclose(x.grad.cpu().numpy(), want, rtol=1e-6, atol=0), "scatter_max grad"
    assert (ref.scatter_add64((want != 0).astype(np.float64), idx, SIZE) > 1).any(), "the data has ties"


@pytest.mark.parametrize("D", (1, 4, 33, 128, 1030))
def test_scatter_mean_composition_equals_fused_kernel(eb, D):
    """with autograd scatter_mean is composed from scatter_add; without, one kernel: the same bits on a sorted index"""
    rs = np.random.RandomState(400 + D)
    idx = _sorted_index(rs, 400)
    u = _updates(rs, idx, D)
    fused = eb.scatter_mean(u, idx, SIZE).cpu().numpy()
    x = torch.tensor(u, device="cuda", requires_grad=True)
    composed = eb.scatter_mean(x, idx, SIZE).detach().cpu().numpy()
    with np.errstate(invalid="ignore"):
        eq_nan(fused, ref.scatter_mean(u, idx, SIZE), "fused")
    eq_nan(composed, fused, "composed")


@pytest.mark.parametrize("order", ("sorted", "unsorted"))
def test_scatter_softmax(eb, order):
    """float64 reference; a segment of only -0.0 logits is a uniform softmax (not exp(0 + 1e9) / inf = NaN)"""
    rs = np.random.RandomState(7)
    idx = _sorted_index(rs, 400)
    x = (rs.randn(len(idx), 5) * 3).astype(np.float32)
    x[idx == ONLY_NEG0] = -0.0
    x[idx == NEG0_AMONG_NEG] = -np.abs(x[idx == NEG0_AMONG_NEG])
    x[np.flatnonzero(idx == NEG0_AMONG_NEG)[0]] = -0.0
    if order == "unsorted":
        p = rs.permutation(len(idx))
        idx, x = idx[p], x[p]
    got = eb.scatter_softmax(x, idx, SIZE).cpu().numpy()
    want = ref.scatter_softmax64(x, idx, SIZE)
    assert not np.isnan(got).any()
    assert np.allclose(got, want, rtol=1e-5, atol=1e-7), np.abs(got - want).max()
    n0 = (idx == ONLY_NEG0).sum()
    assert np.allclose(got[idx == ONLY_NEG0], 1.0 / n0, rtol=1e-6)


# ------------------------------------------------------------------ dense features
def _feature_graph(eb, slot_dims, n, seed, stride):
    """a graph whose feature rows are the dense slots slot_dims concatenated: uniform values over 16 binades, 5% -0.0, a few
    ±inf and NaN; ids 1 + stride * row (stride 1: the direct id -> row map, otherwise the hash table)"""
    rs = np.random.RandomState(seed)
    g = graphs.random_graph(seed=seed, n=n, T=1, avg_deg=2, id_stride=stride)
    fd = int(sum(slot_dims))
    feat = (rs.uniform(-1, 1, (n, fd)) * np.exp2(rs.randint(-8, 8, size=(n, fd)))).astype(np.float32)
    feat[rs.rand(n, fd) < 0.05] = -0.0
    m = rs.rand(n, fd) < 0.002
    feat[m] = rs.choice(SPECIALS[2:5], m.sum())
    eb.set_graph(eb.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], cum_w=g["cum_w"], node_type=g["node_type"],
                                   node_w=g["node_w"], feat=feat, feat_slot_dims=list(slot_dims)))
    return g["ids"], feat


def _ids(rs, gids, M):
    """M ids: mostly present, 6% each of -1 (default fill), 0 and ids not in the graph"""
    ids = gids[rs.randint(0, len(gids), size=M)].astype(np.int64)
    r = rs.rand(M)
    absent = np.asarray([int(gids.max()) + 7, int(gids[0]) + 1 if gids[1] - gids[0] > 1 else int(gids.max()) + 1], np.int64)
    ids[r < 0.06] = -1
    ids[(r >= 0.06) & (r < 0.12)] = 0
    sel = (r >= 0.12) & (r < 0.18)
    ids[sel] = rs.choice(absent, sel.sum())
    return ids


@pytest.mark.parametrize("slot_dims,stride", [((64,), 1), ((33,), 3), ((3, 8, 130), 3), ((4, 128), 1)])
def test_dense_feature(eb, slot_dims, stride):
    rs = np.random.RandomState(sum(slot_dims))
    gids, feat = _feature_graph(eb, slot_dims, 500, 11 + len(slot_dims), stride)
    ids = _ids(rs, gids, 600)
    rows = ref.rows_of(gids, ids)
    d_ids = _dev(ids)
    for fid in list(range(len(slot_dims))) + [len(slot_dims), -1]:
        s = slot_dims[fid] if 0 <= fid < len(slot_dims) else 8
        for dim in sorted({d for d in (1, s - 1, s, s + 1, s + 4, s + 5) if d > 0}):
            want = ref.dense_feature(feat, slot_dims, rows, fid, dim)
            what = "slots %s fid %d dim %d" % (slot_dims, fid, dim)
            cases.eq(eb.get_dense_feature(d_ids, [fid], [dim])[0].cpu().numpy(), want, what)
            got = _raw("eu_get_dense_feature", (len(ids), dim), "out+4", None, d_ids.data_ptr(), len(ids), fid, dim)
            cases.eq(got, want, what + " out+4")


# ------------------------------------------------------------------ fused SAGE mean / add
def _sage(eb, ids, R, count, dim, mean, layout="aligned"):
    d_ids = _dev(ids)
    if mean and layout == "aligned":
        return eb.sage_mean_aggregate(d_ids, count, dim).cpu().numpy()
    name = "eu_sage_mean_aggregate" if mean else "eu_sage_add_aggregate"
    return _raw(name, (R, dim), layout, None, d_ids.data_ptr(), R, count, dim)


def _check_sage(eb, gids, feat, ids, R, count, dim, layout="aligned", single_slot=True):
    rows = ref.rows_of(gids, ids)
    x = ref.whole_rows(feat, rows, dim)
    seg = np.repeat(np.arange(R, dtype=np.int32), count)
    for mean in (True, False):
        what = "%s feat_dim %d dim %d count %d %s" % ("mean" if mean else "add", feat.shape[1], dim, count, layout)
        got = _sage(eb, ids, R, count, dim, mean, layout)
        with np.errstate(invalid="ignore"):
            eq_nan(got, (ref.scatter_mean if mean else ref.scatter_add)(x, seg, R), what)
        if single_slot:   # there the fused op is get_dense_feature of slot 0 followed by scatter_mean / scatter_add
            (f,) = eb.get_dense_feature(_dev(ids), [0], [dim])
            eq_nan(got, (eb.scatter_mean if mean else eb.scatter_add)(f, seg, R).cpu().numpy(), what + " vs composition")


COUNTS = (1, 4, 5, 31, 32, 33, 65)


@pytest.mark.parametrize("feat_dim", (4, 64, 100, 128, 132, 200, 256, 260, 512, 516, 1024, 3, 130, 1028))
def test_fused_sage_widths(eb, feat_dim):
    """dim == feat_dim on one slot: every k_sage_mean instantiation, and the generic kernel at widths it alone takes"""
    rs = np.random.RandomState(feat_dim)
    gids, feat = _feature_graph(eb, (feat_dim,), 700, feat_dim, 1 if feat_dim % 8 else 3)
    for count in COUNTS:
        R = max(8, 1024 // count)
        ids = _ids(rs, gids, R * count)
        ids[:count] = -1   # a row without any neighbor
        _check_sage(eb, gids, feat, ids, R, count, feat_dim)


def test_fused_sage_generic_cases(eb):
    """dim below and above the stored width, an unaligned output, and multi-slot graphs, where every neighbor contributes the
    first dim columns of its whole stored row"""
    rs = np.random.RandomState(9)
    gids, feat = _feature_graph(eb, (64,), 600, 21, 3)
    for count in (1, 5, 33):
        R = max(8, 512 // count)
        ids = _ids(rs, gids, R * count)
        for dim in (40, 63, 70):
            _check_sage(eb, gids, feat, ids, R, count, dim)
        _check_sage(eb, gids, feat, ids, R, count, 64, layout="out+4")
    for slot_dims in ((3, 8, 130), (4, 128)):
        gids, feat = _feature_graph(eb, slot_dims, 600, 22, 1)
        for count in (1, 5, 33):
            R = max(8, 512 // count)
            ids = _ids(rs, gids, R * count)
            for dim in sorted({slot_dims[0], slot_dims[0] + slot_dims[1], feat.shape[1], feat.shape[1] + 9}):
                _check_sage(eb, gids, feat, ids, R, count, dim, single_slot=dim <= slot_dims[0])
    # what a multi-slot graph's fused op reads past slot 0 is slot 1's columns, where get_dense_feature of slot 0 has zeros
    ids = gids[:4].astype(np.int64)
    eq_nan(_sage(eb, ids, 4, 1, 8, False), feat[:4, :8] + np.float32(0), "slot 1's columns")
    assert not eb.get_dense_feature(_dev(ids), [0], [8])[0].cpu().numpy()[:, 4:].any()


@pytest.mark.parametrize("dim", (64, 3))
def test_fused_sage_count_zero(eb, dim):
    """no neighbors at all: zeros (the sum of nothing, / 1e-7 for the mean)"""
    _feature_graph(eb, (dim,), 100, 31, 1)
    ids = _dev(np.ones(1, np.int64))
    for mean in (True, False):
        for layout in ("aligned", "out+4"):
            got = _raw("eu_sage_mean_aggregate" if mean else "eu_sage_add_aggregate", (37, dim), layout, None,
                       ids.data_ptr(), 37, 0, dim)
            cases.eq(got, np.zeros((37, dim), np.float32), "count 0 dim %d %s" % (dim, layout))


@pytest.mark.parametrize("dim,layout", [(64, "aligned"), (128, "aligned"), (3, "aligned"), (64, "out+4")])
def test_fused_sage_dedup_rows(eb, dim, layout):
    """2^17 rows, where each distinct segment is reduced once and copied to its repeats: rows drawn from 3000 segments, among
    them segments with the same ids in another order and segments with no id in the graph"""
    rs = np.random.RandomState(dim)
    gids, feat = _feature_graph(eb, (dim,), 2000, 41, 3)
    R, count = 1 << 17, 5
    pool = _ids(rs, gids, 3000 * count).reshape(3000, count)
    pool[1000:1500] = pool[:500][:, ::-1]          # the same ids, reversed: another sum order
    pool[1500:1600] = -1
    pool[1600:1700] = int(gids.max()) + 7
    seg = pool[rs.randint(0, 3000, size=R)]
    rows = ref.rows_of(gids, seg.reshape(-1)).reshape(R, count)
    for mean in (True, False):
        with np.errstate(invalid="ignore"):
            want = ref.fanout_aggregate(feat, rows, dim, mean)
        eq_nan(_sage(eb, seg.reshape(-1), R, count, dim, mean, layout), want, "dedup dim %d %s mean=%s" % (dim, layout, mean))
