"""GPU: bfloat16 embedding stores.  ops.store_exchange / store_accumulate on bf16 store pairs (eu_store_exchange_dtype /
eu_store_accumulate_dtype) bit for bit against the numpy restatement and the f32 op on the widened tables, at every width
and alignment, with special values, under CUDA-graph replay, past 2^32 elements and on refusal; and ScalableSageEncoder /
ScalableGCNEncoder with store_dtype=torch.bfloat16 against the f32 encoder started from the widened stores."""
import gc

import numpy as np
import pytest
import torch

import bf16_reference as bf
import graphs
import sr_reference as sr
import store_reference as st

pytestmark = pytest.mark.gpu

N_NODES = 400
SEED = 0xDEADBEEF12345678


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = graphs.random_graph(seed=5, n=N_NODES, T=1, avg_deg=6, feat_dim=8, hub=150)
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=1, node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=[8])
    return dict(g=g, gr=gr)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _u16(t):
    return t.detach().cpu().view(torch.int16).numpy().view(np.uint16)


def _i32(t):
    return t.detach().cpu().numpy().view(np.int32)


def _bf16(bits, offset=0):
    """a device bf16 table holding the uint16 bits, its data `offset` elements past a 16-byte boundary"""
    bits = np.ascontiguousarray(bits, np.uint16)
    buf = torch.empty(bits.size + offset, dtype=torch.bfloat16, device="cuda")
    t = buf[offset:].view(bits.shape)
    t.view(torch.int16).copy_(torch.from_numpy(bits.view(np.int16)))
    return t


def _same_rounded(got, want):
    """bf16 bits rounded to nearest on the device against bf16_reference.round_bits: equal bits, except that a NaN is
    compared as NaN-ness (the device's canonical NaN need not be numpy's)"""
    nan = np.isnan(bf.widen(want))
    return np.array_equal(np.isnan(bf.widen(got)), nan) and np.array_equal(got[~nan], want[~nan])


def _f32(x, offset=0):
    x = np.ascontiguousarray(x, np.float32)
    buf = torch.empty(x.size + offset, dtype=torch.float32, device="cuda")
    t = buf[offset:].view(x.shape)
    t.copy_(torch.from_numpy(x))
    return t


def _rows(shape, seed, special=False):
    """f32 N(0, 1) values; special: with every special value of bf16_reference (+-0, subnormals, ties, +-Inf, NaNs with
    payloads) sprinkled in"""
    rng = np.random.RandomState(seed)
    x = rng.randn(*shape).astype(np.float32)
    if special:
        sv = bf.special_values()
        flat = x.reshape(-1)
        k = min(flat.size, 4 * sv.size)
        flat[rng.choice(flat.size, size=k, replace=False)] = np.resize(sv, k)
    return x


def _rand_bits(shape, seed, special=False):
    """the bf16 bits of _rows, rounded to nearest"""
    return bf.round_bits(_rows(shape, seed, special)).reshape(shape)


def _ids(n_rows, M, seed):
    """ids with repeats: random ones, one id 50 times through the list, and a run of one id"""
    rng = np.random.RandomState(seed)
    ids = rng.randint(0, n_rows, size=M)
    if M >= 200:
        ids[rng.choice(M, size=50, replace=False)] = 7
        ids[100:140] = n_rows - 1
    return ids.astype(np.int64)


def _step(v):
    return torch.tensor(v, dtype=torch.int64, device="cuda")


# ---------------------------------------------------------------------------- exchange
@pytest.mark.parametrize("offset", (0, 1, 4))
@pytest.mark.parametrize("dim", (1, 3, 4, 16, 128, 200))
def test_exchange_bits(env, dim, offset):
    import euler_b200
    n_rows, M = 500, 3000
    S0, G0 = _rand_bits((n_rows, dim), 1, special=True), _rand_bits((n_rows, dim), 2, special=True)
    rows, ids = _rows((M, dim), 3, special=True), _ids(n_rows, M, 4)
    store, grad_store = _bf16(S0, offset), _bf16(G0, offset)
    want_s, want_g, want_t = st.exchange(S0, G0, ids, rows)
    taken = euler_b200.store_exchange(store, grad_store, torch.as_tensor(ids, device="cuda"), _f32(rows, offset))
    assert taken.dtype == torch.float32 and taken.shape == (M, dim)
    assert _same_rounded(_u16(store), want_s)                  # every row: the written ones rounded to nearest, the rest kept
    assert np.array_equal(_u16(grad_store), want_g)            # the cleared rows exact zeros
    assert np.array_equal(_i32(taken), want_t.view(np.int32))  # the pre-clear rows widened, NaN payloads included
    # M = 0 touches nothing
    empty = torch.zeros(0, dtype=torch.int64, device="cuda")
    assert euler_b200.store_exchange(store, grad_store, empty, _f32(rows[:0])).shape == (0, dim)
    assert _same_rounded(_u16(store), want_s) and np.array_equal(_u16(grad_store), want_g)


# ---------------------------------------------------------------------------- accumulate
def _accumulate_want(G0, ids, grad, count, pool, seed, step, tensor):
    """the f32 op's sums added to the widened rows (the f32 op run on the widened table), then stochastic rounding with word
    0 of philox_bits(seed, step, tensor, v * dim + f); untouched rows are exact, so their rounding keeps their bits"""
    import euler_b200
    x = torch.from_numpy(bf.widen(G0).reshape(G0.shape)).cuda()
    euler_b200.store_accumulate(x, torch.as_tensor(ids, device="cuda"), _f32(grad), count, pool)
    x = x.cpu().numpy()
    elem = np.arange(x.size, dtype=np.int64)
    return sr.sr_bits(x.reshape(-1), sr.philox_bits(seed, step, tensor, elem)[0]).reshape(G0.shape)


@pytest.mark.parametrize("pool", ("sum", "mean"))
@pytest.mark.parametrize("count", (1, 2, 10, 25))
@pytest.mark.parametrize("dim,offset", [(16, 0), (3, 0), (128, 1), (200, 4)])
def test_accumulate_bits(env, count, pool, dim, offset):
    import euler_b200
    n_rows, R = 600, 240
    ids = _ids(n_rows, R * count, 6)
    grad, G0 = _rows((R, dim), 7), _rand_bits((n_rows, dim), 8)
    G0[5] = bf.round_bits(bf.special_values()[:dim] if dim <= 32 else np.resize(bf.special_values(), dim))   # special values
    gs = _bf16(G0, offset)
    euler_b200.store_accumulate(gs, torch.as_tensor(ids, device="cuda"), _f32(grad, offset), count, pool, seed=SEED,
                                step=_step(3), tensor=2)
    want = _accumulate_want(G0, ids, grad, count, pool, SEED, 3, 2)
    assert np.array_equal(_u16(gs), want)
    if dim == 16:   # the numpy restatement agrees too
        assert np.array_equal(want, st.accumulate(G0, ids, grad, count, pool, SEED, 3, 2))


def test_accumulate_one_id_many_times(env):
    import euler_b200
    ids = np.full(20480, 11, np.int64)
    grad = np.random.RandomState(3).randn(2048, 8).astype(np.float32)
    G0 = _rand_bits((40, 8), 4)
    for pool in ("sum", "mean"):
        gs = _bf16(G0)
        euler_b200.store_accumulate(gs, torch.as_tensor(ids, device="cuda"), _f32(grad), 10, pool, seed=5, step=_step(9), tensor=1)
        want = st.accumulate(G0, ids, grad, 10, pool, 5, 9, 1)
        assert np.array_equal(_u16(gs), want)
        assert np.array_equal(want, _accumulate_want(G0, ids, grad, 10, pool, 5, 9, 1))


def test_accumulate_repeats_per_step_and_changes_with_it(env):
    import euler_b200
    ids = torch.as_tensor(_ids(300, 3000, 2), device="cuda")
    grad, G0 = _f32(_rows((300, 16), 3)), _rand_bits((300, 16), 4)
    out = {}
    for key in ((7, 0, 0), (7, 0, 0), (7, 1, 0), (7, 0, 1), (8, 0, 0)):
        gs = _bf16(G0)
        euler_b200.store_accumulate(gs, ids, grad, 10, "mean", seed=key[0], step=_step(key[1]), tensor=key[2])
        out.setdefault(key, []).append(_u16(gs))
    assert np.array_equal(out[(7, 0, 0)][0], out[(7, 0, 0)][1])
    for other in ((7, 1, 0), (7, 0, 1), (8, 0, 0)):
        assert not np.array_equal(out[(7, 0, 0)][0], out[other][0])


def test_many_sub_ulp_accumulations_stay_unbiased(env):
    """200 steps each adding 2^-10 (an eighth of bf16's ulp at 1.0) to 4096 elements of 1.0: the exact sum is
    1 + 200 / 1024 = 1.1953125.  Each stochastic rounding has mean zero and variance at most ulp^2 / 4 = 2^-16, so one
    element's error has a standard deviation under sqrt(200) 2^-8 = 0.055 and the mean of 4096 independent ones under
    0.00086; the bound is 0.005.  Rounding to nearest would keep every element at 1.0."""
    import euler_b200
    gs = torch.ones(64, 64, dtype=torch.bfloat16, device="cuda")
    ids = torch.arange(64, device="cuda")
    grad = torch.full((64, 64), 2.0 ** -10, device="cuda")
    step = _step(0)
    for _ in range(200):
        euler_b200.store_accumulate(gs, ids, grad, 1, "sum", seed=11, step=step, tensor=0)
        step.add_(1)
    mean = float(gs.double().mean())
    assert abs(mean - (1 + 200 / 1024)) < 0.005, mean
    assert float(gs.double().std()) > 0     # the elements did not all move together


# ---------------------------------------------------------------------------- CUDA graphs
def test_capture_replays_eager_with_the_live_step(env):
    import euler_b200
    ids = torch.as_tensor(_ids(300, 2000, 5), device="cuda")
    rows, grad = _f32(_rows((2000, 16), 3)), _f32(_rows((200, 16), 4))
    S0, G0 = _rand_bits((300, 16), 1), _rand_bits((300, 16), 2)
    store, gs = _bf16(S0), _bf16(G0)
    step = _step(4)

    def call():
        taken = euler_b200.store_exchange(store, gs, ids, rows)
        euler_b200.store_accumulate(gs, ids, grad, 10, "mean", seed=SEED, step=step, tensor=1)
        return taken

    def reset():
        store.view(torch.int16).copy_(torch.from_numpy(S0.view(np.int16)))
        gs.view(torch.int16).copy_(torch.from_numpy(G0.view(np.int16)))

    eager = {}
    for k in (4, 5):
        reset()
        step.fill_(k)
        taken = call()
        eager[k] = (_u16(store), _u16(gs), _i32(taken))
    assert not np.array_equal(eager[4][1], eager[5][1])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()                                      # sizes the scratch outside the capture
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = call()
    torch.cuda.current_stream().wait_stream(s)
    for k in (4, 5):                                # the counter advances between replays
        reset()
        step.fill_(k)
        cg.replay()
        torch.cuda.synchronize()
        got = (_u16(store), _u16(gs), _i32(out))
        assert all(np.array_equal(a, b) for a, b in zip(got, eager[k])), k


# ---------------------------------------------------------------------------- refusals
def test_refusals_leave_every_table_unchanged(env):
    import euler_b200
    from euler_b200 import EulerError, ops
    store, gs = _bf16(_rand_bits((50, 8), 1)), _bf16(_rand_bits((50, 8), 2))
    rows = _f32(_rows((4, 8), 3))
    before = _u16(store), _u16(gs)
    step = _step(0)

    def unchanged():
        torch.cuda.synchronize()
        assert np.array_equal(_u16(store), before[0]) and np.array_equal(_u16(gs), before[1])
        assert int(step) == 0

    for bad in (-1, 50):
        ids = torch.as_tensor([3, bad, 3, 9], device="cuda")
        with pytest.raises(EulerError, match="outside"):
            euler_b200.store_exchange(store, gs, ids, rows)
        with pytest.raises(EulerError, match="outside"):
            euler_b200.store_accumulate(gs, ids, rows, seed=1, step=step)
        unchanged()
    ids = torch.as_tensor([3, 4, 3, 9], device="cuda")
    with pytest.raises(EulerError, match="one dtype"):                       # mixed store dtypes
        euler_b200.store_exchange(store, gs.float(), ids, rows)
    with pytest.raises(EulerError, match="one dtype"):
        euler_b200.store_exchange(store.float(), gs, ids, rows)
    with pytest.raises(EulerError, match="float32"):                         # other dtypes
        euler_b200.store_exchange(store.half(), gs.half(), ids, rows)
    with pytest.raises(EulerError, match="step"):                            # bf16 accumulation without its counter
        euler_b200.store_accumulate(gs, ids, rows)
    with pytest.raises(EulerError, match="step"):
        euler_b200.store_accumulate(gs, ids, rows, step=step.int())
    with pytest.raises(EulerError, match="seed"):
        euler_b200.store_accumulate(gs, ids, rows, seed=-1, step=step)
    unchanged()
    # at the C ABI: an unknown dtype, and bf16 accumulation with a NULL step: EU_ERR_INVALID before any device work
    lib = euler_b200._lib.load()
    n0 = lib.eu_launch_count()
    taken = torch.full((4, 8), 7.0, device="cuda")
    for dt in (2, -1):
        with pytest.raises(EulerError, match="dtype"):
            ops._call("eu_store_exchange_dtype", store, gs, 50, 8, ids, 4, rows, taken, dt)
        with pytest.raises(EulerError, match="dtype"):
            ops._call("eu_store_accumulate_dtype", gs, 50, 8, ids, 4, 1, 0, rows, dt, 0, step, 0)
    with pytest.raises(EulerError, match="step"):
        ops._call("eu_store_accumulate_dtype", gs, 50, 8, ids, 4, 1, 0, rows, 1, 0, None, 0)
    assert lib.eu_launch_count() == n0
    unchanged()
    assert bool((taken == 7.0).all())


# ---------------------------------------------------------------------------- past 2^32 elements
N32 = (1 << 25) + (1 << 13)   # rows of a width-128 table past 2^32 + 2^20 elements


def test_store_pair_past_2_32(env):
    """a bf16 store pair [2^25 + 2^13, 128]: 2 x 8.6 GB.  The touched rows are restated from their own bits with their global
    element indices (store_reference's rows=), never against a compact table, whose random bits would differ."""
    import euler_b200
    dim = 128
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * N32 * dim * 2 + (2 << 30):
        pytest.skip("needs %.1f GB of free device memory" % ((2 * N32 * dim * 2 + (2 << 30)) / 2 ** 30))
    first = 1 << 25                                  # row 2^25 starts at element 2^32
    rng = np.random.RandomState(1)
    touched = np.concatenate([[0, first - 1, first, first + 1, N32 - 1], rng.randint(first, N32, size=300)])
    ids = np.concatenate([touched, np.full(300, first, np.int64), rng.choice(touched, size=400)]).astype(np.int64)
    rng.shuffle(ids)
    ids = ids[:len(ids) // 4 * 4]                    # count 4 divides M
    assert int(ids.max()) * dim >= 1 << 32, "the largest touched element stays under 2^32"
    uniq = np.unique(ids)
    keep = np.setdiff1d(np.unique(np.concatenate([uniq - 1, uniq + 1])), uniq)
    keep = keep[(keep >= 0) & (keep < N32)]          # untouched neighbours of touched rows
    pick = np.concatenate([uniq, keep])
    store = torch.zeros((N32, dim), dtype=torch.bfloat16, device="cuda")
    gs = torch.zeros((N32, dim), dtype=torch.bfloat16, device="cuda")
    S0, G0 = _rand_bits((len(pick), dim), 2), _rand_bits((len(pick), dim), 3)
    pk = torch.as_tensor(pick, device="cuda")
    store.view(torch.int16)[pk] = torch.from_numpy(S0.view(np.int16)).cuda()
    gs.view(torch.int16)[pk] = torch.from_numpy(G0.view(np.int16)).cuda()
    loc = np.searchsorted(uniq, ids)                 # ids as rows of the picked arrays (uniq comes first in pick)
    rows = _rows((len(ids), dim), 4)
    grad = _rows((len(ids) // 4, dim), 5)
    d_ids = torch.as_tensor(ids, device="cuda")
    taken = euler_b200.store_exchange(store, gs, d_ids, _f32(rows))
    want_s, want_g, want_t = st.exchange(S0, G0, loc, rows)
    assert np.array_equal(_i32(taken), want_t.view(np.int32))
    assert np.array_equal(_u16(store[pk]), want_s)
    assert np.array_equal(_u16(gs[pk]), want_g)
    # refill the gradient rows, then accumulate
    G1 = _rand_bits((len(pick), dim), 6)
    gs.view(torch.int16)[pk] = torch.from_numpy(G1.view(np.int16)).cuda()
    euler_b200.store_accumulate(gs, d_ids, _f32(grad), 4, "mean", seed=SEED, step=_step(2 ** 32 + 7), tensor=3)
    want = st.accumulate(G1, loc, grad, 4, "mean", SEED, 2 ** 32 + 7, 3, rows=pick)
    assert np.array_equal(_u16(gs[pk]), want)
    del store, gs


# ---------------------------------------------------------------------------- encoders
def _seeds(step):
    rng = np.random.RandomState(20 + step)
    s = rng.randint(1, N_NODES + 1, size=96)
    s[:8] = s[8:16]                                                 # repeated seeds
    return torch.as_tensor(s, dtype=torch.int64, device="cuda")


def _make(cls, dt, **kw):
    torch.manual_seed(0)
    return cls([0], **kw, feature_idx=["feat0"], feature_dim=[8], max_id=N_NODES, use_id=True, embedding_dim=8,
               store_learning_rate=0.01, store_init_maxval=0.5, device="cuda", store_dtype=dt, store_seed=SEED,
               generator=torch.Generator(device="cuda").manual_seed(1))


def _sync(e32, e16):
    """the f32 arm's stores and gradient stores := the bf16 arm's, widened"""
    with torch.no_grad():
        for a, b in zip(e32.stores + e32.gradient_stores, e16.stores + e16.gradient_stores):
            a.copy_(b.float())


CASES = ([("ScalableSageEncoder", dict(fanout=5, num_layers=L, dim=8, aggregator=a)) for a in ("mean", "gcn") for L in (1, 2, 3)]
         + [("ScalableSageEncoder", dict(fanout=4, num_layers=L, dim=8, aggregator="meanpool")) for L in (1, 2, 3)]
         + [("ScalableGCNEncoder", dict(num_layers=L, dim=8, aggregator=a, use_residual=r, head_num=2))
            for a, L in (("gcn", 2), ("mean", 3), ("attention", 3)) for r in (False, True)])


@pytest.mark.parametrize("name,kw", CASES)
def test_encoder_steps_against_f32_on_the_widened_stores(env, name, kw):
    import euler_b200
    from euler_b200 import encoders
    cls = getattr(encoders, name)
    e16, e32 = _make(cls, torch.bfloat16, **kw), _make(cls, torch.float32, **kw)
    assert all(torch.equal(a, b) for a, b in zip(e16.parameters(), e32.parameters()))
    torch.manual_seed(4)
    head = (torch.randn(e16.dims[-1], 1) * 0.5).cuda()
    heads = {k: head.clone().requires_grad_() for k in ("16", "32")}
    opts = {k: torch.optim.SGD(list(e.parameters()) + [heads[k]], lr=0.05) for k, e in (("16", e16), ("32", e32))}
    n_stores = kw["num_layers"] - 1
    for step in range(3):
        _sync(e32, e16)
        losses = {}
        for k, e in (("16", e16), ("32", e32)):
            euler_b200.seed(100 + step)
            out = e(_seeds(step), training=True)
            losses[k] = torch.tanh(out @ heads[k]).square().mean()
        assert _i32(losses["16"]).tolist() == _i32(losses["32"]).tolist(), step
        assert _i32(e16.store_loss).tolist() == _i32(e32.store_loss).tolist(), step
        for a, b in zip(e16.stores, e32.stores):                  # the exchange: the f32 arm's writes rounded to nearest
            assert np.array_equal(_u16(a), bf.round_bits(b.detach().cpu().numpy())), step
        for a, b in zip(e16.gradient_stores, e32.gradient_stores):
            assert torch.equal(a.float(), b), step                # cleared rows zero, the rest as synced
        assert int(e16.store_sr_step) == step
        e16.train_step(losses["16"], opts["16"])
        e32.train_step(losses["32"], opts["32"])
        assert int(e16.store_sr_step) == step + 1
        for l, (a, b) in enumerate(zip(e16.gradient_stores, e32.gradient_stores)):
            x = b.detach().cpu().numpy()                          # the f32 arm's pre-rounding values
            words = sr.philox_bits(SEED, step, l, np.arange(x.size, dtype=np.int64))[0]
            assert np.array_equal(_u16(a), sr.sr_bits(x.reshape(-1), words).reshape(x.shape)), (step, l)
        for a, b in zip(list(e16.parameters()) + [heads["16"]], list(e32.parameters()) + [heads["32"]]):
            assert torch.equal(a, b), step
    if n_stores:
        assert any(g.any() for g in e16.gradient_stores)          # gradients reached the stores


def test_supervised_training_matches_f32(env):
    """300 full-batch steps of a supervised ScalableSageEncoder (2 layers, 'mean'; every node a seed, its labels the signs of
    its first 4 features; the sampler reseeded per step, so both arms draw the same hops): the mean loss of the last 50
    steps with bf16 stores is within 2 % of f32 training's from the same widened stores"""
    import euler_b200
    from euler_b200 import encoders
    kw = dict(fanout=5, num_layers=2, dim=16, aggregator="mean")
    e16 = _make(encoders.ScalableSageEncoder, torch.bfloat16, **kw)
    e32 = _make(encoders.ScalableSageEncoder, torch.float32, **kw)
    _sync(e32, e16)
    start = [s.clone() for s in e16.stores]
    arms = {}
    for k, e in (("16", e16), ("32", e32)):
        torch.manual_seed(4)
        head = torch.nn.Linear(16, 4).cuda()
        opt = torch.optim.SGD(list(e.parameters()) + list(head.parameters()), lr=0.1)
        losses = []
        for step in range(300):
            euler_b200.seed(1000 + step)
            seeds = torch.arange(1, N_NODES + 1, device="cuda")
            label = (euler_b200.get_dense_feature(seeds, ["feat0"], [4])[0] > 0).float()
            loss = torch.nn.functional.binary_cross_entropy_with_logits(head(e(seeds, training=True)), label)
            e.train_step(loss, opt)
            losses.append(float(loss))
        arms[k] = float(np.mean(losses[-50:]))
        assert arms[k] < float(np.mean(losses[:50])), (k, "the loss did not fall")
    assert abs(arms["16"] - arms["32"]) <= 0.02 * arms["32"], arms
    assert int(e16.store_sr_step) == 300
    assert not all(torch.equal(a, b) for a, b in zip(e16.stores, start))     # the stores moved
