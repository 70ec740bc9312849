"""GPU: ops.neighbor_top_k_feature (eu_neighbor_top_k_feature) bit for bit against a stable descending sort of the
get_dense_feature rows, over slot widths before and past the read width, tie-heavy rows, +-0.0, NaN, absent and -1 ids;
run-to-run and CUDA-graph replay; the refusals.  LGCEncoder fused against the float64 composition on the same draws, and
one LGCN training step against fused=False."""
import copy

import numpy as np
import pytest
import torch

import graphs

pytestmark = pytest.mark.gpu

N_NODES = 600
SLOT_DIMS = (3, 130, 1433)      # the dense slots feat0, feat1, feat2
ABSENT = 10 ** 9                # an id no row has
NAN_A = np.array([0x7fc00001], np.uint32).view(np.float32)[0]   # two NaN payloads, one with the sign bit
NAN_B = np.array([0xffc00002], np.uint32).view(np.float32)[0]


def _features(rng):
    """quarters in [-1, 1] (many ties), -0.0 and +0.0 mixed in, NaNs of two payloads, and rows that are one value"""
    f = (rng.randint(-4, 5, size=(N_NODES, sum(SLOT_DIMS))) / 4).astype(np.float32)
    f[rng.rand(*f.shape) < 0.1] = np.float32(-0.0)
    f[rng.rand(*f.shape) < 0.1] = np.float32(0.0)
    f[rng.rand(*f.shape) < 0.01] = NAN_A
    f[rng.rand(*f.shape) < 0.01] = NAN_B
    f[::7] = np.float32(0.5)
    f[3::11] = np.float32(-0.0)
    return f


@pytest.fixture(scope="module")
def env():
    import euler_b200
    g = graphs.random_graph(seed=5, n=N_NODES, T=1, avg_deg=6)
    g["feat"] = _features(np.random.RandomState(6))
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=1, node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], feat=g["feat"], feat_slot_dims=list(SLOT_DIMS))
    return dict(g=g, gr=gr)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)


def _ids(env, B, count, seed):
    """nodes i64[B] (one absent, one -1) and neighbours i64[B, count]: graph ids, absent ids and -1, one row of a single id"""
    rng = np.random.RandomState(seed)
    ids = env["g"]["ids"].astype(np.int64)
    nodes = ids[rng.randint(0, N_NODES, size=B)]
    nodes[B // 2] = ABSENT
    nodes[-1] = -1
    nbrs = ids[rng.randint(0, N_NODES, size=(B, count))]
    nbrs[rng.rand(B, count) < 0.1] = ABSENT
    nbrs[rng.rand(B, count) < 0.1] = -1
    nbrs[0] = ids[7]                                              # a row of one id: every column one tie
    return torch.as_tensor(nodes, device="cuda"), torch.as_tensor(nbrs, device="cuda")


def _want(nodes, nbrs, slot, dim, k):
    """cat(get_dense_feature(nodes), the first k rows of a stable descending sort of the neighbour rows per column); sorted
    on the CPU, whose stable sort compares values (-0.0 == +0.0, NaN above every number)"""
    import euler_b200
    B, count = nbrs.shape
    node = euler_b200.get_dense_feature(nodes, [slot], [dim])[0].cpu()
    rows = euler_b200.get_dense_feature(nbrs.reshape(-1), [slot], [dim])[0].cpu().reshape(B, count, dim)
    top = torch.sort(rows, dim=1, descending=True, stable=True)[0][:, :k]
    return torch.cat([node[:, None], top], 1)


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def _check(env, B, count, slot, dim, k, seed):
    import euler_b200
    nodes, nbrs = _ids(env, B, count, seed)
    got = euler_b200.neighbor_top_k_feature(nodes, nbrs, slot, dim, k)
    assert got.shape == (B, k + 1, dim) and got.dtype == torch.float32 and not got.requires_grad
    assert torch.equal(_bits(got), _bits(_want(nodes, nbrs, slot, dim, k))), (slot, dim, count, k)
    return got


@pytest.mark.parametrize("k", (1, 3, 6, 16))
@pytest.mark.parametrize("slot,dim", [("feat0", 1), ("feat0", 3), ("feat0", 4), ("feat0", 16), ("feat1", 16), ("feat1", 128),
                                      ("feat1", 1433), ("feat2", 128), ("feat2", 1433)])
def test_bits_over_widths(env, slot, dim, k):
    got = _check(env, 48, 33, slot, dim, k, seed=dim + k)
    width = SLOT_DIMS[int(slot[-1])]
    if dim > width:
        assert not _bits(got[:, :, width:]).any()                      # past the stored width: +0.0 only


@pytest.mark.parametrize("k", (1, 2, 3, 16))
@pytest.mark.parametrize("count", (1, "k", 10, 33, 100))
def test_bits_over_counts(env, count, k):
    count = k if count == "k" else count
    if k > count:
        pytest.skip("k above count is refused")
    for slot, dim in (("feat0", 4), ("feat1", 130)):
        _check(env, 96, count, slot, dim, k, seed=count * 17 + k)


def test_ties_signed_zeros_and_nans_actually_occur(env):
    """the fixture's rows hold what the bit tests are about: -0.0 selected beside +0.0, and both NaN payloads selected"""
    import euler_b200
    nodes, nbrs = _ids(env, 96, 33, 1)
    got = _bits(euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 130, 16))
    for pattern in (np.float32(-0.0), np.float32(0.0), NAN_A, NAN_B):
        assert (got == int(np.array([pattern]).view(np.int32)[0])).any(), pattern


def test_unknown_slot_reads_zeros_and_slot_ids_work(env):
    import euler_b200
    nodes, nbrs = _ids(env, 32, 10, 2)
    assert not _bits(euler_b200.neighbor_top_k_feature(nodes, nbrs, 7, 16, 3)).any()
    by_id = euler_b200.neighbor_top_k_feature(nodes, nbrs, 1, 16, 3)
    assert torch.equal(_bits(by_id), _bits(euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 16, 3)))


def test_empty_batch_and_run_to_run(env):
    import euler_b200
    empty = torch.zeros(0, dtype=torch.int64, device="cuda")
    assert euler_b200.neighbor_top_k_feature(empty, empty.reshape(0, 10), "feat1", 16, 3).shape == (0, 4, 16)
    nodes, nbrs = _ids(env, 4096, 10, 3)
    a = euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat2", 1433, 3)
    b = euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat2", 1433, 3)
    assert torch.equal(_bits(a), _bits(b))


def test_capture_replays_the_eager_bits(env):
    import euler_b200
    nodes, nbrs = _ids(env, 512, 10, 4)
    eager = euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 130, 3)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 130, 3)
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            out = euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 130, 3)
    torch.cuda.current_stream().wait_stream(s)
    out.fill_(7.0)
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(eager))


def _raw(*args):
    from euler_b200 import _lib, ops
    return _lib.load().eu_neighbor_top_k_feature(ops._ctx_on_stream()._h, *args)


def test_refusals_leave_out_untouched(env):
    import euler_b200
    from euler_b200 import _lib
    nodes, nbrs = _ids(env, 16, 20, 5)
    out = torch.full((16, 18, 8), 3.0, device="cuda")
    p = (nodes.data_ptr(), 16, nbrs.data_ptr(), 20, 1, 8)
    assert _raw(*p, 0, out.data_ptr()) == 1                         # k < 1: EU_ERR_INVALID
    assert _raw(nodes.data_ptr(), 16, nbrs.data_ptr(), 5, 1, 8, 6, out.data_ptr()) == 1   # k > count
    assert _raw(*p, _lib.NEIGHBOR_TOP_K_MAX + 1, out.data_ptr()) == 4                    # above the bound: EU_ERR_UNSUPPORTED
    assert _raw(None, 16, nbrs.data_ptr(), 20, 1, 8, 3, out.data_ptr()) == 1              # a NULL pointer
    assert _raw(nodes.data_ptr(), 16, None, 20, 1, 8, 3, out.data_ptr()) == 1
    assert _raw(*p, 3, None) == 1
    assert _raw(nodes.data_ptr(), -1, nbrs.data_ptr(), 20, 1, 8, 3, out.data_ptr()) == 1  # negative B
    assert _raw(nodes.data_ptr(), 16, nbrs.data_ptr(), 20, 1, -8, 3, out.data_ptr()) == 1  # negative dim
    assert _raw(None, 0, None, 20, 1, 8, 3, None) == 0                                    # B = 0: nothing to do
    torch.cuda.synchronize()
    assert bool((out == 3.0).all())
    with pytest.raises(euler_b200.EulerError, match="count"):
        euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 8, 21)
    with pytest.raises(euler_b200.EulerError, match="bound"):
        euler_b200.neighbor_top_k_feature(nodes, nbrs, "feat1", 8, 17)
    with pytest.raises(euler_b200.EulerError, match="count"):
        euler_b200.neighbor_top_k_feature(nodes, nbrs[:8], "feat1", 8, 3)
    assert _raw(*p, _lib.NEIGHBOR_TOP_K_MAX, out.data_ptr()) == 0                        # the bound itself runs


# ---------------------------------------------------------------------------- LGCEncoder and LGCN
def _f64_features(monkeypatch):
    """get_dense_feature hands out float64 rows from here on (the float64 copy's composition reads them)"""
    from euler_b200 import ops
    real = ops.get_dense_feature
    monkeypatch.setattr(ops, "get_dense_feature", lambda *a, **k: [t.double() for t in real(*a, **k)])


def _close(a, b, what):
    a, b = a.double(), b.double()
    assert (a - b).abs().max() <= 1e-5 * max(b.abs().max(), 1e-3), what


def _finite_graph(env):
    """the fixture's graph without its NaNs (a NaN row poisons every gradient it reaches) and with +0.0 for its -0.0s: the
    composition's torch.topk leaves the order of equal values open, so only there could a +-0.0 tie pick other bits"""
    import euler_b200
    g = env["g"]
    feat = np.nan_to_num(g["feat"], nan=0.75) + np.float32(0.0)
    gr = euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=1, node_type=g["node_type"],
                                   node_w=g["node_w"], cum_w=g["cum_w"], feat=feat, feat_slot_dims=list(SLOT_DIMS))
    euler_b200.set_graph(gr, rng="minstd", seed=1)
    return gr


@pytest.mark.parametrize("k,slot,dim", [(3, "feat1", 130), (4, "feat2", 1433), (1, "feat0", 3)])
def test_encoder_fused_matches_the_f64_composition(env, monkeypatch, k, slot, dim):
    import euler_b200
    from euler_b200.encoders import LGCEncoder
    _gr = _finite_graph(env)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)   # torch's default TF32 convolutions round at 1e-3
    seeds = torch.as_tensor(env["g"]["ids"][:256].astype(np.int64), device="cuda")
    torch.manual_seed(0)
    enc = LGCEncoder([0], slot, dim, k, 32, 10, 16, device="cuda")
    ref = copy.deepcopy(enc).double()
    ref.fused = False
    euler_b200.seed(11)
    neighbors = euler_b200.sample_neighbor(seeds, [0], 10)[0]
    composed = copy.deepcopy(enc)
    composed.fused = False
    assert torch.equal(_bits(enc.top_k_rows(seeds, neighbors)), _bits(composed.top_k_rows(seeds, neighbors)))
    euler_b200.seed(11)
    out = enc(seeds)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).cuda()
    (out * w).sum().backward()
    _f64_features(monkeypatch)
    euler_b200.seed(11)
    want = ref(seeds)
    (want * w.double()).sum().backward()
    assert out.shape == (256, 16) and want.dtype == torch.float64
    _close(out, want, "forward")
    for (n, p), (_, q) in zip(enc.named_parameters(), ref.named_parameters()):
        _close(p.grad, q.grad, n)


def test_lgcn_step_against_the_composition(env):
    import euler_b200
    from euler_b200.supervised import LGCN
    _gr = _finite_graph(env)
    seeds = torch.as_tensor(env["g"]["ids"][:512].astype(np.int64), device="cuda")
    torch.manual_seed(0)
    model = LGCN(32, [0], "feat0", 3, feature_idx="feat1", feature_dim=130, k=3, nb_num=10, out_dim=16, device="cuda")
    ref = copy.deepcopy(model)
    ref._encoder.fused = False
    steps = []
    for m in (model, ref):
        opt = torch.optim.SGD(m.parameters(), lr=0.5)
        euler_b200.seed(3)
        emb, loss, name, metric = m(seeds)
        opt.zero_grad()
        loss.backward()
        opt.step()
        steps.append((emb, loss, name, metric, [p.detach().clone() for p in m.parameters()]))
    (emb, loss, name, metric, params), (emb_r, loss_r, _, metric_r, params_r) = steps
    assert emb.shape == (512, 16) and name == "f1" and 0 <= float(metric) <= 1
    _close(emb, emb_r, "embedding")
    assert abs(loss.item() - loss_r.item()) <= 1e-6 * abs(loss_r.item())
    assert float(metric) == float(metric_r)
    for a, b in zip(params, params_r):
        _close(a, b, "updated parameter")
