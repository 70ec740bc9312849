"""GPU: the fused graph auto-encoder step (ops.gae_loss: eu_gae_loss and its backward pass) against float64 restatements of
base_gae.py / gae.py, its determinism, CUDA-graph replay and refusals, and whole GAE / VGAE training steps over SageEncoder
and GCNEncoder, fused against fused=False on the same draws."""
import copy

import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eb():
    import euler_b200
    g = graphs.random_graph(seed=3, n=500, T=1, avg_deg=4, feat_dim=8)
    euler_b200.set_graph(graphs.cuda_graph(g), rng="minstd", seed=1)
    return euler_b200


def _rows(shape, gen, scale, offset):
    """f32 rows of `shape` on the device, 4 bytes past a 16-byte boundary when offset"""
    n = int(np.prod(shape))
    buf = torch.randn(n + 1, generator=gen, device="cuda") * scale
    return (buf[1:] if offset else buf[:n]).view(shape)


def _problem(B, K, D, variational, offset, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    shapes = [(B, D), (B, K, D), (B, K, D)]
    mu = [_rows(s, gen, D ** -0.5, offset) for s in shapes]
    lv = [_rows(s, gen, 0.3, offset) for s in shapes] if variational else None
    nz = [_rows(s, gen, 1.0, offset) for s in shapes] if variational else None
    return mu, lv, nz


def _z64(mu, lv, nz, radius):
    """the float64 rows z = mu + radius noise sqrt(exp(log_var)) of the three sets"""
    z = [m.double() for m in mu]
    if lv is not None and nz is not None:
        z = [m + radius * n.double() * torch.sqrt(torch.exp(v.double())) for m, v, n in zip(z, lv, nz)]
    return z


def _restated(mu, lv, nz, radius):
    """base_gae.py / gae.py in float64: (loss, logits [B, 2K], mag [B, 2K]).  mag bounds what f32 rounding can move a logit
    by, in units of the rounding: the dot of the rows' magnitudes, each element |mu| + |radius noise sqrt(exp(log_var))|,
    since the f32 sum forming z rounds relative to its terms, not to z"""
    e, p, n = _z64(mu, lv, nz, radius)
    logits = torch.cat([torch.einsum('bd,bkd->bk', e, p), torch.einsum('bd,bkd->bk', e, n)], 1)
    ae, ap, an = [m.double().abs() + (z - m.double()).abs() for m, z in zip(mu, (e, p, n))]
    mag = torch.cat([torch.einsum('bd,bkd->bk', ae, ap), torch.einsum('bd,bkd->bk', ae, an)], 1)
    K = p.shape[1]
    z = torch.zeros_like(logits)
    z[:, :K] = 1
    loss = (logits.clamp(min=0) - logits * z + torch.log1p(torch.exp(-logits.abs()))).mean()
    if lv is not None:
        loss = loss + torch.cat([(-0.5 * (v.double() - torch.exp(v.double()) - m.double() ** 2 + 1)).reshape(-1)
                                 for m, v in zip(mu, lv)]).mean()
    return loss, logits, mag


def _composed_correct(logits, K):
    label = torch.zeros_like(logits)
    label[:, :K] = 1
    return int((torch.floor(torch.sigmoid(logits) + 0.5) == label).sum())


def _bits(t):
    return t.detach().contiguous().view(torch.int32) if t.dtype == torch.float32 else t.detach()


@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("variational", [False, True])
@pytest.mark.parametrize("D", [1, 3, 4, 16, 32, 128, 200])
def test_forward_against_float64(eb, D, variational, offset):
    for K in (1, 5, 10, 64):
        for B in (0, 1, 7, 4097):
            mu, lv, nz = _problem(B, K, D, variational, offset, seed=D * 131 + K * 7 + B)
            radius = 0.7
            loss, correct, logits = eb.gae_loss(*mu, log_var=lv, noise=nz, radius=radius, return_logits=True)
            what = "B=%d K=%d D=%d" % (B, K, D)
            assert logits.shape == (B, 2 * K) and correct.dtype == torch.int64, what
            if B == 0:
                assert torch.isnan(loss) and int(correct) == 0, what
                continue
            w_loss, w_logits, mag = _restated(mu, lv, nz, radius)
            assert abs(float(loss) - float(w_loss)) <= 1e-6 * abs(float(w_loss)), (what, float(loss), float(w_loss))
            assert bool(((logits.double() - w_logits).abs() <= 1e-6 * mag + 1e-30).all()), what
            assert int(correct) == _composed_correct(logits, K), what


def test_extreme_logits_are_finite(eb):
    # source [10, 0, 0, 0]; contexts 10, -10 and 0 in column 0: logits +100, -100 and exactly 0, as positives and negatives
    B, K, D = 2, 3, 4
    emb = torch.zeros(B, D, device="cuda")
    emb[:, 0] = 10
    vals = torch.tensor([10.0, -10.0, 0.0], device="cuda")
    pos = torch.zeros(B, K, D, device="cuda")
    pos[:, :, 0] = vals
    neg = pos.flip(1).contiguous()
    loss, correct, logits = eb.gae_loss(emb, pos, neg, return_logits=True)
    assert torch.isfinite(loss)
    assert logits[0].tolist() == [100.0, -100.0, 0.0, 0.0, -100.0, 100.0]
    w_loss, _, _ = _restated([emb, pos, neg], None, None, 0.0)
    assert abs(float(loss) - float(w_loss)) <= 1e-6 * float(w_loss)
    assert int(correct) == _composed_correct(logits, K) == B * 3   # +100 and 0 are predicted 1, -100 is predicted 0
    g = torch.autograd.grad(eb.gae_loss(emb.requires_grad_(), pos, neg)[0], emb)[0]
    assert torch.isfinite(g).all()


def _grads(eb, mu, lv, nz, radius):
    """the fused op's gradients of mu (and log_var)"""
    leaves = [t.detach().clone().requires_grad_() for t in mu + (lv or [])]
    loss, _ = eb.gae_loss(*leaves[:3], log_var=leaves[3:] or None, noise=nz, radius=radius)
    return loss, torch.autograd.grad(loss, leaves)


def _composed_grads(mu, lv, nz, radius, dtype):
    """autograd through the literal composition (gae.py's reparameterisation, PosNegLogits, xent_loss, kl) in dtype"""
    from euler_b200 import autoencoder as ae
    leaves = [t.detach().to(dtype).clone().requires_grad_() for t in mu + (lv or [])]
    m, v = leaves[:3], leaves[3:]
    z = m if not v or nz is None else [a + radius * n.to(dtype) * torch.sqrt(torch.exp(b)) for a, b, n in zip(m, v, nz)]
    loss, _ = ae.composed_gae_loss(z[0].unsqueeze(1), z[1], z[2])
    if v:
        loss = loss + torch.cat([ae.kl(a, b) for a, b in zip(m, v)]).mean()
    return loss, torch.autograd.grad(loss, leaves)


def _close(got, want, what, tol=1e-5):
    scale = max(float(want.abs().max()), 1e-30)
    err = float((got.double() - want.double()).abs().max())
    assert err <= tol * scale, "%s: error %g, largest entry %g" % (what, err, scale)


@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("form", ["gae", "vgae", "vgae_eval"])
@pytest.mark.parametrize("B,K,D", [(1, 1, 1), (7, 5, 3), (7, 10, 32), (300, 10, 128), (64, 64, 200)])
def test_backward_against_float64(eb, B, K, D, form, offset):
    mu, lv, nz = _problem(B, K, D, form != "gae", offset, seed=B + K + D)
    if form == "vgae_eval":
        nz = None
    radius = 0.8
    loss, got = _grads(eb, mu, lv, nz, radius)
    _, want = _composed_grads(mu, lv, nz, radius, torch.float64)
    _, comp = _composed_grads(mu, lv, nz, radius, torch.float32)
    names = ["emb", "pos", "neg", "log_var emb", "log_var pos", "log_var neg"]
    for name, g, w, c in zip(names, got, want, comp):
        assert g.shape == w.shape
        _close(g, w, "%s vs float64" % name)
        _close(g, c, "%s vs the float32 composition" % name)


def test_bits_repeat_and_graph_replay_equals_eager(eb):
    B, K, D = 513, 10, 32
    mu, lv, nz = _problem(B, K, D, True, False, seed=4)
    runs = []
    for _ in range(2):
        loss, g = _grads(eb, mu, lv, nz, 1.0)
        runs.append([loss] + list(g))
    for a, b in zip(*runs):
        assert torch.equal(_bits(a), _bits(b))
    from euler_b200 import ops
    logits = torch.empty(B, 2 * K, device="cuda")
    loss = torch.empty((), device="cuda")
    correct = torch.empty((), dtype=torch.int64, device="cuda")
    gl = torch.ones(1, device="cuda")
    g_mu = [torch.empty_like(t) for t in mu]
    g_lv = [torch.empty_like(t) for t in mu]

    def step():
        ops._call("eu_gae_loss", B, K, D, mu, lv, nz, 1.0, logits, loss, correct)
        ops._call("eu_gae_loss_backward", gl, B, K, D, mu, lv, nz, 1.0, logits, g_mu, g_lv)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        eager = [t.clone() for t in [logits, loss, correct] + g_mu + g_lv]
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            step()
    torch.cuda.current_stream().wait_stream(s)
    for t in [logits, loss, correct] + g_mu + g_lv:
        t.fill_(7)
    cg.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, [logits, loss, correct] + g_mu + g_lv):
        assert torch.equal(_bits(a), _bits(b))
    assert torch.equal(_bits(eager[1]), _bits(runs[0][0]))


def test_refusals_leave_the_outputs_untouched(eb):
    from euler_b200 import _lib, ops
    lib = _lib.load()
    B, K, D = 4, 2, 8
    mu, lv, nz = _problem(B, K, D, True, False, seed=9)
    logits = torch.full((B, 2 * K), 7.0, device="cuda")
    loss = torch.full((), 7.0, device="cuda")
    correct = torch.full((), 7, dtype=torch.int64, device="cuda")
    gl = torch.ones(1, device="cuda")
    g_mu = [torch.full_like(t, 7.0) for t in mu]
    g_lv = [torch.full_like(t, 7.0) for t in mu]
    h = ops._ctx_on_stream()._h
    a = ops._arg
    bad = [  # (B, K, D, mu, lv, nz, radius)
        (B, 0, D, mu, lv, nz, 1.0), (-1, K, D, mu, lv, nz, 1.0), (B, K, 0, mu, lv, nz, 1.0),
        (B, K, D, mu, lv, nz, float("nan")), (B, K, D, mu, lv, nz, float("inf")), (B, K, D, mu, None, nz, 1.0),
        (B, K, D, [mu[0], None, mu[2]], lv, nz, 1.0), (B, K, D, mu, [lv[0], lv[1], None], nz, 1.0), (B, K, D, None, lv, nz, 1.0)]
    for Bx, Kx, Dx, m, v, n, r in bad:
        rc = lib.eu_gae_loss(h, Bx, Kx, Dx, a(m), a(v), a(n), r, a(logits), a(loss), a(correct))
        assert rc == 1, (Bx, Kx, Dx, r)
        rc = lib.eu_gae_loss_backward(h, a(gl), Bx, Kx, Dx, a(m), a(v), a(n), r, a(logits), a(g_mu), a(g_lv))
        assert rc == 1, (Bx, Kx, Dx, r)
    assert lib.eu_gae_loss(h, B, K, D, a(mu), a(lv), a(nz), 1.0, a(logits), None, a(correct)) == 1
    assert lib.eu_gae_loss_backward(h, a(gl), B, K, D, a(mu), a(lv), a(nz), 1.0, a(logits), a(g_mu), None) == 1
    assert lib.eu_gae_loss(h, B, 1 << 29, D, a(mu), a(lv), a(nz), 1.0, a(logits), a(loss), a(correct)) == 4
    torch.cuda.synchronize()
    for t in [logits, loss] + g_mu + g_lv:
        assert bool((t == 7.0).all())
    assert int(correct) == 7
    with pytest.raises(eb.EulerError):
        eb.gae_loss(mu[0], mu[1], mu[1][:, :1].contiguous())
    with pytest.raises(eb.EulerError):
        eb.gae_loss(*mu, log_var=lv, noise=nz, radius=float("nan"))


# ---------------------------------------------------------------------------- whole steps over the device encoders
N_NODES, FEAT, DIM = 3000, 16, 32


@pytest.fixture(scope="module")
def rmat():
    import euler_b200
    g = euler_b200.Graph.rmat(N_NODES, 30000, seed=42, feat_dim=FEAT, device=0)
    euler_b200.set_graph(g, rng="minstd", seed=5)
    return euler_b200


def _encoder(kind):
    from euler_b200 import encoders
    torch.manual_seed(0)
    if kind == "sage":
        return encoders.SageEncoder([[0], [0]], [10, 10], DIM, 'mean', feature_idx=0, feature_dim=FEAT, max_id=N_NODES,
                                    device="cuda")
    return encoders.GCNEncoder([[0], [0]], DIM, 'gcn', feature_idx=0, feature_dim=FEAT, device="cuda")


def _recorded(model):
    """model with its to_sample draws kept in model.draws"""
    model.draws = []
    inner = model.to_sample

    def to_sample(inputs):
        out = inner(inputs)
        model.draws.append(out)
        return out
    model.to_sample = to_sample
    return model


@pytest.mark.parametrize("variational", [False, True])
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_training_step_fused_equals_composed(rmat, kind, variational):
    from euler_b200 import autoencoder as ae
    enc = _encoder(kind)
    steps = []
    inputs = torch.as_tensor(np.random.RandomState(3).randint(1, N_NODES + 1, size=256), device="cuda")
    for fused in (True, False):
        gen = torch.Generator(device="cuda").manual_seed(17)
        e = copy.deepcopy(enc)
        if variational:
            torch.manual_seed(1)
            model = ae.VariationalGraphAutoEncoder(1.0, e, 0, [0], N_NODES, num_negs=10, generator=gen, fused=fused,
                                                   device="cuda")
        else:
            model = ae.GraphAutoEncoder(e, 0, [0], N_NODES, num_negs=10, fused=fused)
        model = _recorded(model)
        opt = torch.optim.Adam(model.parameters(), lr=0.01)
        rmat.seed(23)
        emb, loss, name, acc = model(inputs)
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        opt.step()
        steps.append((model.draws[0], emb.detach(), loss.detach(), acc, grads))
    (da, ea, la, aa, ga), (db, eb_, lb, ab, gb) = steps
    for x, y in zip(da, db):
        assert torch.equal(x, y)                     # the same ids, bit for bit
    assert ea.shape == (256, 1, DIM)
    _close(la, lb, "loss")
    assert abs(float(aa) - float(ab)) <= 1.0 / (2 * 256 * 10) + 1e-7   # at most one logit on the other side of 0.5
    assert set(ga) == set(gb) and len(ga) > 0
    for k in ga:
        _close(ga[k], gb[k], "grad " + k)
