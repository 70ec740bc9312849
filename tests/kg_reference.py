"""The knowledge-graph step's test helpers: random device tables and ids, one raw eu_kg_loss call, and the float64 autograd
of knowledge.composed_kg_scores (the torch composition of upstream's models) that the GPU tests of ops.kg_margin_loss compare
against.  (Test infrastructure.)"""
import torch


def tables(model, n_ent, n_rel, ent_dim, rel_dim, rng, offset=0):
    """random f32 tables on the device; offset shifts each data pointer off a 16-byte boundary"""
    def t(rows, cols):
        v = torch.tensor(rng.randn(rows * cols + offset) * 0.3, dtype=torch.float32).cuda()
        return v[offset:].view(rows, cols)
    tabs = [t(n_ent, ent_dim), t(n_rel, rel_dim)]
    if model == 'transh':
        tabs.append(t(n_rel, ent_dim))
    elif model == 'transr':
        tabs.append(t(n_rel, ent_dim * rel_dim))
    elif model == 'transd':
        tabs += [t(n_ent, ent_dim), t(n_rel, rel_dim)]
    return tabs


def ids(rng, B, K, n_ent, n_rel):
    d = lambda a: torch.as_tensor(a, dtype=torch.int64).cuda()   # noqa: E731
    return (d(rng.randint(0, n_ent - 4, size=B)), d(rng.randint(0, n_ent - 4, size=B)),
            d(rng.randint(0, n_ent - 4, size=(B, K))), d(rng.randint(0, n_rel - 1, size=B)))   # the last rows stay untouched


def raw(model, tabs, src, dst, neg, rel, l1, corrupt, margin, with_emb=False):
    """one eu_kg_loss: (scores, rank, loss, embeddings or None)"""
    from euler_b200 import ops
    m = ops.KG_MODELS[model]
    slots = [None] * 4
    for t, tb in zip(ops._KG_SLOTS[m], tabs):
        slots[t] = tb
    cfg = (m, l1, ops.KG_CORRUPT[corrupt], margin, tabs[0].shape[1], tabs[1].shape[1], False, with_emb)
    return ops._raw_kg(*slots, src, dst, rel, neg, cfg)


def ref64(model, tabs, src, dst, neg, rel, l1, corrupt, margin):
    """float64: (pos [B, 1], neg [B, C K], loss, every table's gradient, the embeddings)"""
    from euler_b200.knowledge import composed_kg_scores
    t64 = [t.detach().double().requires_grad_(True) for t in tabs]
    pos, negs, emb = composed_kg_scores(model, t64, src, dst, neg, rel, l1=l1, corrupt=corrupt)
    B = pos.shape[0]
    loss = torch.clamp(margin + negs.reshape(B, -1).mean(-1, keepdim=True).reshape(-1, 1, 1) - pos, min=0).mean()
    loss.backward()
    return pos.reshape(B, 1), negs.reshape(B, -1), loss, [t.grad for t in t64], emb


def rel_err(a, b):
    """the largest difference relative to b's largest entry"""
    b = b.detach().double().cpu()
    return float((a.detach().double().cpu() - b).abs().max() / max(1e-12, float(b.abs().max())))


def check_against_float64(model, tabs, src, dst, neg, rel, l1, corrupt, margin, absolute=False):
    """The fused step against float64: scores and loss within 1e-6; ranks exact; every table's gradient within 1e-5 of
    float64 autograd, bit-identical run to run, zero on untouched rows, and the sparse COO equal to the dense rows.  absolute:
    hold the embeddings and gradients to an absolute 1e-4 instead (dim 1, where f32 leaves a cancellation residue of about
    eps |gy| / |x| on entries whose exact gradient is 0).  Returns the scores."""
    from euler_b200 import ops
    what = (model, l1, corrupt, tabs[0].shape[1], tabs[1].shape[1], neg.shape[1])
    n_ent, n_rel = tabs[0].shape[0], tabs[1].shape[0]
    scores, rank, loss, embs = raw(model, tabs, src, dst, neg, rel, l1, corrupt, margin, with_emb=True)
    pos64, neg64, loss64, grads64, emb64 = ref64(model, tabs, src, dst, neg, rel, l1, corrupt, margin)
    s64 = torch.cat([pos64, neg64], 1).detach()
    assert rel_err(scores, s64) <= 1e-6, what
    assert abs(float(loss) - float(loss64.detach())) <= 1e-6 * abs(float(loss64)), what

    def close(a, b, tol):
        if not absolute:
            return rel_err(a, b) <= tol
        return float((a.detach().double().cpu() - b.detach().double().cpu()).abs().max()) <= 1e-4
    for e, e64 in zip(embs, emb64):
        assert close(e, e64, 1e-6), what
    sc = scores.cpu()
    own = (sc[:, 1:] >= sc[:, :1]).sum(1)
    assert torch.equal(rank.cpu().long(), own), what
    s64c = s64.cpu()
    far = ((s64c[:, 1:] - s64c[:, :1]).abs() > 1e-5).all(1)
    assert torch.equal(own[far], (s64c[far, 1:] >= s64c[far, :1]).sum(1)), what

    t = [tb.clone().requires_grad_(True) for tb in tabs]
    runs = []
    for _ in range(2):
        for x in t:
            x.grad = None
        l, _m = ops.kg_margin_loss(src, dst, neg, rel, t, model, l1=l1, corrupt=corrupt, margin=margin)
        l.backward()
        runs.append([x.grad.clone() for x in t])
    touched_ent = torch.zeros(n_ent, dtype=torch.bool)
    touched_ent[torch.cat([src, dst, neg.reshape(-1)]).cpu()] = True
    touched_rel = torch.zeros(n_rel, dtype=torch.bool)
    touched_rel[rel.cpu()] = True
    for k, (g, g2, g64) in enumerate(zip(runs[0], runs[1], grads64)):
        assert g.cpu().numpy().tobytes() == g2.cpu().numpy().tobytes(), what + (k,)
        assert close(g, g64, 1e-5), what + (k, rel_err(g, g64))
        touched = touched_ent if g.shape[0] == n_ent else touched_rel
        assert not g.cpu()[~touched].any(), what + (k,)
    for x in t:
        x.grad = None
    l, _m = ops.kg_margin_loss(src, dst, neg, rel, t, model, l1=l1, corrupt=corrupt, margin=margin, sparse_grad=True)
    l.backward()
    for k, (x, g) in enumerate(zip(t, runs[0])):
        assert x.grad.is_sparse and x.grad.coalesce()._nnz() == x.grad._nnz(), what + (k,)   # one entry per distinct row
        assert x.grad.to_dense().cpu().numpy().tobytes() == g.cpu().numpy().tobytes(), what + (k,)
    return scores
