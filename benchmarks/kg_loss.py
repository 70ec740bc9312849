#!/usr/bin/env python
"""The knowledge-graph embedding step on one H100: the fused op (ops.kg_margin_loss) against the literal torch composition of
upstream's TransX / DistMult code (knowledge.composed_kg_loss: tile, normalise, project, norm, hinge, stable sort).

    python benchmarks/kg_loss.py [--steps K] [--warmup W] [--only W1,W2,W3]

Workloads:
  W1  training at upstream's TransX README configuration: an FB15k-shaped graph (14 951 entities, 1 345 relations with Zipf-like
      frequencies, 483 142 train triples) built from a seed with Graph.from_csr + set_edges; B = 1200 triples from sample_edge,
      relation ids from the 'id' edge feature, K = 1 from sample_node, dim 50, margin 0.5, corrupt 'both'; fwd and fwd_bwd;
      all five models.
  W2  training at scale: tables of 10M entities and 1 000 relations; B = 8192 triples, K = 64, dim 128; the ids are drawn from
      the seed directly (uniform entities, Zipf relations) rather than from a 100M-triple graph, which the op never reads;
      fwd_bwd with dense and with sparse gradients (the composition: dense); TransE, TransR, DistMult.
  W3  evaluation as run_mode='evaluate' runs it: the FB15k-shaped graph, B = 128, K = 14 951, 'both', dim 100, forward only
      (the mr and hit10 metrics); all five models.
A GATE runs first: on W1's shapes, every model's fused loss and gradients against the float64 composition (loss within 1e-6,
gradients within 1e-5 of the largest entry).  The arms alternate round by round in one process; each reports the median ms
per call over --steps calls after --warmup, and the torch allocator's peak above the inputs during one call (the fused op's
ctx scratch is reported beside: the growth of the device's used memory outside torch).  A composed arm whose tensors cannot
fit is reported "not run" with its largest tiled tensor estimated from the shapes.  The card's name and power limit are read
in the same run.  One JSON line on stdout."""
import argparse

import harness
import numpy as np


MODELS = ('transe', 'transh', 'transr', 'transd', 'distmult')
SEED = 20201


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--only", default="W1,W2,W3")
    return p.parse_args(argv)


def fb15k_graph():
    """an FB15k-shaped knowledge graph from the seed: entities of node type 0, train triples of edge type 0 whose relation id
    (Zipf-like, exponent 1.1) is the dense edge feature 'id'"""
    import euler_b200 as eb
    rng = np.random.RandomState(SEED)
    n_ent, n_rel, n_tri = 14951, 1345, 483142
    p = 1.0 / np.arange(1, n_rel + 1) ** 1.1
    rel = rng.choice(n_rel, size=n_tri, p=p / p.sum())
    src, dst = rng.randint(0, n_ent, n_tri), rng.randint(0, n_ent, n_tri)
    order = np.lexsort((dst, src))
    src, dst, rel = src[order], dst[order], rel[order]
    ptr = np.zeros(n_ent + 1, np.int64)
    np.add.at(ptr, src + 1, 1)
    g = eb.Graph.from_csr(np.arange(n_ent), np.cumsum(ptr), dst, w=np.ones(n_tri, np.float32))
    g.set_edges(src, dst, np.zeros(n_tri, np.int32), dense=rel.reshape(-1, 1).astype(np.float32), dense_names=['id'])
    eb.set_graph(g, rng="minstd", seed=SEED)
    return g, n_ent, n_rel


def graph_ids(B, K):
    import torch
    import euler_b200 as eb
    edges = eb.sample_edge(B, 0)
    rel = eb.get_edge_dense_feature(edges, ['id'], [1])[0].to(torch.int64).reshape(B)
    neg = eb.sample_node(B * K, 0).reshape(B, K)
    return edges[:, 0].contiguous(), edges[:, 1].contiguous(), neg, rel


def make_tables(model, n_ent, n_rel, ent_dim, rel_dim, grad=True):
    import torch
    g = torch.Generator(device="cuda").manual_seed(SEED)

    def t(r, c):
        return (torch.randn(r, c, device="cuda", generator=g) * 0.1).requires_grad_(grad)
    tabs = [t(n_ent + 2, ent_dim), t(n_rel + 2, rel_dim)]
    tabs += {'transh': lambda: [t(n_rel + 2, ent_dim)], 'transr': lambda: [t(n_rel + 2, ent_dim * rel_dim)],
             'transd': lambda: [t(n_ent + 2, ent_dim), t(n_rel + 2, rel_dim)]}.get(model, lambda: [])()
    return tabs


def call(kind, model, tabs, ids, arm, margin, metric, sparse=False):
    import torch
    import euler_b200 as eb
    from euler_b200.knowledge import composed_kg_loss
    src, dst, neg, rel = ids
    with torch.set_grad_enabled(arm != "fwd"):
        if kind == "fused":
            loss, m = eb.kg_margin_loss(src, dst, neg, rel, tabs, model, l1=True, corrupt='both', margin=margin, metric=metric,
                                        sparse_grad=sparse)
        else:
            loss, m, _ = composed_kg_loss(model, tabs, src, dst, neg, rel, l1=True, corrupt='both', margin=margin, metric=metric)
        if arm != "fwd":
            for t in tabs:
                t.grad = None
            loss.backward()
    return loss, m


def gate(ids, n_ent, n_rel):
    """fused against the float64 composition on W1's shapes, every model"""
    import torch
    from euler_b200.knowledge import composed_kg_loss
    out = {}
    for model in MODELS:
        tabs = make_tables(model, n_ent, n_rel, 50, 50)
        loss, _ = call("fused", model, tabs, ids, "fwd_bwd", 0.5, "mrr")
        g = [t.grad.clone() for t in tabs]
        t64 = [t.detach().double().requires_grad_(True) for t in tabs]
        l64, _, _ = composed_kg_loss(model, t64, *ids, l1=True, corrupt='both', margin=0.5)
        l64.backward()
        lerr = abs(float(loss) - float(l64)) / max(1e-30, abs(float(l64)))
        gerr = max(float((a.double() - b.grad).abs().max() / b.grad.abs().max().clamp_min(1e-30)) for a, b in zip(g, t64))
        out[model] = {"loss_rel_err": lerr, "grad_rel_err": gerr}
        if lerr > 1e-6 or gerr > 1e-5:
            raise SystemExit("GATE failed for %s: %s" % (model, out[model]))
        del tabs, t64
        torch.cuda.empty_cache()
    return out


def measure(arms, steps, warmup):
    """arms: name -> thunk.  Alternate the arms round by round; median ms per call and the allocator peak above the inputs."""
    import torch
    res = {}
    for name, fn in arms.items():
        try:
            peak, outside = harness.memory_of(fn)
            res[name] = {"peak_mb": round(peak / 2**20, 1), "ctx_scratch_mb": round(max(0, outside) / 2**20, 1)}
        except torch.OutOfMemoryError:
            res[name] = {"not_run": "out of memory"}
            torch.cuda.empty_cache()
    live = {n: fn for n, fn in arms.items() if "not_run" not in res[n]}
    for n, ms in harness.time_arms(live, steps, warmup).items():
        res[n]["ms_median"] = round(float(np.median(ms)), 3)
    return res


def main(argv=None):
    import torch
    args = parse(argv)
    only = set(args.only.split(","))
    out = {"gpu": harness.gpu_info(torch.cuda.current_device())}
    g, n_ent, n_rel = fb15k_graph()
    torch.manual_seed(SEED)
    w1 = graph_ids(1200, 1)
    out["gate"] = gate(w1, n_ent, n_rel)
    if "W1" in only:
        r = {}
        for model in MODELS:
            tabs = make_tables(model, n_ent, n_rel, 50, 50)
            arms = {"%s_%s" % (kind, arm): (lambda kind=kind, arm=arm: call(kind, model, tabs, w1, arm, 0.5, "mrr"))
                    for arm in ("fwd", "fwd_bwd") for kind in ("fused", "composed")}
            r[model] = measure(arms, args.steps, args.warmup)
            del tabs
            torch.cuda.empty_cache()
        out["W1"] = r
    if "W2" in only:
        rng = np.random.RandomState(SEED + 2)
        B, K, N, R = 8192, 64, 10_000_000, 1000
        p = 1.0 / np.arange(1, R + 1) ** 1.1
        d = lambda a: torch.as_tensor(a, dtype=torch.int64, device="cuda")   # noqa: E731
        w2 = (d(rng.randint(0, N, B)), d(rng.randint(0, N, B)), d(rng.randint(0, N, (B, K))), d(rng.choice(R, B, p=p / p.sum())))
        r = {}
        for model in ('transe', 'transr', 'distmult'):
            tabs = make_tables(model, N, R, 128, 128)
            arms = {"%s_%s" % (kind, arm): (lambda kind=kind, arm=arm: call(kind, model, tabs, w2, "fwd_bwd", 1.0, "mrr",
                                                                            sparse=arm == "sparse"))
                    for arm, kind in (("dense", "fused"), ("sparse", "fused"), ("dense", "composed"))}
            if model == 'transr':
                est = B * K * 128 * 128 * 4 / 2**30
                arms = {k: v for k, v in arms.items() if k.startswith("fused")}
                r["transr_composed"] = "not run: the tiled [B, K, ent_dim * rel_dim] matrix alone is %.1f GB" % est
            r[model] = measure(arms, args.steps, args.warmup)
            del tabs
            torch.cuda.empty_cache()
        out["W2"] = r
    if "W3" in only:
        w3 = graph_ids(128, 14951)
        r = {}
        for model in MODELS:
            tabs = make_tables(model, n_ent, n_rel, 100, 100, grad=False)
            arms = {"%s_%s" % (kind, metric): (lambda kind=kind, metric=metric: call(kind, model, tabs, w3, "fwd", 1.0, metric))
                    for metric in ("mr", "hit10") for kind in ("fused", "composed")}
            if model == 'transr':
                est = 128 * 14951 * 100 * 100 * 4 / 2**30
                arms = {k: v for k, v in arms.items() if k.startswith("fused")}
                r["transr_composed"] = "not run: the tiled [B, K, ent_dim * rel_dim] matrix alone is %.1f GB" % est
            r[model] = measure(arms, args.steps, args.warmup)
            del tabs
            torch.cuda.empty_cache()
        out["W3"] = r
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    main()
