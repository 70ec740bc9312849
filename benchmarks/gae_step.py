#!/usr/bin/env python
"""One GAE and one VGAE training step (euler_b200/autoencoder.py) on one H100, and the auto-encoder loss alone, fused
(ops.gae_loss) against the torch composition of base_gae.py / gae.py.

    python benchmarks/gae_step.py [--steps K] [--warmup W] [--nodes N --edges E]

Graph: the R-MAT of BASELINE configs[1] (10M nodes / 100M edges) with a dense slot of 128 columns.  The example's shape
(examples/gae: dims [32, 32, 32], 2 layers, fanouts [10, 10], num_negs 10, batch 1024) and the same at dim 128: the
encoder is SageEncoder([[0], [0]], [10, 10], dim, 'mean') or GCNEncoder([[0], [0]], dim, 'gcn') over the slot's first dim
columns.  A step is forward, backward and one Adam step, with fused=True (the default) and fused=False.  The loss alone
times ops.gae_loss's forward and backward against the composition's on random rows of the step's shapes.
A GATE first: at each shape the fused step's loss, and every parameter's gradient, within 1e-4 of the largest entry of the
fused=False step's on the same draws; a mismatch aborts.  tests/test_gae_gpu.py checks the op against float64 at 1e-6.
Reported per arm: ms per call and torch's allocator peak above the inputs; the card's name, power limit and max SM clock read
in the same run.  One JSON line on stdout.  It needs a GPU: without one it fails rather than measure anything else."""
import argparse
import time

import harness
import numpy as np
from harness import timed


FEAT, DIMS, FANOUTS, NEGS, BATCH = 128, (32, 128), [10, 10], 10, 1024
MODELS, ENCODERS = ("gae", "vgae"), ("sage", "gcn")


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    return p.parse_args(argv)


def make_model(args, model, encoder, dim, fused):
    from euler_b200 import autoencoder, encoders
    torch.manual_seed(0)
    if encoder == "sage":
        enc = encoders.SageEncoder([[0]] * len(FANOUTS), FANOUTS, dim, 'mean', feature_idx=0, feature_dim=dim, max_id=args.nodes,
                                   device="cuda")
    else:
        enc = encoders.GCNEncoder([[0]] * len(FANOUTS), dim, 'gcn', feature_idx=0, feature_dim=dim, device="cuda")
    if model == "gae":
        m = autoencoder.GraphAutoEncoder(enc, 0, [0], args.nodes, num_negs=NEGS, fused=fused)
    else:
        m = autoencoder.VariationalGraphAutoEncoder(1.0, enc, 0, [0], args.nodes, num_negs=NEGS, fused=fused, device="cuda",
                                                    generator=torch.Generator(device="cuda").manual_seed(3))
    return m, torch.optim.Adam(m.parameters(), lr=0.01)


def step(eb, m, opt, seeds, seed=5):
    eb.seed(seed)
    opt.zero_grad(set_to_none=True)
    _, loss, _, acc = m(seeds)
    loss.backward()
    opt.step()
    return loss, acc


def gate(eb, args, seeds):
    for model in MODELS:
        for encoder in ENCODERS:
            for dim in DIMS:
                res = []
                for fused in (True, False):
                    m, _ = make_model(args, model, encoder, dim, fused)
                    eb.seed(5)
                    _, loss, _, _ = m(seeds)
                    params = [p for p in m.parameters() if p.requires_grad]
                    res.append((loss.detach(), torch.autograd.grad(loss, params, allow_unused=True)))
                    del m
                (a, ga), (b, gb) = res
                what = "%s over %s at dim %d" % (model, encoder, dim)
                if float((a - b).abs() / b.abs()) > 1e-4:
                    raise SystemExit("GATE FAILED: %s: the fused loss %r is not the composition's %r" % (what, float(a), float(b)))
                for t, (x, y) in enumerate(zip(ga, gb)):
                    if (x is None) != (y is None):
                        raise SystemExit("GATE FAILED: %s: parameter %d has a gradient on one path only" % (what, t))
                    if x is not None and float((x - y).abs().max()) > 1e-4 * float(y.abs().max()):
                        raise SystemExit("GATE FAILED: %s: parameter %d's gradient differs from the composition's" % (what, t))


def loss_arms(dim):
    """the loss alone at the step's shapes: forward + backward, fused and composed, GAE and VGAE"""
    from euler_b200 import autoencoder, ops
    gen = torch.Generator(device="cuda").manual_seed(dim)
    shapes = [(BATCH, dim), (BATCH, NEGS, dim), (BATCH, NEGS, dim)]
    mu = [(torch.randn(s, generator=gen, device="cuda") * dim ** -0.5).requires_grad_() for s in shapes]
    lv = [(torch.randn(s, generator=gen, device="cuda") * 0.1).requires_grad_() for s in shapes]
    nz = [torch.randn(s, generator=gen, device="cuda") for s in shapes]

    def fused(var):
        loss, _ = ops.gae_loss(*mu, log_var=lv if var else None, noise=nz if var else None, radius=1.0)
        torch.autograd.grad(loss, mu + (lv if var else []))

    def composed(var):
        z = [m + 1.0 * n * torch.sqrt(torch.exp(v)) for m, v, n in zip(mu, lv, nz)] if var else mu
        loss, _ = autoencoder.composed_gae_loss(z[0].unsqueeze(1), z[1], z[2])
        if var:
            loss = loss + torch.mean(torch.cat([autoencoder.kl(m, v) for m, v in zip(mu, lv)], 0))
        torch.autograd.grad(loss, mu + (lv if var else []))
    return {"loss_%s_d%d_%s" % (m, dim, k): (lambda f=f, v=(m == "vgae"): f(v))
            for m in MODELS for k, f in (("fused", fused), ("composed", composed))}


def run(args):
    global torch
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/gae_step.py needs a GPU; nothing is measured without one")
    import euler_b200 as eb
    torch.cuda.set_device(0)
    t0 = time.time()
    g = eb.Graph.rmat(args.nodes, args.edges, seed=42, feat_dim=FEAT, device=0)
    eb.set_graph(g, rng="minstd", seed=5)
    seeds = torch.from_numpy(np.random.RandomState(BATCH).randint(1, args.nodes + 1, size=BATCH).astype(np.int64)).cuda()
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    gate(eb, args, seeds)
    arms = {}
    for dim in DIMS:
        arms.update(loss_arms(dim))
    loss_res = timed(arms, max(args.steps * 10, 50), args.warmup)
    step_res = {}
    for model in MODELS:
        for encoder in ENCODERS:
            for dim in DIMS:
                pair = {}
                for fused in (True, False):
                    m, opt = make_model(args, model, encoder, dim, fused)
                    pair["step_%s_%s_d%d_%s" % (model, encoder, dim, "fused" if fused else "composed")] = \
                        (lambda m=m, opt=opt: step(eb, m, opt, seeds))
                step_res.update(timed(pair, args.steps, args.warmup))   # the two arms alternate round by round
                del pair, m, opt
    harness.emit({"metric": "gae_step_sage_d32_fused_ms", "value": step_res["step_gae_sage_d32_fused"]["ms_per_call"], "gate": "passed",
                  "gpu": harness.gpu_info(0), "batch": BATCH, "fanouts": FANOUTS, "dims": list(DIMS), "num_negs": NEGS, "setup_s": setup_s,
                  "steps": step_res, "loss_alone": loss_res})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
