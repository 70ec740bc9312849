#!/usr/bin/env python
"""ScalableSageEncoder's one-hop training step over per-layer embedding stores on one H100, against the SageEncoder step it
replaces, and the two store ops against their torch composition.

    python benchmarks/scalable_encoder.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Graph: the R-MAT of BASELINE configs[1] (10M nodes / 100M edges) with its dense slot of 128 columns (benchmarks/
shallow_encoder.py's graph).  Workload: batch 8192, dim 128, 'mean', 2 layers; the node encoder is the dense slot.  The
scalable encoder samples one hop of fanout 10 (81,920 neighbours) and reads layer 1's neighbour rows from a store of
[N + 2, 128] f32 (5.1 GB at 10M nodes, its gradient store as much again); SageEncoder samples fanouts [10, 10] (819,200
deepest-hop rows).  Both feed the same supervised head (Linear(128, 16), sigmoid cross-entropy on seeded labels) and SGD.
A GATE first, on the batch's own ids: store_exchange's taken rows equal the pre-call gather bit for bit, the written rows are
each id's last occurrence and the cleared rows zero; store_accumulate is within 1e-5 of a float64 index_add_; a mismatch
aborts.  Then, alternating in rounds in one process:
  (a) a ScalableSageEncoder training step (forward(training=True), loss, train_step);
  (b) a SageEncoder step (forward, loss, backward, SGD step), the same seeds;
  (c) the two store ops alone: store_exchange over the batch, store_accumulate over the hop (count 10, 'mean');
  (d) their torch composition: gather, index_put_ (no defined winner), index_put_ of zeros, index_add_.
Reported per arm: ms per call, torch's allocator peak above the inputs, and the store bytes computed from the shapes; the
card's name, power limit and max SM clock read in the same run.  One JSON line on stdout.  It needs a GPU: without one it
fails rather than measure anything else."""
import argparse
import time

import harness
import numpy as np
from harness import DENSE_DIM, build_graph, timed


LABELS = 16


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=8192)
    p.add_argument("--fanout", type=int, default=10)
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def shapes(args):
    """what the workload holds and moves, from its shapes alone"""
    table = (args.nodes + 2) * args.dim * 4
    return {"store_rows": args.nodes + 2, "store_bytes": table, "store_and_gradient_bytes": 2 * table,
            "hop_neighbours": args.batch * args.fanout, "sage_deepest_hop_rows": args.batch * args.fanout ** 2}


def gate(eb, store, grad_store, node, neighbor, dim):
    gen = torch.Generator(device="cuda").manual_seed(2)
    rows = torch.randn(node.numel(), dim, device="cuda", generator=gen)
    grad = torch.randn(node.numel(), dim, device="cuda", generator=gen)
    before = grad_store[node].clone()
    taken = eb.store_exchange(store, grad_store, node, rows)
    pos = torch.arange(node.numel(), device="cuda")
    last = torch.full((store.shape[0],), -1, dtype=torch.int64, device="cuda").scatter_reduce(0, node, pos, "amax")
    if not (torch.equal(taken, before) and torch.equal(store[node], rows[last[node]]) and not grad_store[node].any()):
        raise SystemExit("GATE FAILED: store_exchange differs from its definition")
    count = neighbor.numel() // node.numel()
    uniq = torch.unique(neighbor)
    want = grad_store[uniq].double().index_add_(0, torch.searchsorted(uniq, neighbor),
                                                 grad.double().repeat_interleave(count, 0) / count)
    eb.store_accumulate(grad_store, neighbor, grad, count, "mean")
    err = float((grad_store[uniq].double() - want).abs().max() / want.abs().max())
    if err > 1e-5:
        raise SystemExit("GATE FAILED: store_accumulate is %.3g of the largest entry from float64 index_add_" % err)


def run(args):
    global torch
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/scalable_encoder.py needs a GPU; nothing is measured without one")
    import euler_b200 as eb
    from euler_b200.encoders import SageEncoder, ScalableSageEncoder
    torch.cuda.set_device(0)
    sh = shapes(args)
    t0 = time.time()
    _g = build_graph(args)
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=args.batch).astype(np.int64)).cuda()
    labels = (torch.rand(args.batch, LABELS, generator=torch.Generator().manual_seed(3)) < 0.5).float().cuda()
    kw = dict(aggregator="mean", feature_idx="feat0", feature_dim=DENSE_DIM, max_id=args.nodes, device="cuda")
    torch.manual_seed(0)
    scal = ScalableSageEncoder([0], args.fanout, 2, args.dim, generator=torch.Generator(device="cuda").manual_seed(1), **kw)
    torch.manual_seed(0)
    sage = SageEncoder([[0], [0]], [args.fanout] * 2, args.dim, **kw)
    heads = {k: torch.nn.Linear(args.dim, LABELS).cuda() for k in ("scal", "sage")}
    opts = {"scal": torch.optim.SGD(list(scal.parameters()) + list(heads["scal"].parameters()), lr=0.01),
            "sage": torch.optim.SGD(list(sage.parameters()) + list(heads["sage"].parameters()), lr=0.01)}
    eb.seed(5)
    node, neighbor = eb.sample_fanout(seeds, [[0]], [args.fanout], default_node=args.nodes + 1)[0]
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    gate(eb, scal.stores[0], scal.gradient_stores[0], node, neighbor, args.dim)

    def loss_of(out, head):
        return torch.nn.functional.binary_cross_entropy_with_logits(head(out), labels)

    def scal_step():
        out = scal(seeds, training=True)
        scal.train_step(loss_of(out, heads["scal"]), opts["scal"])

    def sage_step():
        opts["sage"].zero_grad()
        loss_of(sage(seeds), heads["sage"]).backward()
        opts["sage"].step()

    gen = torch.Generator(device="cuda").manual_seed(4)
    rows = torch.randn(node.numel(), args.dim, device="cuda", generator=gen)
    grad = torch.randn(node.numel(), args.dim, device="cuda", generator=gen)
    store, grad_store = scal.stores[0], scal.gradient_stores[0]

    def store_ops():
        eb.store_exchange(store, grad_store, node, rows)
        eb.store_accumulate(grad_store, neighbor, grad, args.fanout, "mean")

    def store_ops_torch():
        grad_store[node]
        store.index_put_((node,), rows)
        grad_store.index_put_((node,), torch.zeros((), device="cuda"))
        grad_store.index_add_(0, neighbor, grad.repeat_interleave(args.fanout, 0) / args.fanout)

    arms = {"scalable_sage_step": scal_step, "sage_step": sage_step, "store_ops": store_ops, "store_ops_torch": store_ops_torch}
    res = timed(arms, args.steps, args.warmup)
    harness.emit({"metric": "scalable_sage_step_ms", "value": res["scalable_sage_step"]["ms_per_call"], "gate": "passed",
                  "gpu": harness.gpu_info(0), "batch": args.batch, "dim": args.dim, "fanout": args.fanout, "shapes": sh, "setup_s": setup_s,
                  "arms": res})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
