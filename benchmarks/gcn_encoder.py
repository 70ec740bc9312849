#!/usr/bin/env python
"""GCNEncoder on one H100: the neighbour mean over a hop's CSR adjacency (ops.adjacency_mean) against the two ways a user
would compose it (gather + scatter_add through an [nnz, D] message matrix, and torch.sparse.mm), alone and inside the
whole encoder.

    python benchmarks/gcn_encoder.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Graph: the R-MAT of benchmarks/full_dataflow.py (BASELINE configs[1], 10M nodes / 100M edges) with its dense slot of
D = 128 columns (built as benchmarks/shallow_encoder.py does).  Workload: batch 2048, metapath [[0], [0]], dim 128, the node
encoder the dense slot alone.  get_multi_hop_neighbor's adjacency of hop 1 (rows = the hop-1 nodes, columns = the hop-2
nodes) lists the batch's ~13-16M hop-2 entries.
A GATE first: GCNEncoder(fused=True) against fused=False with float64 parameters, 'gcn' and 'attention', the forward within
1e-5 of its largest entry and every parameter's gradient within 1e-5 of its largest entry; a mismatch aborts.  The gate runs
on the batch's first 256 seeds: the float64 composition of the whole batch would hold several [nnz, 128] float64 matrices.
Then, alternating in rounds in one process:
  (a) the hop-1 adjacency alone, forward and forward + backward (the gradient of x_neigh): adjacency_mean, gather +
      scatter_add (then the division), torch.sparse.mm of the ones-valued COO matrix (then the division);
  (b) the whole GCNEncoder (the hops included), forward + backward, 'gcn' and 'attention' (4 heads), fused vs fused=False.
Reported per arm: ms per call and torch's allocator peak above the inputs; the [nnz, D] message bytes, computed from the
shapes; the card's name, power limit and max SM clock read in the same run.  One JSON line on stdout.  It needs a GPU:
without one it fails rather than measure anything else."""
import argparse
import time

import harness
import numpy as np
from harness import DENSE_DIM, build_graph, timed


METAPATH = [[0], [0]]
GATE_SEEDS = 256


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def make_encoder(args, aggregator, fused):
    from euler_b200.encoders import GCNEncoder
    torch.manual_seed(0)
    return GCNEncoder(METAPATH, args.dim, aggregator, feature_idx="feat0", feature_dim=DENSE_DIM, head_num=4, fused=fused,
                      device="cuda")


def encoder_step(enc, seeds):
    out = enc(seeds)
    torch.autograd.grad(out, list(enc.parameters()), torch.ones_like(out))


def gate(eb, args, seeds):
    """fused (float32) against the composition with float64 parameters (and float64 feature rows)"""
    from euler_b200 import ops
    real = ops.get_dense_feature
    for aggregator in ("gcn", "attention"):
        res = []
        for fused in (True, False):
            enc = make_encoder(args, aggregator, fused)
            if not fused:
                enc = enc.double()
                ops.get_dense_feature = lambda *a, **k: [t.double() for t in real(*a, **k)]
            try:
                out = enc(seeds)
                res.append((out.detach(), torch.autograd.grad(out.square().sum(), list(enc.parameters()))))
            finally:
                ops.get_dense_feature = real
            del enc
        (a, ga), (b, gb) = res
        err = float((a.double() - b).abs().max() / b.abs().max())
        if err > 1e-5:
            raise SystemExit("GATE FAILED: %s: the fused encoder's forward is %.3g of the largest entry from the composition's"
                             % (aggregator, err))
        for t, (x, y) in enumerate(zip(ga, gb)):
            err = float((x.double() - y).abs().max() / y.abs().max())
            if err > 1e-5:
                raise SystemExit("GATE FAILED: %s: parameter %d's gradient is %.3g of its largest entry from the composition's"
                                 % (aggregator, t, err))


def run(args):
    global torch
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/gcn_encoder.py needs a GPU; nothing is measured without one")
    import euler_b200 as eb
    torch.cuda.set_device(0)
    t0 = time.time()
    _g = build_graph(args)
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=args.batch).astype(np.int64)).cuda()
    nodes, adjs = eb.get_multi_hop_neighbor(seeds, METAPATH)
    indptr, cols, _ = adjs[1]
    n, m, nnz = nodes[1].numel(), nodes[2].numel(), cols.numel()
    x = torch.randn(m, args.dim, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)).requires_grad_(True)
    deg = (indptr[1:] - indptr[:-1]).to(torch.float32)[:, None].clamp(min=1e-7)
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), indptr[1:] - indptr[:-1], output_size=nnz)
    rows32, cols32 = rows.to(torch.int32), cols.to(torch.int32)
    coo = torch.sparse_coo_tensor(torch.stack([rows, cols]), torch.ones(nnz, device="cuda"), (n, m)).coalesce()
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    gate(eb, args, seeds[:GATE_SEEDS])

    def fused_mean():
        return eb.adjacency_mean(x, (indptr, cols))

    def gather_scatter():
        return eb.scatter_add(eb.gather(x, cols32), rows32, n) / deg

    def sparse_mm():
        return torch.sparse.mm(coo, x) / deg

    def fwd_bwd(fn):
        out = fn()
        torch.autograd.grad(out, [x], torch.ones_like(out))

    encs = {(a, f): make_encoder(args, a, f) for a in ("gcn", "attention") for f in (True, False)}
    arms = {
        "adj_fused_fwd": fused_mean, "adj_gather_scatter_fwd": gather_scatter, "adj_sparse_mm_fwd": sparse_mm,
        "adj_fused_fwd_bwd": lambda: fwd_bwd(fused_mean), "adj_gather_scatter_fwd_bwd": lambda: fwd_bwd(gather_scatter),
        "adj_sparse_mm_fwd_bwd": lambda: fwd_bwd(sparse_mm),
    }
    for (a, f), enc in encs.items():
        arms["encoder_%s_%s_fwd_bwd" % (a, "fused" if f else "composed")] = (lambda e: lambda: encoder_step(e, seeds))(enc)
    res = timed(arms, args.steps, args.warmup)
    harness.emit({"metric": "gcn_encoder_adjacency_mean_fwd_ms", "value": res["adj_fused_fwd"]["ms_per_call"], "gate": "passed",
                  "gpu": harness.gpu_info(0), "batch": args.batch, "dim": args.dim, "setup_s": setup_s, "arms": res,
                  "shapes": {"hop1_rows": n, "hop2_nodes": m, "hop1_entries": nnz, "message_bytes": nnz * args.dim * 4,
                     "seed_entries": int(adjs[0][1].numel()), "gate_seeds": GATE_SEEDS}})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
