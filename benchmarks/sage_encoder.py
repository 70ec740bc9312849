#!/usr/bin/env python
"""SageEncoder over trainable inputs on one H100: the deepest hop pooled by ops.shallow_encode_pool against the composition
it replaces (shallow_encode's rows, then a mean over each fanout segment), alone and inside the whole encoder.

    python benchmarks/sage_encoder.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Graph and inputs: those of benchmarks/shallow_encoder.py -- the R-MAT of BASELINE configs[1] (10M nodes / 100M edges) with a
dense slot of D = 128 columns and the two seeded uint64 slots of benchmarks/sparse_embedding.py; an id table of N + 2 rows
and both slot tables at dim 16 (sum): rows of W = 16 + 128 + 32 = 176 columns.  Workload: batch 8192, fanout [15, 10],
'mean' aggregator, dim 128; the deepest hop is 8192 * 15 * 10 = 1,228,800 nodes pooled into 122,880 rows.
A GATE first: SageEncoder(fused=True) against fused=False with float64 parameters on the same draws, the forward within 1e-5
and every parameter's gradient within 1e-5 of its largest entry; a mismatch aborts.  Then, alternating in rounds in one process:
  (a) the deepest hop alone, shallow_encode_pool vs shallow_encode + view(-1, 10, W).mean(1): forward, forward + backward
      with dense table gradients, forward + backward with sparse COO gradients;
  (b) the whole SageEncoder (sampling included, the same seeds), forward + backward, fused vs fused=False.
Reported per arm: ms per call, torch's allocator peak above the inputs, and the growth of the library's ctx scratch (device
memory in use outside torch's allocator) over the run; the bytes the [M, W] matrix would take, computed from the shapes; the
card's name, power limit and max SM clock read in the same run.  One JSON line on stdout.  It needs a GPU: without one it
fails rather than measure anything else."""
import argparse
import time

import harness
import numpy as np
from harness import DENSE_DIM, DIM, SLOTS, build_graph, timed


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=8192)
    p.add_argument("--fanout", default="15,10")
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def shapes(args):
    """what the workload moves, from its shapes alone: the deepest hop's nodes M, the pooled rows R, the row width W and the
    bytes of the [M, W] matrix the composition writes (and of its gradient, the same again)"""
    fanout = [int(x) for x in args.fanout.split(",")]
    R = args.batch * int(np.prod(fanout[:-1]))
    M, W = R * fanout[-1], DIM + DENSE_DIM + DIM * len(SLOTS)
    return {"fanout": fanout, "deepest_hop_nodes": M, "pooled_rows": R, "row_width": W, "row_matrix_bytes": M * W * 4,
            "pooled_bytes": R * W * 4}


def make_encoder(eb, args, fanout, fused, sparse_grad=False):
    from euler_b200.encoders import SageEncoder
    torch.manual_seed(0)
    return SageEncoder([[0]] * len(fanout), fanout, args.dim, aggregator="mean", feature_idx="feat0", feature_dim=DENSE_DIM,
                       max_id=args.nodes, use_id=True, sparse_feature_idx=[n for n, _ in SLOTS],
                       sparse_feature_max_id=[m - 1 for _, m in SLOTS], embedding_dim=DIM, fused=fused, sparse_grad=sparse_grad,
                       device="cuda")


def encoder_step(eb, enc, seeds):
    eb.seed(5)
    out = enc(seeds)
    torch.autograd.grad(out, list(enc.parameters()), torch.ones_like(out))


def gate(eb, args, fanout, seeds):
    """fused (float32) against the composition with float64 parameters: the composition's own float32 sums (index_add's
    atomics over a hot row's ~10^5 entries) are not accurate enough to arbitrate at 1e-5"""
    res = []
    for fused in (True, False):
        enc = make_encoder(eb, args, fanout, fused)
        if not fused:
            enc = enc.double()
        eb.seed(5)
        out = enc(seeds)
        res.append((out.detach(), torch.autograd.grad(out.square().sum(), list(enc.parameters()))))
        del enc
    (a, ga), (b, gb) = res
    err = float((a - b).abs().max() / b.abs().max())
    if err > 1e-5:
        raise SystemExit("GATE FAILED: the fused encoder's forward is %.3g of the largest entry from the composition's" % err)
    for t, (x, y) in enumerate(zip(ga, gb)):
        err = float((x - y).abs().max() / y.abs().max())
        if err > 1e-5:
            raise SystemExit("GATE FAILED: parameter %d's gradient is %.3g of its largest entry from the composition's" % (t, err))


def run(args):
    global torch
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/sage_encoder.py needs a GPU; nothing is measured without one")
    import euler_b200 as eb
    torch.cuda.set_device(0)
    sh = shapes(args)
    fanout = sh["fanout"]
    t0 = time.time()
    _g = build_graph(args)
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=args.batch).astype(np.int64)).cuda()
    deep = eb.sample_fanout(seeds, [[0]] * len(fanout), fanout, default_node=args.nodes + 1)[0][-1]
    gen = torch.Generator(device="cuda").manual_seed(1)
    id_table = (torch.randn(args.nodes + 2, DIM, device="cuda", generator=gen) * 0.1).requires_grad_(True)
    tables = [(torch.randn(m + 1, DIM, device="cuda", generator=gen) * 0.01).requires_grad_(True) for _, m in SLOTS]
    params = [id_table] + tables
    sparse = [(name, t, dflt) for (name, dflt), t in zip(SLOTS, tables)]
    dense = [("feat0", DENSE_DIM)]
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    res = {}

    def gated_run():
        gate(eb, args, fanout, seeds)

        def pooled(sg=False):
            return eb.shallow_encode_pool(deep, fanout[-1], id_table, dense, sparse, "mean", sparse_grad=sg)

        def composed(sg=False):
            return eb.shallow_encode(deep, id_table, dense, sparse, "concat", sparse_grad=sg).view(-1, fanout[-1], sh["row_width"]).mean(1)

        def fwd_bwd(fn, sg):
            out = fn(sg)
            torch.autograd.grad(out, params, torch.ones_like(out))

        encs = {(f, s): make_encoder(eb, args, fanout, f, s) for f in (True, False) for s in (False, True)}
        arms = {
            "hop_pooled_fwd": pooled, "hop_composed_fwd": composed,
            "hop_pooled_fwd_bwd_dense": lambda: fwd_bwd(pooled, False), "hop_composed_fwd_bwd_dense": lambda: fwd_bwd(composed, False),
            "hop_pooled_fwd_bwd_sparse": lambda: fwd_bwd(pooled, True), "hop_composed_fwd_bwd_sparse": lambda: fwd_bwd(composed, True),
            "encoder_fused_fwd_bwd_dense": lambda: encoder_step(eb, encs[True, False], seeds),
            "encoder_composed_fwd_bwd_dense": lambda: encoder_step(eb, encs[False, False], seeds),
            "encoder_fused_fwd_bwd_sparse": lambda: encoder_step(eb, encs[True, True], seeds),
            "encoder_composed_fwd_bwd_sparse": lambda: encoder_step(eb, encs[False, True], seeds),
        }
        res.update(timed(arms, args.steps, args.warmup))
    scratch_growth = harness.memory_of(gated_run)[1]      # the library's ctx scratch over the gate and every arm
    harness.emit({"metric": "sage_encoder_deepest_hop_fwd_ms", "value": res["hop_pooled_fwd"]["ms_per_call"], "gate": "passed",
                  "gpu": harness.gpu_info(0), "batch": args.batch, "dim": args.dim, "shapes": sh, "setup_s": setup_s, "arms": res,
                  "ctx_scratch_growth_bytes": max(0, scratch_growth)})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
