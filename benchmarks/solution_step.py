#!/usr/bin/env python
"""One unsupervised GraphSAGE training step through solution.UnsuperviseSolution on one H100, and sample_node_with_src alone.

    python benchmarks/solution_step.py [--steps K] [--warmup W] [--nodes N --edges E]

Graph: the R-MAT of BASELINE configs[1] (10M nodes / 100M edges) with a dense slot of 128 columns.  Step: target and context
encoders are SageEncoder([[0], [0]], [10, 10], 128, 'mean') over the dense slot; one positive per input from
SamplePosWithTypes([0]), K = 5 negatives from SampleNegWithTypes(0); PosNegLogits + xent_loss + mrr; forward, backward and one
SGD step.  Arms: batch 512 and 2048, each with fused=True encoders (the deepest hop pooled by ops.shallow_encode_pool) and
fused=False (the composition); and sample_node_with_src over 2048 sources x 5.
A GATE first: at each batch the fused step's loss, and every parameter's gradient, within 5e-4 of the largest entry of the
fused=False step's on the same draws; a mismatch aborts.  Both arms are float32 and the composition sums in another order, so
the gate allows for the rounding of either; tests/test_solution_gpu.py checks the step against float64 at 1e-5.
Reported per arm: ms per step and torch's allocator peak above the inputs; the card's name, power limit and max SM clock read in
the same run.  One JSON line on stdout.  It needs a GPU: without one it fails rather than measure anything else."""
import argparse
import time

import harness
import numpy as np
from harness import timed


FEAT, DIM, FANOUTS, NEGS, BATCHES = 128, 128, [10, 10], 5, (512, 2048)


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def make_solution(args, fused):
    from euler_b200 import encoders, solution
    torch.manual_seed(0)

    def enc():
        return encoders.SageEncoder([[0]] * len(FANOUTS), FANOUTS, DIM, 'mean', feature_idx=0, feature_dim=FEAT, max_id=args.nodes,
                                    fused=fused, device="cuda")
    sol = solution.UnsuperviseSolution(enc(), enc(), solution.SamplePosWithTypes([0], 1, max_id=args.nodes),
                                       solution.SampleNegWithTypes(0, NEGS), metric_name='mrr')
    return sol, torch.optim.SGD(sol.parameters(), lr=0.01)


def step(eb, sol, opt, seeds, seed=5):
    eb.seed(seed)
    opt.zero_grad(set_to_none=True)
    _, loss, _, metric = sol(seeds)
    loss.backward()
    opt.step()
    return loss, metric


def gate(eb, args, seeds):
    res = []
    for fused in (True, False):
        sol, _ = make_solution(args, fused)
        eb.seed(5)
        _, loss, _, _ = sol(seeds)
        res.append((loss.detach(), torch.autograd.grad(loss, list(sol.parameters()))))
        del sol
    (a, ga), (b, gb) = res
    err = float((a - b).abs() / b.abs())
    if err > 5e-4:
        raise SystemExit("GATE FAILED: the fused step's loss is %.3g from the composition's" % err)
    for t, (x, y) in enumerate(zip(ga, gb)):
        err = float((x - y).abs().max() / y.abs().max())
        if err > 5e-4:
            raise SystemExit("GATE FAILED: parameter %d's gradient is %.3g of its largest entry from the composition's" % (t, err))


def run(args):
    global torch
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/solution_step.py needs a GPU; nothing is measured without one")
    import euler_b200 as eb
    torch.cuda.set_device(0)
    t0 = time.time()
    g = eb.Graph.rmat(args.nodes, args.edges, seed=42, feat_dim=FEAT, device=0)
    eb.set_graph(g, rng="minstd", seed=5)
    seeds = {B: torch.from_numpy(np.random.RandomState(B).randint(1, args.nodes + 1, size=B).astype(np.int64)).cuda()
             for B in BATCHES}
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    for B in BATCHES:
        gate(eb, args, seeds[B])
    sols = {f: make_solution(args, f) for f in (True, False)}
    arms = {}
    for B in BATCHES:
        for f in (True, False):
            arms["step_b%d_%s" % (B, "fused" if f else "composed")] = (lambda s=sols[f], x=seeds[B]: step(eb, s[0], s[1], x))
    arms["sample_node_with_src_2048x5"] = lambda: eb.sample_node_with_src(seeds[2048], NEGS)
    res = timed(arms, args.steps, args.warmup)
    harness.emit({"metric": "unsupervised_sage_step_b2048_fused_ms", "value": res["step_b2048_fused"]["ms_per_call"], "gate": "passed",
                  "gpu": harness.gpu_info(0), "batches": list(BATCHES), "fanouts": FANOUTS, "dim": DIM, "num_negs": NEGS, "setup_s": setup_s,
                  "arms": res})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
