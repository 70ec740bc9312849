#!/usr/bin/env python
"""DeepWalk's training step on float32 against bfloat16 id tables (unsupervised.DeepWalk(table_dtype=...), train_step), at one
shape, in one run on one GPU.

    python benchmarks/bf16_tables.py [--nodes N] [--edges E] [--dim D] [--batch B] [--optimizer NAME] [--steps K] [--warmup W]

A step is train_step: the walks, pairs and negatives drawn on the device, the fused skip-gram forward, its sparse backward,
and the optimizer's fused update of both tables and their slots (bf16: stochastic rounding on every store).  Both arms
draw the same ids (the sampler is reseeded before each step of each arm) and start from the same tables (the f32 arm
holds the bf16 arm's widened values).  The arms alternate round by round, timed with device events.  Reported per arm:
ms per step, the tables' and slots' bytes, and the mean loss of the timed steps; the card's name, power limit and max SM
clock are read in the same run.  One JSON line on stdout.  It needs a GPU: without one it fails."""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from full_dataflow import emit, gpu_info  # noqa: E402
import full_dataflow  # noqa: E402


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--batch", type=int, default=512)
    p.add_argument("--optimizer", default="adam")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def run(args):
    import numpy as np
    import torch
    import euler_b200 as eb
    from euler_b200 import optimizers, unsupervised as un
    torch.cuda.set_device(0)
    eb.set_graph(eb.Graph.rmat(args.nodes, args.edges, seed=11), rng="philox", seed=1)
    models = {}
    for name, dt in (("bf16", torch.bfloat16), ("f32", torch.float32)):
        torch.manual_seed(3)
        models[name] = un.DeepWalk(0, [0], args.nodes, args.dim, walk_len=3, num_negs=5, device="cuda", table_dtype=dt)
    with torch.no_grad():
        for p16, p32 in zip(models["bf16"].parameters(), models["f32"].parameters()):
            p32.copy_(p16.float())
    opts = {k: optimizers.get(args.optimizer)(list(m.parameters()), 0.01, **({"seed": 5} if k == "bf16" else {}))
            for k, m in models.items()}
    batches = [torch.from_numpy(np.random.RandomState(100 + i).randint(1, args.nodes + 1, size=args.batch)).cuda()
               for i in range(args.warmup + args.steps)]
    losses = {k: [] for k in models}

    def step(k, i):
        eb.seed(1000 + i)
        losses[k].append(models[k].train_step(batches[i], opts[k])[0])

    for i in range(args.warmup):
        for k in models:
            step(k, i)
    torch.cuda.synchronize()
    for k in losses:
        losses[k].clear()
    rounds = max(1, min(5, args.steps))
    per = -(-args.steps // rounds)
    tot = {k: [0.0, 0] for k in models}
    i = args.warmup
    for _ in range(rounds):
        n = min(per, args.warmup + args.steps - i)
        if n <= 0:
            break
        for k in models:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for j in range(n):
                step(k, i + j)
            e1.record()
            torch.cuda.synchronize()
            tot[k][0] += e0.elapsed_time(e1)
            tot[k][1] += n
        i += n

    def state_bytes(k):
        ps = list(models[k].parameters())
        return sum(p.numel() * p.element_size() for p in ps) + sum(
            t.numel() * t.element_size() for p in ps for t in opts[k].state[p].values() if torch.is_tensor(t))

    out = {"workload": "deepwalk_train_step", "nodes": args.nodes, "edges": args.edges, "dim": args.dim, "batch": args.batch,
           "optimizer": args.optimizer, "gpu": gpu_info(0)}
    for k, (ms, n) in tot.items():
        out[k] = {"ms_per_step": ms / n, "steps": n, "table_and_slot_bytes": state_bytes(k),
                  "mean_loss": float(np.mean([float(x) for x in losses[k]]))}
    out["bf16_over_f32_time"] = out["bf16"]["ms_per_step"] / out["f32"]["ms_per_step"]
    emit(out)


if __name__ == "__main__":
    sys.stdout.flush()
    full_dataflow._REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    run(parse())
