#!/usr/bin/env python
"""LGCEncoder's input block on one H100: the fused op (ops.neighbor_top_k_feature) against the composition a user writes
today, get_dense_feature of the nodes and of their neighbours, cat, transpose and torch.topk; and a whole LGCN training
step (forward + backward) with the encoder fused=True against fused=False.

    python benchmarks/lgcn_encoder.py [--steps K] [--warmup W] [--batch B] [--nb-num N] [--k K] [--nodes N --edges E]
                                      [--wide-nodes N --wide-edges E --wide-dim D]

Headline graph: the R-MAT of BASELINE configs[1] (10M nodes / 100M edges) with its dense slot of 128 columns, built as
benchmarks/shallow_encoder.py builds it.  A second graph with one unaligned width (cora's 1433 columns) is smaller
(1M nodes / 10M edges: 5.7 GB of features), so the two graphs fit on the card together.  Workload: batch 8192 seeds,
nb_num = 10 neighbours from sample_neighbor (default_node -1), k = 3, the examples/lgcn defaults.  The LGCN step uses
hidden 128 / out 64 and the slot's first 16 columns as its labels (the R-MAT graph has no label slot; the loss's value
does not change the work).
A GATE first checks the op bit for bit against a stable descending sort of the get_dense_feature rows (on the CPU, whose
sort compares values: -0.0 == +0.0, NaN above every number) on the timed batch -- every row at 128 columns, the first 2048
rows at the wide width; a mismatch aborts.  The arms of a graph alternate in rounds in one process.  Reported per arm: ms
per call and torch's allocator peak above the inputs; the card's name, power limit and SM clock read in the same run.  One
JSON line on stdout."""
import argparse
import time

import harness
import numpy as np

from bench import GRAPH_SEED
from harness import DENSE_DIM, build_graph, timed

LABEL_DIM, HIDDEN, OUT = 16, 128, 64


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--wide-nodes", type=int, default=1_000_000)
    p.add_argument("--wide-edges", type=int, default=10_000_000)
    p.add_argument("--wide-dim", type=int, default=1433)
    p.add_argument("--batch", type=int, default=8192)
    p.add_argument("--nb-num", type=int, default=10)
    p.add_argument("--k", type=int, default=3)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def gate(eb, nodes, nbrs, slot, dim, k, rows):
    got = eb.neighbor_top_k_feature(nodes[:rows], nbrs[:rows], slot, dim, k).cpu()
    node = eb.get_dense_feature(nodes[:rows], [slot], [dim])[0].cpu()
    nb = eb.get_dense_feature(nbrs[:rows].reshape(-1), [slot], [dim])[0].cpu().reshape(rows, nbrs.shape[1], dim)
    want = torch.cat([node[:, None], torch.sort(nb, dim=1, descending=True, stable=True)[0][:, :k]], 1)
    if not torch.equal(got.view(torch.int32), want.view(torch.int32)):
        raise SystemExit("GATE FAILED: neighbor_top_k_feature differs from the stable sort at dim %d" % dim)


def arms_of(eb, args, nodes, nbrs, slot, dim):
    from euler_b200.encoders import LGCEncoder
    from euler_b200.supervised import LGCN
    enc = {f: LGCEncoder([0], slot, dim, args.k, HIDDEN, args.nb_num, OUT, fused=f, device="cuda") for f in (True, False)}
    models = {}
    for f in (True, False):
        torch.manual_seed(0)
        models[f] = LGCN(HIDDEN, [0], slot, LABEL_DIM, feature_idx=slot, feature_dim=dim, k=args.k, nb_num=args.nb_num,
                         out_dim=OUT, fused=f, device="cuda")

    def step(m):
        loss = m(nodes)[1]
        torch.autograd.grad(loss, list(m.parameters()))

    return {
        "op_fused": lambda: enc[True].top_k_rows(nodes, nbrs),
        "op_composed": lambda: enc[False].top_k_rows(nodes, nbrs),
        "lgcn_step_fused": lambda: step(models[True]),
        "lgcn_step_composed": lambda: step(models[False]),
    }


def measure(eb, args, slot, dim, gate_rows):
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes_now + 1, size=args.batch).astype(np.int64)).cuda()
    nbrs = eb.sample_neighbor(seeds, [0], args.nb_num)[0]
    gate(eb, seeds, nbrs, slot, dim, args.k, min(gate_rows, args.batch))
    res = timed(arms_of(eb, args, seeds, nbrs, slot, dim), args.steps, args.warmup)
    for a, b in (("op_fused", "op_composed"), ("lgcn_step_fused", "lgcn_step_composed")):
        res[a]["speedup_vs_composed"] = res[b]["ms_per_call"] / res[a]["ms_per_call"]
    # the bytes the op must move: each node row and nb_num neighbour rows read once, k + 1 rows written
    res["op_fused"]["algorithmic_bytes"] = args.batch * dim * 4 * (1 + args.nb_num + args.k + 1)
    res["op_fused"]["algorithmic_GBps"] = res["op_fused"]["algorithmic_bytes"] / (res["op_fused"]["ms_per_call"] * 1e6)
    return {"dim": dim, "arms": res}


def run(args):
    global torch
    import torch
    import euler_b200 as eb
    torch.cuda.set_device(0)
    t0 = time.time()
    _g = build_graph(args)
    args.nodes_now = args.nodes
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    head = measure(eb, args, 0, DENSE_DIM, args.batch)
    wide = eb.Graph.rmat(args.wide_nodes, args.wide_edges, seed=GRAPH_SEED, feat_dim=args.wide_dim, device=0)
    eb.set_graph(wide, rng="philox", seed=5)
    args.nodes_now = args.wide_nodes
    wide_res = measure(eb, args, 0, args.wide_dim, 2048)
    wide_res["graph"] = {"nodes": args.wide_nodes, "edges": args.wide_edges}
    harness.emit({"metric": "lgcn_top_k_op_ms", "value": head["arms"]["op_fused"]["ms_per_call"], "gate": "passed", "gpu": harness.gpu_info(0),
                  "batch": args.batch, "nb_num": args.nb_num, "k": args.k, "setup_s": setup_s,
                  "graph": {"nodes": args.nodes, "edges": args.edges}, "headline": head, "wide": wide_res})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
