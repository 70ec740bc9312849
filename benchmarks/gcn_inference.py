#!/usr/bin/env python
"""Embedding every node with GCNEncoder on one H100: layer-by-layer inference over the whole-graph adjacency
(GCNEncoder.infer over ops.graph_adjacency) against encoding the nodes batch by batch with forward.

    python benchmarks/gcn_inference.py [--steps K] [--warmup W] [--nodes N --edges E] [--batch B] [--chunk-rows C]

Graph and model: README's GCNEncoder workload (benchmarks/gcn_encoder.py): the R-MAT of 10M nodes / 100M edges with its
dense slot of 128 columns, metapath [[0], [0]], dim 128, the node encoder the dense slot alone.
A GATE first: infer(ids) against forward(ids) on 4096 random ids, 'gcn' and 'mean', within 1e-5 of the largest entry; a
mismatch aborts.  Then:
  (a) ops.graph_adjacency([0]) alone, ms per call (events, after warmup);
  (b) infer() over every node, 'gcn' and 'mean': ms per call, torch's allocator peak above what was allocated before, and
      the growth of device memory outside torch's allocator (the ctx scratch) over the first call;
  (c) forward over batches of `batch` seeds: --steps batches timed, EXTRAPOLATED to all nodes (ceil(N / batch) batches);
  (d) 'attention' (4 heads): the gate on 1024 ids and infer() once, timed.
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout.  It needs a GPU."""
import argparse
import time

import harness
import numpy as np
from harness import DENSE_DIM, build_graph


METAPATH = [[0], [0]]


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--chunk-rows", type=int, default=1 << 20)
    p.add_argument("--gate-ids", type=int, default=4096)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    return p.parse_args(argv)


def make_encoder(args, aggregator):
    from euler_b200.encoders import GCNEncoder
    torch.manual_seed(0)
    return GCNEncoder(METAPATH, args.dim, aggregator, feature_idx="feat0", feature_dim=DENSE_DIM, head_num=4, device="cuda")


def forward_batches(enc, ids, batch):
    with torch.no_grad():
        return torch.cat([enc(ids[a:a + batch]) for a in range(0, ids.numel(), batch)])


def gate(enc, args, ids, what):
    want = forward_batches(enc, ids, args.batch)
    got = enc.infer(ids, chunk_rows=args.chunk_rows)
    err = float((got.double() - want.double()).abs().max() / want.abs().max())
    if not err <= 1e-5:
        raise SystemExit("GATE FAILED: %s: infer(ids) is %.3g of the largest entry from forward(ids)" % (what, err))
    return err


def event_ms(fn, reps):
    return harness.time_arms({"call": fn}, 1, 0, reps)["call"][0]


def measure_infer(enc, args):
    first = {}

    def call():
        t0 = time.time()
        out = enc.infer(chunk_rows=args.chunk_rows)
        torch.cuda.synchronize()
        first.update(first_call_s=time.time() - t0, rows=int(out.shape[0]))
        return out
    peak, scratch = harness.memory_of(call)
    return {"first_call_s": first["first_call_s"], "torch_peak_bytes": peak, "scratch_growth_bytes": scratch, "rows": first["rows"]}


def run(args):
    global torch
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/gcn_inference.py needs a GPU; nothing is measured without one")
    import euler_b200 as eb
    torch.cuda.set_device(0)
    t0 = time.time()
    _g = build_graph(args)
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    rng = np.random.RandomState(7000)
    gate_ids = torch.from_numpy(rng.randint(1, args.nodes + 1, size=args.gate_ids).astype(np.int64)).cuda()
    encs = {a: make_encoder(args, a) for a in ("gcn", "mean")}
    gates = {a: gate(enc, args, gate_ids, a) for a, enc in encs.items()}

    res = {}
    for _ in range(args.warmup):
        eb.graph_adjacency([0])
    adj = eb.graph_adjacency([0])
    res["graph_adjacency"] = {"ms_per_call": event_ms(lambda: eb.graph_adjacency([0]), max(args.steps, 1)),
                              "entries": int(adj[1].numel()), "absent_ids": int(adj[3].numel())}
    del adj
    for a, enc in encs.items():
        first = measure_infer(enc, args)
        res["infer_%s" % a] = dict(first, ms_per_call=event_ms(lambda: enc.infer(chunk_rows=args.chunk_rows), 2))
    seeds = torch.from_numpy(rng.randint(1, args.nodes + 1, size=(args.warmup + args.steps) * args.batch).astype(np.int64)).cuda()
    n_batches = -(-args.nodes // args.batch)
    for a, enc in encs.items():
        with torch.no_grad():
            for k in range(args.warmup):
                enc(seeds[k * args.batch:(k + 1) * args.batch])
            base = args.warmup * args.batch
            ms = event_ms(lambda it=iter(range(args.steps)): enc(seeds[base + next(it) * args.batch:][:args.batch]), args.steps)
        res["forward_batches_%s" % a] = {"ms_per_batch": ms, "batches_timed": args.steps, "batches_for_all_nodes": n_batches,
                                         "extrapolated_ms_all_nodes": ms * n_batches}
    del encs
    att = make_encoder(args, "attention")
    gates["attention"] = gate(att, args, gate_ids[:1024], "attention")
    res["infer_attention"] = measure_infer(att, args)
    harness.emit({"metric": "gcn_infer_all_nodes_ms", "value": res["infer_gcn"]["ms_per_call"], "gate": "passed", "gate_err": gates,
                  "gpu": harness.gpu_info(0), "nodes": args.nodes, "edges": args.edges, "dim": args.dim, "batch": args.batch,
                  "chunk_rows": args.chunk_rows, "setup_s": setup_s, "arms": res})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
