#!/usr/bin/env python
"""Full-neighborhood minibatch construction on one H100: the fused full-neighbor hop (GCNDataFlow) against the same blocks
composed from the separate ops (get_full_neighbor, torch cat / repeat_interleave, unique once per hop).

    python benchmarks/full_dataflow.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Default workload = the gcn example's 'full' dataflow: 2-hop GCNDataFlow [[0],[0]] with self loops, batch 2048, on the R-MAT
graph of BASELINE configs[1] (10M nodes / 100M edges, D=128 features).  Batch 2048 lists ~13-16M entries at hop 2 (next
frontier ~2.2M), sized on the host with oracle/rmat_gen.c: far below 2^31 entries and the card's memory.

Before anything is timed a PARITY GATE compares batch 0 bit-exactly with the oracle's listing on the exported CSR plus a numpy
restatement of gcn_dataflow.py / neighbor_dataflow.py, and the composition with the fused op; a mismatch aborts.
metric = block entries/s: edge_index columns of all hops (listed edges + self loops) per second.  One JSON line on stdout;
nothing is written to the tree."""
import argparse
import os
import time

import harness
import numpy as np

from bench import FEAT_SEED, GRAPH_SEED, Clocks

FULL_METAPATH = [[0], [0]]


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--steps", type=int, default=40)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--no-gate", action="store_true", help="skip the pre-timing parity gate (debugging only)")
    return p.parse_args(argv)


def composed_gcn_flow(eb, n_id, metapath, add_self_loops=True):
    """GCNDataFlow's blocks written over the separate ops, the way a user would without the fused hop: get_full_neighbor,
    torch cat / repeat_interleave and one unique per hop.  Returns [(n_id, res_n_id, edge_index)] in hop order."""
    import torch
    blocks = []
    for et in metapath:
        n = n_id.numel()
        indptr, ids, _w, _t = eb.get_full_neighbor(n_id, et)
        rows = torch.repeat_interleave(torch.arange(n, device=n_id.device), indptr[1:] - indptr[:-1], output_size=ids.numel())
        new_n_id, inv = eb.unique(torch.cat([ids, n_id]))
        inv = inv.to(torch.int64)
        res = inv[inv.numel() - n:]
        if add_self_loops:
            ei = torch.stack([torch.cat([rows, torch.arange(n, device=n_id.device)]), inv])
        else:
            ei = torch.stack([rows, inv[:inv.numel() - n]])
        blocks.append((new_n_id, res, ei))
        n_id = new_n_id
    return blocks


def np_unique_first(x):
    """tf.unique on the host: distinct values in first-occurrence order, and the inverse"""
    vals, first, inv = np.unique(x, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return vals[order], rank[inv]


def run_full(args):
    """A step = the 2-hop GCNDataFlow [[0],[0]] of one batch of seeds (block construction only, no features).
    metric = block entries/s: edge_index columns of all hops (listed edges + self loops) per second.  The same blocks built
    over the separate ops (composed_gcn_flow) are timed in the same process, alternating with the fused op round by round."""
    import torch
    import euler_b200 as eb
    from euler_b200.dataflow import GCNDataFlow
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    B = args.batch
    t0 = time.time()
    graph = eb.Graph.rmat(args.nodes, args.edges, seed=GRAPH_SEED, feat_dim=args.dim, feat_seed=FEAT_SEED, device=local)
    torch.cuda.synchronize()
    t_graph = time.time() - t0
    eb.set_graph(graph)
    n_sb = args.warmup + args.steps
    host_seeds = [np.random.RandomState(7000 + i).randint(1, args.nodes + 1, size=B).astype(np.int64) for i in range(n_sb)]
    dev_seeds = [torch.from_numpy(s).cuda() for s in host_seeds]
    fused = GCNDataFlow(FULL_METAPATH)

    def fused_step(seeds):
        return [(b.n_id, b.res_n_id, b.edge_index) for b in fused(seeds).blocks]

    def composed_step(seeds):
        return composed_gcn_flow(eb, seeds, FULL_METAPATH)

    gate = {"passed": None, "skipped": "--no-gate"}
    if not args.no_gate:
        from oracle import pyoracle as po
        tg = time.time()
        f_blocks = fused_step(dev_seeds[0])
        got = [[x.cpu().numpy() for x in blk] for blk in f_blocks]
        for h, (a, b) in enumerate(zip(f_blocks, composed_step(dev_seeds[0]))):
            if not all(torch.equal(x, y) for x, y in zip(a, b)):
                raise SystemExit("PARITY GATE FAILED: hop %d of the composition differs from the fused op" % (h + 1))
        ex = graph.export(with_feat=False)
        og = po.OracleGraph(ex["ids"], ex["node_type"], ex["node_w"], 1, ex["grp_ptr"], ex["nbr"], ex["cum_w"], None)
        cur = host_seeds[0]
        for h, et in enumerate(FULL_METAPATH):          # gcn_dataflow.py get_neighbors + UniqueDataFlow.produce_subgraph
            lens, ids, _, _ = og.get_full_neighbor(cur.astype(np.uint64), et)
            rows = np.repeat(np.arange(len(cur)), lens)
            new, inv = np_unique_first(np.concatenate([ids.astype(np.int64), cur]))
            want = (new, inv[len(inv) - len(cur):], np.stack([np.concatenate([rows, np.arange(len(cur))]), inv]))
            for nm, g_, w_ in zip(("n_id", "res_n_id", "edge_index"), got[h], want):
                if not np.array_equal(g_, w_):
                    raise SystemExit("PARITY GATE FAILED: %s of hop %d differs from the oracle listing + numpy restatement" % (nm, h + 1))
            cur = new
        gate = {"passed": True, "seconds": round(time.time() - tg, 2),
                "what": "batch 0: n_id, res_n_id and edge_index of both hops bit-exact vs the oracle's listing on the exported CSR + "
                        "a numpy restatement of gcn_dataflow.py / neighbor_dataflow.py; the composition equal to the fused op"}
        del og, ex

    def timed(fn, first, n):
        """n steps on seed sets first.. ; returns (ms, entries, per-hop sizes)"""
        hops, seq = [], iter(range(first, first + n))

        def step():
            hops.append([(int(ei.shape[1]), int(nid.numel())) for nid, _, ei in fn(dev_seeds[next(seq) % n_sb])])
        ms = harness.time_arms({"step": step}, 1, 0, n)["step"][0] * n
        return ms, sum(h[0] for hop in hops for h in hop), hops

    arms = {"fused": fused_step, "composition": composed_step}
    for fn in arms.values():
        # every seed set once: the op scratch and torch's caching allocator grow to the largest batch outside the timed
        # rounds (a growth synchronises and reallocates), then the warm-up steps
        timed(fn, 0, n_sb)
        timed(fn, 0, max(args.warmup, 1))
    rounds, per = harness.rounds_of(args.steps)
    tot = {k: [0.0, 0, 0] for k in arms}
    per_round, hop_sizes = [], []
    clocks = Clocks(local)
    clocks.start()
    time.sleep(0.3)
    w0 = time.time()
    for r in range(rounds):
        row = {}
        for k, fn in arms.items():
            ms, entries, hops = timed(fn, args.warmup + r * per, per)
            tot[k][0] += ms
            tot[k][1] += entries
            tot[k][2] += per
            row[k] = round(entries / (ms * 1e-3), 1)
            if k == "fused":
                hop_sizes += hops
        per_round.append(row)
    w1 = time.time()
    clk = clocks.stop(w0, w1)
    rate = {k: v[1] / (v[0] * 1e-3) for k, v in tot.items()}
    hs = np.asarray(hop_sizes, np.float64)          # [steps, hops, (edge_index columns, next frontier)]
    hops = [{"hop": h + 1, "entries_mean": float(hs[:, h, 0].mean()), "listed_E_mean": float(hs[:, h, 0].mean() - (hs[:, h - 1, 1].mean() if h else B)),
             "frontier_mean": float(hs[:, h, 1].mean()), "entries_max": int(hs[:, h, 0].max())} for h in range(hs.shape[1])]
    out = {"metric": "block_entries_per_sec", "value": rate["fused"], "unit": "entries/s", "n_gpus": 1, "steps": tot["fused"][2],
           "warmup": args.warmup, "ms_per_step": tot["fused"][0] / tot["fused"][2], "higher_is_better": True, "vs_baseline": None,
           "data": "synthetic",
           "config": {"workload": "synthetic power-law (R-MAT 0.57/0.19/0.19/0.05) graph %dM nodes/%dM edges, 2-hop GCNDataFlow "
                                  "metapath %s with self loops, batch=%d, 1 GPU" % (args.nodes // 10**6, args.edges // 10**6,
                                                                                    FULL_METAPATH, B),
                      "nodes": args.nodes, "edges": args.edges, "batch": B, "metapath": FULL_METAPATH, "feat_dim": args.dim},
           "composition": {"value": rate["composition"], "unit": "entries/s",
                           "ms_per_step": tot["composition"][0] / tot["composition"][2],
                           "what": "get_full_neighbor + torch repeat_interleave / cat + unique, once per hop"},
           "speedup_vs_composition": rate["fused"] / rate["composition"], "rounds": per_round, "hops": hops,
           "parity_gate": gate, "clocks": clk, "gpu": harness.gpu_info(local), "graph_build_s": round(t_graph, 2)}
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    run_full(parse())
