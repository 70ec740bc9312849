#!/usr/bin/env python
"""Layer-wise minibatch construction on one H100: LayerwiseDataFlow ('adapt') with its adjacency from the sparse op
(sample_neighbor_layerwise_coo) against the same flow with its adjacency taken from the dense op and `nonzero`.

    python benchmarks/layerwise_dataflow.py [--steps K] [--warmup W] [--nodes N --edges E]

Graph: the R-MAT graph of BASELINE configs[1] (10M nodes / 100M edges).  Two workloads of LayerwiseDataFlow, metapath
[[0],[0]] with self loops: the adaptivegcn example's shape (batch 512, fanouts [400, 400]) and a large one (batch 4096,
fanouts [4096, 4096]).  Hop 1 draws total_fanout neighbors for the whole batch and takes its edges from the adjacency; hop 2
lists the frontier's full neighborhoods.

Before anything is timed a PARITY GATE runs batch 0 of each workload through both arms under one seed and requires identical
blocks, and compares the adjacency of sample_neighbor_layerwise_coo bit-exactly with a numpy restatement of the reference's
builder (tf_euler/kernels/sparse_get_adj_op.cc:84-117) over the oracle's listing on the exported CSR; a mismatch aborts.
metric = edge_index columns of all hops per second.  One JSON line on stdout; nothing is written to the tree."""
import argparse
import os
import time

import harness
import numpy as np

from bench import GRAPH_SEED, Clocks

METAPATH = [[0], [0]]
WORKLOADS = [{"name": "example", "batch": 512, "fanouts": [400, 400]},
             {"name": "large", "batch": 4096, "fanouts": [4096, 4096]}]


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--no-gate", action="store_true", help="skip the pre-timing parity gate (debugging only)")
    return p.parse_args(argv)


class DenseAdjacency:
    """euler_b200 with sample_neighbor_layerwise_coo rebuilt from the dense op: sample_neighbor_layerwise's f32[batch, n, count]
    view, then its nonzero entries plus the filler (b, n-1, count-1) = 0 of every batch row where that entry is 0"""

    def __init__(self, eb):
        self.eb = eb

    def sample_neighbor_layerwise_coo(self, nodes, edge_types, count, default_node=-1, weight_func=''):
        out, adj = self.eb.sample_neighbor_layerwise(nodes, edge_types, count, default_node, weight_func)
        keep = adj != 0
        keep[:, -1, -1] = True
        return out, (keep.nonzero(), (adj[keep] != 0).long(), tuple(adj.shape))

    def __getattr__(self, name):
        return getattr(self.eb, name)


def restated_adjacency(og, nodes, nb):
    """sparse_get_adj_op.cc:84-117 for one batch row, vectorised: entry (0, j, k) = 1 iff (nodes[j], nb[k]) is among the
    listed (src, dst) pairs, in row-major order, and (0, N-1, M-1) = 0 if it is not"""
    lens, ids, _, _ = og.get_full_neighbor(nodes.astype(np.uint64), METAPATH[0])
    ids = ids.astype(np.int64)
    vocab = np.unique(np.concatenate([nodes, ids, nb]))
    U = np.int64(len(vocab))
    code = lambda x: np.searchsorted(vocab, x).astype(np.int64)          # noqa: E731
    listed = code(np.repeat(nodes, lens)) * U + code(ids)
    hit = np.isin(code(nodes)[:, None] * U + code(nb)[None, :], listed)
    keep = hit.copy()
    keep[-1, -1] = True
    jk = np.argwhere(keep)
    return np.concatenate([np.zeros((len(jk), 1), np.int64), jk], 1), hit[keep].astype(np.int64)


def run(args):
    import torch
    import euler_b200 as eb
    from euler_b200.dataflow import LayerwiseDataFlow
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    t0 = time.time()
    graph = eb.Graph.rmat(args.nodes, args.edges, seed=GRAPH_SEED, device=local)
    torch.cuda.synchronize()
    t_graph = time.time() - t0
    eb.set_graph(graph)
    n_sb = args.warmup + args.steps
    dense = DenseAdjacency(eb)
    og = None
    results, gates = [], {}
    for wl in WORKLOADS:
        B, fanouts = wl["batch"], wl["fanouts"]
        host_seeds = [np.random.RandomState(9000 + i).randint(1, args.nodes + 1, size=B).astype(np.int64) for i in range(n_sb)]
        dev_seeds = [torch.from_numpy(s).cuda() for s in host_seeds]
        arms = {"sparse": LayerwiseDataFlow(fanouts, METAPATH), "dense_nonzero": LayerwiseDataFlow(fanouts, METAPATH, sampler=dense)}

        def step(flow, seeds):
            return [(b.n_id, b.res_n_id, b.edge_index) for b in flow(seeds).blocks]

        if not args.no_gate:
            tg = time.time()
            blocks = {}
            for k, flow in arms.items():
                eb.seed(11)
                blocks[k] = step(flow, dev_seeds[0])
            for h, (a, b) in enumerate(zip(blocks["sparse"], blocks["dense_nonzero"])):
                if not all(torch.equal(x, y) for x, y in zip(a, b)):
                    raise SystemExit("PARITY GATE FAILED: %s hop %d differs between the sparse and the dense adjacency" % (wl["name"], h + 1))
            eb.seed(11)
            nb, (idx, val, _) = eb.sample_neighbor_layerwise_coo(dev_seeds[0].reshape(1, -1), METAPATH[0], fanouts[0])
            if og is None:
                from oracle import pyoracle as po
                ex = graph.export(with_feat=False)
                og = po.OracleGraph(ex["ids"], ex["node_type"], ex["node_w"], 1, ex["grp_ptr"], ex["nbr"], ex["cum_w"], None)
                del ex
            w_idx, w_val = restated_adjacency(og, host_seeds[0], nb.reshape(-1).cpu().numpy())
            if not (np.array_equal(idx.cpu().numpy(), w_idx) and np.array_equal(val.cpu().numpy(), w_val)):
                raise SystemExit("PARITY GATE FAILED: %s: the adjacency differs from the numpy restatement" % wl["name"])
            gates[wl["name"]] = {"passed": True, "seconds": round(time.time() - tg, 2), "hop1_entries": int(len(w_idx)),
                                 "hop1_ones": int(w_val.sum())}

        def timed(flow, first, n, engine_seed):
            """n steps on seed sets first.. with the engine seeded by engine_seed: both arms draw the same neighbors and build
            the same blocks.  Returns (ms, edge_index columns, per-hop sizes)"""
            eb.seed(engine_seed)
            hops, seq = [], iter(range(first, first + n))

            def call():
                hops.append([(int(ei.shape[1]), int(nid.numel())) for nid, _, ei in step(flow, dev_seeds[next(seq) % n_sb])])
            ms = harness.time_arms({"step": call}, 1, 0, n)["step"][0] * n
            return ms, sum(h[0] for hop in hops for h in hop), hops

        rounds, per = harness.rounds_of(args.steps)
        for flow in arms.values():
            timed(flow, 0, max(args.warmup, 1), 0)
            for r in range(rounds):       # the timed steps once: scratch and the caching allocator reach their size
                timed(flow, args.warmup + r * per, per, 100 + r)
        tot = {k: [0.0, 0, 0] for k in arms}
        per_round, hop_sizes = [], []
        clocks = Clocks(local)
        clocks.start()
        time.sleep(0.3)
        w0 = time.time()
        for r in range(rounds):
            row = {}
            for k, flow in arms.items():
                ms, cols, hops = timed(flow, args.warmup + r * per, per, 100 + r)
                tot[k][0] += ms
                tot[k][1] += cols
                tot[k][2] += per
                row[k] = round(cols / (ms * 1e-3), 1)
                if k == "sparse":
                    hop_sizes += hops
            per_round.append(row)
        clk = clocks.stop(w0, time.time())
        hs = np.asarray(hop_sizes, np.float64)
        res = {"workload": wl["name"], "batch": B, "fanouts": fanouts, "metapath": METAPATH, "steps": tot["sparse"][2],
               "hops": [{"hop": h + 1, "edge_index_cols_mean": float(hs[:, h, 0].mean()), "n_id_mean": float(hs[:, h, 1].mean())}
                        for h in range(hs.shape[1])],
               "rounds": per_round, "clocks": clk}
        for k, (ms, cols, steps) in tot.items():
            res[k] = {"cols_per_sec": cols / (ms * 1e-3), "ms_per_step": ms / steps}
        res["speedup_vs_dense_nonzero"] = res["sparse"]["cols_per_sec"] / res["dense_nonzero"]["cols_per_sec"]
        # the two adjacency builders alone, on hop 1's inputs of the timed seed sets (the rest of a step is common to both)
        eb.seed(5)
        hop1 = [(s.reshape(1, -1), eb.sample_neighbor_layerwise(s.reshape(1, -1), METAPATH[0], fanouts[0])[0])
                for s in dev_seeds[args.warmup:]]

        def coo(nd, nb):
            return eb.sparse_get_adj_coo(nd.reshape(-1), nb.reshape(-1), METAPATH[0], B, fanouts[0])[0]

        def dense_nonzero(nd, nb):
            adj = eb.sparse_get_adj(nd.reshape(-1), nb.reshape(-1), METAPATH[0], B, fanouts[0])
            keep = adj != 0
            keep[:, -1, -1] = True
            return keep.nonzero()
        op = {}
        for k, fn in (("sparse", coo), ("dense_nonzero", dense_nonzero)):
            for nd, nb in hop1:
                fn(nd, nb)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            for nd, nb in hop1:
                fn(nd, nb)
            torch.cuda.synchronize()
            op[k] = (time.perf_counter() - t1) * 1e3 / len(hop1)
        res["adjacency_op_ms"] = {"sparse": op["sparse"], "dense_nonzero": op["dense_nonzero"],
                                  "what": "sparse_get_adj_coo vs sparse_get_adj + nonzero + filler on hop 1's [1, %d] x [1, %d] "
                                          "inputs, host wall time per call" % (B, fanouts[0])}
        results.append(res)
        del dev_seeds
    head = results[0]
    out = {"metric": "edge_index_cols_per_sec", "value": head["sparse"]["cols_per_sec"], "unit": "cols/s", "n_gpus": 1,
           "steps": args.steps, "warmup": args.warmup, "ms_per_step": head["sparse"]["ms_per_step"], "higher_is_better": True,
           "data": "synthetic",
           "config": {"workload": "synthetic power-law (R-MAT 0.57/0.19/0.19/0.05) graph %dM nodes/%dM edges, 2-hop "
                                  "LayerwiseDataFlow metapath %s with self loops, 1 GPU; value = the %s workload"
                                  % (args.nodes // 10**6, args.edges // 10**6, METAPATH, head["workload"]),
                      "nodes": args.nodes, "edges": args.edges},
           "workloads": results, "parity_gate": gates or {"passed": None, "skipped": "--no-gate"}, "gpu": harness.gpu_info(local),
           "graph_build_s": round(t_graph, 2)}
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
