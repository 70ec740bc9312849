#!/usr/bin/env python
"""Secondary BASELINE.json configs on one H100 (bench.py runs the headline line):
  C3  node2vec biased walk p=0.5 q=2.0 walk_len=80 batch=4096 on RMAT 10M/100M   (+ p=q=1 deepwalk path)
  C4  50M nodes / 500M edges, D=256 on ONE 80 GB GPU: 2-hop [15,10] batch=8192 (the 1-GPU point of configs[3])
  C5  heterogeneous 3 node types / 5 edge types, 50M nodes: per-edge-type sample_neighbor + scatter_add, D=64
Usage: python benchmarks/run_configs.py [c3] [c4] [c5] [--small]
One JSON line per config on stdout, each with the card's name, power limit and max SM clock read in the same run."""
import argparse
import time

import harness
import numpy as np


def timeit(fn, iters, warm=2):
    return harness.time_arms({"call": fn}, 1, warm, iters)["call"][0]


def c3(small):
    n, E = (1_000_000, 10_000_000) if small else (10_000_000, 100_000_000)
    g = eb.Graph.rmat(n, E)
    out = {"config": "C3 walk", "nodes": n, "edges": E, "batch": 4096, "walk_len": 80}
    for rng in ("minstd", "philox"):
        eb.set_graph(g, rng=rng, seed=12345)
        seeds = torch.from_numpy(np.random.RandomState(1).randint(1, n + 1, size=4096)).cuda()
        et = [[0]] * 80
        ms = timeit(lambda: eb.random_walk(seeds, et, 0.5, 2.0), 5 if not small else 3, warm=1)
        w = eb.random_walk(seeds, et, 0.5, 2.0)
        live = float((w != -1).float().mean().item())
        out["node2vec_%s_ms" % rng] = ms
        out["node2vec_%s_walker_steps_per_s" % rng] = 4096 * 80 / (ms * 1e-3)
        out["node2vec_live_fraction"] = live
        ms1 = timeit(lambda: eb.random_walk(seeds, et, 1.0, 1.0), 5, warm=1)
        out["deepwalk_%s_ms" % rng] = ms1
        out["deepwalk_%s_walker_steps_per_s" % rng] = 4096 * 80 / (ms1 * 1e-3)
    harness.emit(dict(out, gpu=harness.gpu_info(0)))
    g.close()


def c4(small):
    n, E, D = (10_000_000, 100_000_000, 256) if small else (50_000_000, 500_000_000, 256)
    t0 = time.time()
    g = eb.Graph.rmat(n, E, seed=43, feat_dim=D)
    torch.cuda.synchronize()
    build_s = time.time() - t0
    eb.set_graph(g, rng="minstd", seed=12345)
    B, counts = 8192, [15, 10]
    seeds = [torch.from_numpy(np.random.RandomState(10 + i).randint(1, n + 1, size=B)).cuda() for i in range(8)]
    state = {"i": 0}

    def step():
        s = seeds[state["i"] % 8]
        state["i"] += 1
        ids, ws, ts = eb.sample_fanout(s, [[0], [0]], counts)
        x0, = eb.get_dense_feature(ids[0], [0], [D])
        x1, = eb.get_dense_feature(ids[1], [0], [D])
        a0 = eb.sage_mean_aggregate(ids[1], counts[0], D)
        a1 = eb.sage_mean_aggregate(ids[2], counts[1], D)
        return ids, a0, a1
    ms = timeit(step, 50, warm=5)
    ids, a0, a1 = step()
    edges = B * 15 + B * 150
    ok = bool(((ids[2] >= -1) & (ids[2] <= n)).all().item()) and bool(torch.isfinite(a1).all().item())
    harness.emit({"config": "C4 on one GPU", "nodes": n, "edges": E, "feat_dim": D, "hbm_graph_gb": g.hbm_bytes / 1e9,
                  "graph_build_s": build_s, "batch": B, "fanout": counts, "ms_per_step_single_lane": ms,
                  "sampled_edges_per_s_single_lane": edges / (ms * 1e-3), "outputs_in_range": ok,
                  "valid_fraction_hop2": float((ids[2] != -1).float().mean().item()), "gpu": harness.gpu_info(0)})
    g.close()


def c5(small):
    n, E, T, NT, D = (5_000_000, 40_000_000, 5, 3, 64) if small else (50_000_000, 400_000_000, 5, 3, 64)
    g = eb.Graph.rmat_hetero(n, E, T, NT, feat_dim=D)
    eb.set_graph(g, rng="minstd", seed=12345)
    B, count = 8192, 10
    seeds = eb.sample_node(B, '-1')            # global weighted node sampler produces the batch (node_estimator.py:30-33)
    src = torch.arange(B, dtype=torch.int32, device="cuda").repeat_interleave(count)

    def step():
        outs = []
        for t in range(T):                      # RGCN: one relation at a time (K = 1 edge type per call)
            ids, w, ty = eb.sample_neighbor(seeds, [t], count)
            x, = eb.get_dense_feature(ids.reshape(-1), [0], [D])
            outs.append(eb.scatter_add(x, src, B))
        return outs
    ms = timeit(step, 20, warm=3)
    outs = step()
    types = eb.sample_neighbor(seeds, list(range(T)), count)[2]
    harness.emit({"config": "C5 hetero on one GPU", "nodes": n, "edges": E, "edge_types": T, "node_types": NT, "feat_dim": D,
                  "batch": B, "count": count, "ms_per_step": ms, "sampled_edges_per_s": B * count * T / (ms * 1e-3),
                  "agg_finite": bool(all(torch.isfinite(o).all().item() for o in outs)),
                  "types_seen_all_mode": sorted(set(types.unique().tolist())), "gpu": harness.gpu_info(0)})
    g.close()


if __name__ == "__main__":
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", choices=["c3", "c4", "c5"], help="default: all three")
    p.add_argument("--small", action="store_true")
    args = p.parse_args()
    harness.divert_stdout()
    import torch
    import euler_b200 as eb
    for w in args.configs or ["c3", "c4", "c5"]:
        {"c3": c3, "c4": c4, "c5": c5}[w](args.small)
