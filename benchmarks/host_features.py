#!/usr/bin/env python
"""Dense node features in mapped pinned host memory on one H100: the headline step's feature work with the table in HBM and
with it on the host behind HBM caches of several sizes.

    python benchmarks/host_features.py [--full] [--rounds R] [--iters K]

Part A.  R-MAT 10M nodes / 100M edges, D = 256, for f32 and bf16.  One batch-8192 [15, 10] fanout is sampled once; the
step's feature work is get_dense_feature of the seeds and of hop 1, and sage_mean_aggregate of hops 1 and 2 (the means of
the hop-1 and hop-2 segments).  Arms: the device-placed table, and host-placed tables with feat_cache_rows C = 0, 1 %, 10 %
and 25 % of n, built one at a time.  Each host arm is first CHECKED, else the run aborts: its four outputs must equal the
device arm's bit for bit.  Then the device arm and the host arm alternate round by round, timed with device events.
Reported per arm: ms per step, the cache hit rate (rows read from HBM / rows read, over the existing rows the four calls
read), and the row bytes read from the host table (rows not in the cache x D x element size; the GPU's caches may serve
some of them again, so this bounds what crosses the host link).
Part B (--full, only when MemAvailable exceeds the f32 table by 32 GB).  Graph.rmat(100M, 1B, feat_dim=256) with the f32
table on the host (102.4 GB pinned) and a 10 % cache: one batch-8192 [15, 10] fanout with both means timed, and 4096 hop-2
rows checked against the oracle's R-MAT feature rows (oracle/pyoracle.py).
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout; it needs a GPU."""
import argparse
import sys
import time

import harness
import numpy as np
import torch


D, FEAT_SEED, GRAPH_SEED = 256, 7, 42
CACHE_FRACTIONS = (0.0, 0.01, 0.10, 0.25)


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--full", action="store_true")
    p.add_argument("--rounds", type=int, default=7)
    p.add_argument("--iters", type=int, default=5)
    p.add_argument("--nodes", type=int, default=10_000_000)
    return p.parse_args(argv)


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def bits(t):
    return t.contiguous().view(torch.int32)


def sample(graph, batch=8192, fanout=(15, 10), seed=8192):
    import euler_b200
    euler_b200.set_graph(graph, rng="minstd", seed=seed)
    seeds = torch.randint(1, graph.num_nodes + 1, (batch,), generator=torch.Generator().manual_seed(seed)).cuda()
    ids, _, _ = euler_b200.sample_fanout(seeds, [[0], [0]], list(fanout))
    return ids[0], ids[1], ids[2]


def step(graph, seeds, hop1, hop2):
    """the headline step's feature work"""
    import euler_b200
    euler_b200.set_graph(graph)
    return [euler_b200.get_dense_feature(seeds, [0], [D])[0], euler_b200.get_dense_feature(hop1, [0], [D])[0],
            euler_b200.sage_mean_aggregate(hop1, 15, D), euler_b200.sage_mean_aggregate(hop2, 10, D)]


def reads(slots, n, seeds, hop1, hop2):
    """(rows read, rows read from the cache) over the existing rows the four calls read"""
    ids = np.concatenate([x.cpu().numpy() for x in (seeds, hop1, hop1, hop2)]).astype(np.int64)
    ids = ids[(ids >= 1) & (ids <= n)]
    return int(ids.size), int((slots[ids - 1] >= 0).sum())


def part_a(args):
    import euler_b200
    n, E = args.nodes, 10 * args.nodes
    out = {"graph": "rmat %dM nodes / %dM edges, D = %d" % (n // 10**6, E // 10**6, D), "batch": 8192, "fanout": [15, 10],
           "arms": []}
    for dt in ("float32", "bfloat16"):
        es = 4 if dt == "float32" else 2
        if mem_available() < 2 * n * D * es:
            out["arms"].append({"dtype": dt, "skipped": "MemAvailable %.1f GB < twice the %.1f GB table"
                                % (mem_available() / 1e9, n * D * es / 1e9)})
            continue
        gd = euler_b200.Graph.rmat(n, E, seed=GRAPH_SEED, feat_dim=D, feat_seed=FEAT_SEED, feat_dtype=dt)
        seeds, hop1, hop2 = sample(gd)
        want = step(gd, seeds, hop1, hop2)
        torch.cuda.synchronize()
        for frac in CACHE_FRACTIONS:
            C = int(round(frac * n))
            t0 = time.time()
            gh = euler_b200.Graph.rmat(n, E, seed=GRAPH_SEED, feat_dim=D, feat_seed=FEAT_SEED, feat_dtype=dt, feat_place="host",
                                       feat_cache_rows=C)
            torch.cuda.synchronize()
            build_s = time.time() - t0
            got = step(gh, seeds, hop1, hop2)
            for a, b in zip(want, got):
                if not torch.equal(bits(a), bits(b)):
                    raise SystemExit("CHECK FAILED: host-placed %s C=%d differs from the device arm" % (dt, C))
            rows, hits = reads(gh.feat_cache_slots(), n, seeds, hop1, hop2)
            ms = harness.time_arms({"device": lambda: step(gd, seeds, hop1, hop2), "host": lambda: step(gh, seeds, hop1, hop2)},
                                   args.rounds, 1, args.iters)
            ms = {k: float(np.mean(v)) for k, v in ms.items()}
            out["arms"].append({"dtype": dt, "cache_rows": C, "cache_fraction": frac, "check": "bit-exact",
                                "device_ms": round(ms["device"], 3), "host_ms": round(ms["host"], 3),
                                "host_over_device": round(ms["host"] / ms["device"], 2),
                                "rows_read": rows, "cache_hit_rate": round(hits / max(rows, 1), 4),
                                "host_row_bytes": (rows - hits) * D * es, "build_s": round(build_s, 1),
                                "hbm_bytes": gh.hbm_bytes, "host_bytes": gh.host_bytes, "device_hbm_bytes": gd.hbm_bytes})
            print(out["arms"][-1], file=sys.stderr, flush=True)
            euler_b200.set_graph(gd)          # drops this thread's context of gh before gh is freed
            gh.close()
            del gh
        euler_b200.set_graph(None)
        gd.close()
        del gd
    return out


def part_b():
    import euler_b200
    from oracle import pyoracle as po
    n, E = 100_000_000, 1_000_000_000
    table = n * D * 4
    if mem_available() < table + (32 << 30):
        return {"skipped": "MemAvailable %.1f GB < the %.1f GB f32 table + 32 GB" % (mem_available() / 1e9, table / 1e9)}
    t0 = time.time()
    g = euler_b200.Graph.rmat(n, E, seed=GRAPH_SEED, feat_dim=D, feat_seed=FEAT_SEED, feat_place="host",
                              feat_cache_rows=n // 10)
    torch.cuda.synchronize()
    res = {"graph": "rmat 100M / 1B, D = 256, f32 on the host, 10 % cache", "build_s": round(time.time() - t0, 1),
           "hbm_bytes": g.hbm_bytes, "host_bytes": g.host_bytes, "free_device_bytes": torch.cuda.mem_get_info()[0]}
    seeds, hop1, hop2 = sample(g)
    res["step_feature_ms"] = round(harness.time_arms({"step": lambda: step(g, seeds, hop1, hop2)}, 1, 1)["step"][0], 3)
    pick = hop2[torch.randperm(hop2.numel(), generator=torch.Generator().manual_seed(1))[:4096].cuda()]
    got = euler_b200.get_dense_feature(pick, [0], [D])[0].cpu().numpy()
    want = po.rmat_feat_rows(pick.cpu().numpy(), n, D, FEAT_SEED)
    res["check_4096_hop2_rows"] = "bit-exact" if np.array_equal(got.view(np.uint32), want.view(np.uint32)) else "FAILED"
    euler_b200.set_graph(None)
    g.close()
    return res


def main(argv=None):
    args = parse(argv)
    out = {"benchmark": "host_features", "gpu": harness.gpu_info(0), "part_a": part_a(args)}
    if args.full:
        out["part_b"] = part_b()
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    main()
