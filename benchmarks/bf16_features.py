#!/usr/bin/env python
"""bfloat16 dense-feature storage on one H100: the same graph with an f32 and a bf16 feature table, and the graph that only
fits with bf16.

    python benchmarks/bf16_features.py [--part A|B|AB] [--rounds R] [--iters K]

Part A.  R-MAT 20M nodes / 200M edges, D = 256, the same seeds, built once per dtype and both resident.  On the hop-2 ids of
a batch-1024 [25, 10], a batch-8192 [15, 10] and a batch-16384 [15, 10] fanout (the last one's 245,760 mean rows cross the
2^17-row segment-dedup path; the batch-8192 one's 122,880 stay below it):
  - a CHECK first, else it aborts: get_dense_feature on the bf16 graph equals the f32 graph's rows rounded to bf16, and
    sage_mean_aggregate on the bf16 graph equals the f32 op's defined order (rows added left to right from +0.0, divided by
    fl(count + 1e-7)) over those rounded rows, bit for bit;
  - then get_dense_feature and sage_mean_aggregate, f32 and bf16 alternating round by round, timed with device events.
  Reported per arm: ms per call, the algorithmic bytes (get_dense_feature: M (s + 4) D, the row read at s bytes an element
  and written as f32; the mean: rows (count s D + 4 D)) and the achieved GB/s.  Hub rows are served from L2, so the rate
  can exceed what HBM alone would give and the bf16 gain can fall short of the byte ratio.
Part B.  Graph.rmat(100M, 1B, feat_dim=256, feat_dtype='bfloat16'): hbm_bytes, free device memory after the build and the
lowest free memory seen during it (sampled every 20 ms), then one batch-8192 [15, 10] fanout with mean aggregation timed, and
4096 sampled hop-2 rows checked against the oracle's R-MAT feature rows (oracle/pyoracle.py) rounded to bf16.  A build that
does not fit is reported with what was seen, not retried smaller.
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout; it needs a GPU."""
import argparse
import threading
import time

import harness
import numpy as np
import torch

import bf16_reference as br

D, FEAT_SEED, GRAPH_SEED = 256, 7, 42
WORKLOADS = [(1024, [25, 10]), (8192, [15, 10]), (16384, [15, 10])]


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--part", default="AB", choices=["A", "B", "AB"])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--iters", type=int, default=10)
    return p.parse_args(argv)


def bits(t):
    return t.contiguous().view(torch.int32)


def as_bf16(t):
    """f32 tensor -> its bf16 rounding widened back (torch's device conversion: round to nearest even)"""
    return t.to(torch.bfloat16).float()


def mean_in_order(rows, count):
    """the fused mean's defined order over [R * count, D] fetched rows: added left to right from +0.0, divided once"""
    x = rows.view(-1, count, rows.shape[1])
    acc = torch.zeros_like(x[:, 0])
    for j in range(count):
        acc = acc + x[:, j]
    return acc / (torch.tensor(float(count), dtype=torch.float32) + torch.tensor(1e-7, dtype=torch.float32)).cuda()


def hop2(graph, batch, fanout, seed):
    import euler_b200
    euler_b200.set_graph(graph, rng="minstd", seed=seed)
    seeds = torch.randint(1, graph.num_nodes + 1, (batch,), generator=torch.Generator().manual_seed(seed)).cuda()
    ids, _, _ = euler_b200.sample_fanout(seeds, [[0], [0]], fanout)
    return ids[2]


def part_a(args):
    import euler_b200
    t0 = time.time()
    gf = euler_b200.Graph.rmat(20_000_000, 200_000_000, seed=GRAPH_SEED, feat_dim=D, feat_seed=FEAT_SEED)
    gb = euler_b200.Graph.rmat(20_000_000, 200_000_000, seed=GRAPH_SEED, feat_dim=D, feat_seed=FEAT_SEED, feat_dtype="bfloat16")
    torch.cuda.synchronize()
    out = {"graph": "rmat 20M nodes / 200M edges, D = 256", "build_s": round(time.time() - t0, 1),
           "hbm_bytes": {"float32": gf.hbm_bytes, "bfloat16": gb.hbm_bytes}, "workloads": []}
    graphs = {"float32": gf, "bfloat16": gb}
    for batch, fanout in WORKLOADS:
        ids = hop2(gf, batch, fanout, seed=batch)
        count, M = fanout[1], ids.numel()
        R = M // count
        res = {"batch": batch, "fanout": fanout, "feature_rows": M, "mean_rows": R}
        got = {}
        for name, g in graphs.items():
            euler_b200.set_graph(g)
            got[name] = (euler_b200.get_dense_feature(ids, [0], [D])[0], euler_b200.sage_mean_aggregate(ids, count, D))
        want_rows = as_bf16(got["float32"][0])
        if not torch.equal(bits(got["bfloat16"][0]), bits(want_rows)):
            raise SystemExit("CHECK FAILED: bf16 get_dense_feature differs from the rounded f32 rows (batch %d)" % batch)
        if not torch.equal(bits(got["bfloat16"][1]), bits(mean_in_order(want_rows, count))):
            raise SystemExit("CHECK FAILED: bf16 sage_mean_aggregate differs from the f32 order over the rounded rows (batch %d)" % batch)
        res["check"] = "bit-exact"
        del got, want_rows
        for op in ("get_dense_feature", "sage_mean_aggregate"):
            arms = {}
            for name, g in graphs.items():
                ctx = euler_b200.Context(g)
                ctx.set_stream(torch.cuda.current_stream().cuda_stream)
                o = torch.empty((M if op == "get_dense_feature" else R, D), device="cuda")
                if op == "get_dense_feature":
                    arms[name] = (lambda c=ctx, o=o: euler_b200._lib.check(euler_b200._lib.load().eu_get_dense_feature(
                        c._h, ids.data_ptr(), M, 0, D, o.data_ptr())), ctx)
                else:
                    arms[name] = (lambda c=ctx, o=o: euler_b200._lib.check(euler_b200._lib.load().eu_sage_mean_aggregate(
                        c._h, ids.data_ptr(), R, count, D, o.data_ptr())), ctx)
            ms = {k: float(np.mean(v)) for k, v in harness.time_arms({k: v[0] for k, v in arms.items()}, args.rounds, 1, args.iters).items()}
            for name in graphs:
                s = 4 if name == "float32" else 2
                nbytes = M * (s + 4) * D if op == "get_dense_feature" else R * (count * s * D + 4 * D)
                res["%s_%s" % (op, name)] = {"ms": round(ms[name], 4), "bytes": nbytes, "GB_per_s": round(nbytes / ms[name] / 1e6, 1)}
            res["%s_f32_over_bf16" % op] = round(ms["float32"] / ms["bfloat16"], 3)
            for _, ctx in arms.values():
                ctx.close()
        out["workloads"].append(res)
        del ids
    euler_b200.set_graph(None)
    gf.close()
    gb.close()
    torch.cuda.empty_cache()
    return out


def part_b(args):
    import euler_b200
    from oracle import pyoracle as po
    n, E = 100_000_000, 1_000_000_000
    free0, total = torch.cuda.mem_get_info()
    low = [free0]
    stop = threading.Event()

    def watch():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info()[0])
            time.sleep(0.02)
    th = threading.Thread(target=watch, daemon=True)
    th.start()
    t0 = time.time()
    out = {"graph": "rmat 100M nodes / 1B edges, D = 256, bfloat16", "free_before_bytes": free0, "device_bytes": total}
    try:
        g = euler_b200.Graph.rmat(n, E, seed=GRAPH_SEED, feat_dim=D, feat_seed=FEAT_SEED, feat_dtype="bfloat16")
        torch.cuda.synchronize()
    except euler_b200.EulerError as e:
        stop.set()
        th.join()
        out.update(fits=False, error=str(e), lowest_free_during_build_bytes=low[0])
        return out
    stop.set()
    th.join()
    out.update(fits=True, build_s=round(time.time() - t0, 1), hbm_bytes=g.hbm_bytes, free_after_build_bytes=torch.cuda.mem_get_info()[0],
               lowest_free_during_build_bytes=low[0])
    euler_b200.set_graph(g, rng="minstd", seed=5)
    seeds = torch.randint(1, n + 1, (8192,), generator=torch.Generator().manual_seed(5)).cuda()

    last = {}

    def step():
        last["ids"], _, _ = euler_b200.sample_fanout(seeds, [[0], [0]], [15, 10])
        return euler_b200.sage_mean_aggregate(last["ids"][2], 10, D)
    times = harness.time_arms({"step": step}, args.rounds, 1)["step"]
    ids = last["ids"]
    out["fanout_mean_step_ms"] = {"min": round(min(times), 3), "median": round(float(np.median(times)), 3), "steps": len(times)}
    pick = ids[2][torch.randint(0, ids[2].numel(), (4096,), generator=torch.Generator().manual_seed(6)).cuda()]
    got = euler_b200.get_dense_feature(pick, [0], [D])[0].cpu().numpy()
    want = br.rounded(po.rmat_feat_rows(pick.cpu().numpy(), n, D, FEAT_SEED))
    if not np.array_equal(got.view(np.uint32), want.view(np.uint32)):
        raise SystemExit("CHECK FAILED: 100M-node bf16 rows differ from the oracle's R-MAT rows rounded to bf16")
    out["rows_checked"] = {"rows": 4096, "against": "oracle R-MAT feature rows rounded to bf16", "result": "bit-exact"}
    euler_b200.set_graph(None)
    g.close()
    return out


def main():
    args = parse()
    if not torch.cuda.is_available():
        raise SystemExit("bf16_features.py needs a GPU")
    res = {"benchmark": "bf16_features", "gpu": harness.gpu_info(torch.cuda.current_device())}
    if "A" in args.part:
        res["A"] = part_a(args)
    if "B" in args.part:
        res["B"] = part_b(args)
    harness.emit(res)


if __name__ == "__main__":
    harness.divert_stdout()
    main()
