#!/usr/bin/env python
"""ShallowEncoder's input row on one H100: the fused op (ops.shallow_encode) against the composition a user writes today,
cat(F.embedding, get_dense_feature, sparse_feature_embedding per slot).

    python benchmarks/shallow_encoder.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E] [--big-rows R]

Graph: the R-MAT of BASELINE configs[1] (10M nodes / 100M edges) with a dense slot of D = 128 columns, rebuilt by
Graph.from_csr with the two seeded uint64 slots of benchmarks/sparse_embedding.py (u64_0: 0-8 values, Zipf-like over
[0, 10^6), 0.1 % of the nodes with 300-2000 values; u64_1: 1-4 values uniform over [0, 10^7)).  Encoder: an id table of
N + 2 rows at dim 16, the dense slot, and both slots at dim 16 (sum), 'concat': rows of 16 + 128 + 32 = 176 columns.
Workload: SageEncoder's input step, batch 8192, fanout [15, 10]: every hop's ids encoded (1.36M rows; a row without
neighbours is padded with node N + 1, the id table's last row, as upstream pads with max_id + 1).  Arms, fused and
composed: forward; forward + backward with dense table gradients; forward + backward with sparse COO gradients (composed:
F.embedding(sparse=True) and sparse_feature_embedding(sparse_grad=True)).  A GATE first checks, on the timed hops, the fused
forward bit for bit against the composition, the fused slot-table gradients bit for bit against sparse_feature_embedding's,
the id-table gradient within 1e-5 of F.embedding's, and every sparse gradient equal to its dense rows; a mismatch aborts.
The arms alternate in rounds in one process.  Then a large-vocabulary case: slot u64_1's table grown to --big-rows rows
(100M x 16 = 6.4 GB), forward + backward with dense and with sparse gradients, fused.  Reported per arm: ms per call, rows
per second and torch's allocator peak above the inputs; the card's name, power limit and SM clock read in the same run.
Anything not run is reported as "not measured".  One JSON line on stdout."""
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
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--big-rows", type=int, default=100_000_000, help="rows of the large-vocabulary slot table (0: skip)")
    return p.parse_args(argv)


def composed(eb, F, nodes, id_table, tables, sparse_grad):
    parts = [F.embedding(nodes, id_table, sparse=sparse_grad)] + eb.get_dense_feature(nodes, ["feat0"], [DENSE_DIM])
    parts += [eb.sparse_feature_embedding(nodes, name, t, dflt, "sum", sparse_grad=sparse_grad) for (name, dflt), t in zip(SLOTS, tables)]
    return torch.cat(parts, 1)


def fused(eb, nodes, id_table, tables, sparse_grad):
    sparse = [(name, t, dflt) for (name, dflt), t in zip(SLOTS, tables)]
    return eb.shallow_encode(nodes, id_table, [("feat0", DENSE_DIM)], sparse, "concat", sparse_grad=sparse_grad)


def make_arms(eb, F, hops, id_table, tables):
    params = [id_table] + list(tables)

    def fwd(fn, sparse_grad=False):
        return [fn(h, sparse_grad) for h in hops]

    def fwd_bwd(fn, sparse_grad):
        outs = fwd(fn, sparse_grad)
        torch.autograd.grad(outs, params, [torch.ones_like(o) for o in outs])

    fu = lambda n, s: fused(eb, n, id_table, tables, s)          # noqa: E731
    co = lambda n, s: composed(eb, F, n, id_table, tables, s)     # noqa: E731
    return {
        "fused_fwd": lambda: fwd(fu),
        "composed_fwd": lambda: fwd(co),
        "fused_fwd_bwd_dense": lambda: fwd_bwd(fu, False),
        "composed_fwd_bwd_dense": lambda: fwd_bwd(co, False),
        "fused_fwd_bwd_sparse": lambda: fwd_bwd(fu, True),
        "composed_fwd_bwd_sparse": lambda: fwd_bwd(co, True),
    }


def gate(eb, F, hops, id_table, tables):
    params = [id_table] + list(tables)
    nodes = torch.cat(hops)
    a = fused(eb, nodes, id_table, tables, False)
    b = composed(eb, F, nodes, id_table, tables, False)
    if not torch.equal(a.view(torch.int32), b.view(torch.int32)):
        raise SystemExit("GATE FAILED: the fused forward differs from the composition")
    g = torch.randn_like(a)
    ga = torch.autograd.grad(a, params, g)
    gb = torch.autograd.grad(b, params, g, retain_graph=True)
    for t in range(1, len(params)):
        if not torch.equal(ga[t], gb[t]):
            raise SystemExit("GATE FAILED: slot table %d's gradient differs from sparse_feature_embedding's" % t)
    mag = torch.autograd.grad(b, params[:1], g.abs())[0]
    if ((ga[0] - gb[0]).abs() > 1e-5 * mag + 1e-7).any():
        raise SystemExit("GATE FAILED: the id table's gradient differs from F.embedding's")
    gs = torch.autograd.grad(fused(eb, nodes, id_table, tables, True), params, g)
    for t in range(len(params)):
        if not (gs[t].is_sparse and torch.equal(gs[t].to_dense(), ga[t])):
            raise SystemExit("GATE FAILED: table %d's sparse gradient differs from its dense one" % t)


def run(args):
    global torch
    import torch
    import torch.nn.functional as F
    import euler_b200 as eb
    torch.cuda.set_device(0)
    fanout = [int(x) for x in args.fanout.split(",")]
    t0 = time.time()
    _g = build_graph(args)
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=args.batch).astype(np.int64)).cuda()
    hops = eb.sample_fanout(seeds, [[0]] * len(fanout), fanout, default_node=args.nodes + 1)[0]   # the id table's last row
    rows = sum(h.numel() for h in hops)
    gen = torch.Generator(device="cuda").manual_seed(1)
    id_table = (torch.randn(args.nodes + 2, DIM, device="cuda", generator=gen) * 0.1).requires_grad_(True)
    tables = [(torch.randn(m + 1, DIM, device="cuda", generator=gen) * 0.01).requires_grad_(True) for _, m in SLOTS]
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    gate(eb, F, hops, id_table, tables)
    res = timed(make_arms(eb, F, hops, id_table, tables), args.steps, args.warmup)
    for v in res.values():
        v["rows_per_sec"] = rows / (v["ms_per_call"] * 1e-3)
    big = {"fused_fwd_bwd_dense": "not measured", "fused_fwd_bwd_sparse": "not measured"}
    if args.big_rows:
        big_tables = [tables[0], torch.zeros(args.big_rows, DIM, device="cuda").requires_grad_(True)]
        arms = make_arms(eb, F, hops, id_table, big_tables)
        big = timed({k: arms[k] for k in big}, max(1, args.steps // 4), 1)
        big["table_bytes"] = args.big_rows * DIM * 4
        del big_tables, arms
    harness.emit({"metric": "shallow_encoder_fwd_rows_per_sec", "value": res["fused_fwd"]["rows_per_sec"], "gate": "passed",
                  "gpu": harness.gpu_info(0), "batch": args.batch, "fanout": fanout, "rows": rows, "row_width": DIM + DENSE_DIM + DIM * len(SLOTS),
                  "setup_s": setup_s, "arms": res, "large_vocabulary": {"rows": args.big_rows, "dim": DIM, "arms": big}})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
