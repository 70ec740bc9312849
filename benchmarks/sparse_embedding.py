#!/usr/bin/env python
"""SparseEmbedding's input path on one H100: the fused lookup from node ids (ops.sparse_feature_embedding) against the
composition a user writes today, get_sparse_feature + torch.nn.functional.embedding_bag.

    python benchmarks/sparse_embedding.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Graph: the R-MAT of BASELINE configs[1] (10M nodes / 100M edges), exported and rebuilt by Graph.from_csr with two seeded
uint64 slots: u64_0 ("A") 0-8 values per node, about 20 % empty, Zipf-like over [0, 10^6), plus 0.1 % of the nodes with
300-2000 values; u64_1 ("B") 1-4 values, uniform over [0, 10^7).  Tables have max_id + 2 rows, the default the last one.
Workload: SageEncoderNew's input step, batch 8192, fanout [15, 10] (1.36M embedded rows per slot), dim 16 and 64, sum and
mean.  Arms:
  (a) lookup: the embedding of every hop's rows for both slots, fused vs get_sparse_feature + embedding_bag;
  (b) step:   sample_fanout + the fused lookups vs sample_fanout_with_feature + embedding_bag (the reference's input step);
each forward and forward + backward (the gradient reaches the tables).  Before timing a GATE checks, per (dim, combiner),
the fused forward bit for bit against the float32 restatement on 512 sampled rows and the fused gradient within 1e-5 of
float64 on 4096 hop-2 rows; a mismatch aborts.  The arms alternate in rounds in one process.  Reported per arm: ms per
call, embedded rows per second, torch's allocator peak above the inputs, the algorithmic bytes (entries * dim * 4 read,
rows * dim * 4 written), and the card's name, power limit and SM clock read in the same run.  One JSON line on stdout."""
import argparse
import time

import harness
import numpy as np

from bench import GRAPH_SEED
from harness import SLOTS, slot_arrays


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=8192)
    p.add_argument("--fanout", default="15,10")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def build_graph(args):
    import euler_b200 as eb
    g0 = eb.Graph.rmat(args.nodes, args.edges, seed=GRAPH_SEED, device=0)
    csr = g0.export(with_feat=False)
    g0.close()
    ptr, vals = slot_arrays(args.nodes)
    g = eb.Graph.from_csr(csr["ids"], csr["grp_ptr"], csr["nbr"], n_edge_types=csr["T"], cum_w=csr["cum_w"], grp_cum=csr["grp_cum"],
                          node_type=csr["node_type"], node_w=csr["node_w"], u64_ptr=ptr, u64_val=vals, n_u64_slots=2)
    eb.set_graph(g, rng="philox", seed=5)
    return g, csr["ids"], ptr, vals


def composed(eb, F, nodes, name, table, default, combiner):
    (idx, v, _), = eb.get_sparse_feature(nodes, [name], [default])
    offsets = torch.searchsorted(idx[:, 0].contiguous(), torch.arange(nodes.numel(), device=nodes.device))
    return F.embedding_bag(v, table, offsets, mode=combiner)


def bag_sums(F, sparse, tables, combiner):
    """embedding_bag over sample_fanout_with_feature's hop-major (indices, values, dense_shape) triples"""
    out = []
    for k, (idx, v, shape) in enumerate(sparse):
        offsets = torch.searchsorted(idx[:, 0].contiguous(), torch.arange(shape[0], device=v.device))
        out.append(F.embedding_bag(v, tables[k % len(SLOTS)], offsets, mode=combiner))
    return out


def make_arms(eb, F, seeds, fanout, hops, tables, combiner):
    def lookups(fn, hop_ids):
        return [fn(h, name, tables[k], SLOTS[k][1], combiner) for h in hop_ids for k, (name, _) in enumerate(SLOTS)]

    fused = lambda n, nm, t, d, c: eb.sparse_feature_embedding(n, nm, t, d, c)   # noqa: E731
    comp = lambda n, nm, t, d, c: composed(eb, F, n, nm, t, d, c)                # noqa: E731

    def sample():
        return eb.sample_fanout(seeds, [[0]] * len(fanout), fanout)[0]

    def step_composed():   # the reference's input step: sample_fanout_with_feature, then embedding_lookup_sparse per hop and slot
        sparse = eb.sample_fanout_with_feature(seeds, [[0]] * len(fanout), fanout, -1, [], [], [n for n, _ in SLOTS],
                                               [d for _, d in SLOTS])[4]
        return bag_sums(F, sparse, tables, combiner)

    def backward(outs):
        torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
        for t in tables:
            t.grad = None

    return {
        "lookup_fused_fwd": lambda: lookups(fused, hops),
        "lookup_composed_fwd": lambda: lookups(comp, hops),
        "lookup_fused_fwd_bwd": lambda: backward(lookups(fused, hops)),
        "lookup_composed_fwd_bwd": lambda: backward(lookups(comp, hops)),
        "step_fused_fwd": lambda: lookups(fused, sample()),
        "step_composed_fwd": step_composed,
        "step_fused_fwd_bwd": lambda: backward(lookups(fused, sample())),
        "step_composed_fwd_bwd": lambda: backward(step_composed()),
    }


def gate(eb, er, ids, ptr, vals, hops, tables, combiner):
    rng = np.random.RandomState(1)
    for k, (name, dflt) in enumerate(SLOTS):
        table = tables[k].detach()
        rows = torch.cat(hops)[torch.as_tensor(rng.randint(0, sum(h.numel() for h in hops), size=512), device="cuda")]
        bl = er.bags(ids, ptr, vals, 2, rows.cpu().numpy(), k, dflt)
        sub = torch.as_tensor(sorted({v for b in bl for v in b}), device="cuda")
        want = er.lookup_f32(table[sub].cpu().numpy(), [list(np.searchsorted(sub.cpu().numpy(), b)) for b in bl], combiner)
        got = eb.sparse_feature_embedding(rows, name, table, dflt, combiner).cpu().numpy()
        if got.tobytes() != want.tobytes():
            raise SystemExit("GATE FAILED: fused forward differs from the float32 restatement (%s, %s)" % (name, combiner))
        rows = hops[-1][:4096]
        g = torch.randn(rows.numel(), table.shape[1], device="cuda")
        t = table.clone().requires_grad_(True)
        eb.sparse_feature_embedding(rows, name, t, dflt, combiner).backward(g)
        bl = er.bags(ids, ptr, vals, 2, rows.cpu().numpy(), k, dflt)
        touched = np.asarray(sorted({v for b in bl for v in b}))
        want, mag = np.zeros((len(touched), table.shape[1])), np.zeros((len(touched), table.shape[1]))
        pos = {int(v): j for j, v in enumerate(touched)}
        gn = g.cpu().numpy().astype(np.float64)
        for i, b in enumerate(bl):
            for v in b:
                want[pos[v]] += gn[i] / (len(b) if combiner == "mean" else 1.0)
                mag[pos[v]] += np.abs(gn[i]) / (len(b) if combiner == "mean" else 1.0)
        got = t.grad[torch.as_tensor(touched, device="cuda")].cpu().numpy()
        # within 1e-5 of float64, relative to the sum of the terms' magnitudes (a long sum may cancel, its rounding may not)
        if (np.abs(got - want) > 1e-5 * mag + 1e-7).any() or int((t.grad != 0).any(1).sum()) > len(touched):
            raise SystemExit("GATE FAILED: fused gradient differs from float64 (%s, %s): worst relative error %g"
                             % (name, combiner, float((np.abs(got - want) / (mag + 1e-30)).max())))


def run(args):
    global torch
    import torch
    import torch.nn.functional as F
    import euler_b200 as eb
    import embedding_reference as er
    torch.cuda.set_device(0)
    fanout = [int(x) for x in args.fanout.split(",")]
    t0 = time.time()
    _g, ids, ptr, vals = build_graph(args)
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=args.batch).astype(np.int64)).cuda()
    hops = eb.sample_fanout(seeds, [[0]] * len(fanout), fanout)[0]
    torch.cuda.synchronize()
    setup_s = time.time() - t0
    rows = sum(h.numel() for h in hops)
    entries = {}
    for k, (name, dflt) in enumerate(SLOTS):
        (idx, _, _), = [x for x in eb.get_sparse_feature(torch.cat(hops), [name], [dflt])]
        entries[name] = int(idx.shape[0])
    results = []
    for dim in (16, 64):
        for combiner in ("sum", "mean"):
            gen = torch.Generator(device="cuda").manual_seed(dim)
            tables = [(torch.randn(m + 1, dim, device="cuda", generator=gen) * 0.01).requires_grad_(True) for _, m in SLOTS]
            gate(eb, er, ids, ptr, vals, hops, tables, combiner)
            res = harness.timed(make_arms(eb, F, seeds, fanout, hops, tables, combiner), args.steps, args.warmup)
            alg = 4 * dim * (sum(entries.values()) + rows * len(SLOTS))
            for v in res.values():
                v["rows_per_sec"] = rows * len(SLOTS) / (v["ms_per_call"] * 1e-3)
            results.append({"dim": dim, "combiner": combiner, "algorithmic_fwd_bytes": alg, "arms": res})
            del tables
    head = [r for r in results if r["dim"] == 64 and r["combiner"] == "sum"][0]["arms"]
    harness.emit({"metric": "sparse_embedding_lookup_rows_per_sec", "value": head["lookup_fused_fwd"]["rows_per_sec"],
                  "gate": "passed", "gpu": harness.gpu_info(0), "batch": args.batch, "fanout": fanout, "rows_per_slot": rows,
                  "entries_per_slot": entries, "setup_s": setup_s, "results": results})


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
