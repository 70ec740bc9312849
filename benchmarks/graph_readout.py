#!/usr/bin/env python
"""Graph classification's batch construction and readout on one H100: the fused attention readout
(ops.graph_attention_readout) against the same readout composed from the mp ops (scatter_softmax, multiply, scatter_add; for
Set2Set the gather -> multiply -> sum logits first), forward and forward + backward, and the two batch-construction ops alone.

    python benchmarks/graph_readout.py [--steps K] [--warmup W] [--graphs G] [--batch B]

Workload: a disjoint union of G = 1M molecule-like graphs (a ring of 10-60 nodes, every fifth node with a chord across the
ring), built with Graph.from_csr, with a binary graph_label slot.  A step = sample_graph_label(B = 4096) ->
get_graph_by_label -> the 5-hop GCNDataFlow without self loops the gin example runs -> the readout of the batch's rows
(x = seeded random [nnz, D], D = 64 and 128; AttentionPool's gate and Set2Set's query are seeded random tensors).

Before anything is timed a PARITY GATE checks, per D, AttentionPool's fused forward bit for bit against the composition
(every graph has at most 256 rows) and Set2Set's within 1e-5, and both fused backward passes within 1e-4 of autograd through
the composition; a mismatch aborts.  The arms then alternate in rounds in one process.  Reported: ms per call per arm, the
torch allocator's peak above the inputs per arm (the library's own ctx scratch is not in it), the batch-construction ops'
ms per call, and the card's name and power limit read in the same run.  One JSON line on stdout; nothing is written to the
tree."""
import argparse
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402

from full_dataflow import emit, gpu_info  # noqa: E402

DIMS = (64, 128)


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--graphs", type=int, default=1_000_000)
    p.add_argument("--batch", type=int, default=4096)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def molecule_union(G, seed=11):
    """CSR arrays of G ring-with-chords graphs of 10-60 nodes and each node's graph label b'<k>'"""
    rs = np.random.RandomState(seed)
    s = rs.randint(10, 61, size=G).astype(np.int64)
    base = np.concatenate([[0], np.cumsum(s)[:-1]])
    N = int(s.sum())
    g = np.repeat(np.arange(G), s)
    i = np.arange(N) - base[g]
    sz, b = s[g], base[g]
    chord = i % 5 == 0
    deg = 2 + chord.astype(np.int64)
    grp_ptr = np.concatenate([[0], np.cumsum(deg)])
    nbr = np.empty(int(grp_ptr[-1]), np.uint64)
    nbr[grp_ptr[:-1]] = (b + (i - 1) % sz + 1).astype(np.uint64)          # ids are rows + 1 (0 is not a node)
    nbr[grp_ptr[:-1] + 1] = (b + (i + 1) % sz + 1).astype(np.uint64)
    nbr[grp_ptr[:-1][chord] + 2] = (b + (i + sz // 2) % sz + 1)[chord].astype(np.uint64)
    names = [b"%d" % k for k in range(G)]
    lens = np.asarray([len(x) for x in names], np.int64)
    bin_ptr = np.concatenate([[0], np.cumsum(lens[g])])
    bin_val = np.frombuffer(b"".join(names[k] for k in g.tolist()), np.uint8)
    return np.arange(1, N + 1, dtype=np.uint64), grp_ptr, nbr, bin_ptr, bin_val


def composition(ops, x, index, B, logits=None, q=None):
    e = logits.view(-1, 1) if q is None else (x * ops.gather(q, index)).sum(-1, keepdim=True)
    a = ops.scatter_softmax(e, index, B)
    return ops.scatter_add(a * x, index, B)


def main(args):
    import torch
    import euler_b200
    from euler_b200 import ops
    from euler_b200.dataflow import GCNDataFlow
    assert torch.cuda.is_available(), "graph_readout.py measures on the GPU; there is no CPU path"
    t0 = time.time()
    ids, grp_ptr, nbr, bin_ptr, bin_val = molecule_union(args.graphs)
    g = euler_b200.Graph.from_csr(ids, grp_ptr, nbr, w=np.ones(len(nbr), np.float32), bin_ptr=bin_ptr, bin_val=bin_val,
                                  n_bin_slots=1, binary_feature_names=["graph_label"])
    euler_b200.set_graph(g, rng="philox", seed=5)
    n_labels = len(ops.graph_labels())
    build_s = time.time() - t0
    B = args.batch
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731

    def timed(fn, n):
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n

    # ---- batch construction alone
    labels = ops.sample_graph_label(B)
    for _ in range(args.warmup):
        ops.get_graph_by_label(ops.sample_graph_label(B))
    construct = {"sample_graph_label_ms": timed(lambda: ops.sample_graph_label(B), max(args.steps, 1) * 5),
                 "get_graph_by_label_ms": timed(lambda: ops.get_graph_by_label(labels), max(args.steps, 1) * 5)}
    idx, vals, _ = ops.get_graph_by_label(labels)
    flow = GCNDataFlow([[0]] * 5, add_self_loops=False)
    construct["gcn_dataflow_5hop_ms"] = timed(lambda: flow(vals), max(args.steps, 1))
    index = idx[:, 0].to(torch.int32).contiguous()
    nnz = int(index.numel())
    torch.manual_seed(0)

    results, gate = {}, {}
    for D in DIMS:
        x = torch.randn(nnz, D, device="cuda")
        lg = torch.randn(nnz, device="cuda")
        q = torch.randn(B, D, device="cuda") / D ** 0.5
        g_out = torch.randn(B, D, device="cuda")
        # parity gate
        f = ops.graph_attention_readout(x, index, B, logits=lg)
        c = composition(ops, x, index, B, logits=lg)
        if not torch.equal(f, c):
            raise SystemExit("parity gate: AttentionPool forward differs from the composition at D=%d" % D)
        f = ops.graph_attention_readout(x, index, B, q=q)
        c = composition(ops, x, index, B, q=q)
        if not torch.allclose(f, c, rtol=1e-5, atol=1e-5):
            raise SystemExit("parity gate: Set2Set forward differs from the composition at D=%d" % D)
        for mode in ("logits", "q"):
            grads = []
            for fused in (True, False):
                xx = x.clone().requires_grad_()
                ww = (q if mode == "q" else lg).clone().requires_grad_()
                kw = {mode: ww}
                out = ops.graph_attention_readout(xx, index, B, **kw) if fused else composition(ops, xx, index, B, **kw)
                out.backward(g_out)
                grads.append((xx.grad, ww.grad))
            for a, b in zip(*grads):
                if not torch.allclose(a, b, rtol=1e-4, atol=1e-4):
                    raise SystemExit("parity gate: %s backward differs from autograd at D=%d" % (mode, D))
        gate[D] = "passed"

        def arm(mode, fused, backward):
            # each arm its own leaves: a forward arm runs without autograd state, as a user's no-grad readout does
            xx = x.detach().clone().requires_grad_(backward)
            ww = (q if mode == "q" else lg).detach().clone().requires_grad_(backward)

            def run():
                kw = {mode: ww}
                out = ops.graph_attention_readout(xx, index, B, **kw) if fused else composition(ops, xx, index, B, **kw)
                if backward:
                    out.backward(g_out)
                    xx.grad = None
                    ww.grad = None
            return run

        names = [(m, fu, bw) for m in ("logits", "q") for bw in (False, True) for fu in (True, False)]
        runs = {n: arm(*n) for n in names}
        mem = {}
        for n, fn in runs.items():
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            mem[n] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        times = {n: [] for n in names}
        for _ in range(3):                                   # alternate the arms in rounds
            for n, fn in runs.items():
                times[n].append(timed(fn, args.steps))
        for (m, fu, bw) in names:
            key = "D%d_%s_%s_%s" % (D, "attention_pool" if m == "logits" else "set2set_step", "fused" if fu else "composition",
                                    "fwd_bwd" if bw else "fwd")
            results[key] = {"ms_median": float(np.median(times[(m, fu, bw)])), "ms_all": times[(m, fu, bw)],
                            "peak_alloc_MiB": mem[(m, fu, bw)]}
    emit({"bench": "graph_readout", "gpu": gpu_info(0), "graphs": args.graphs, "nodes": int(len(ids)), "labels": n_labels,
          "batch": B, "batch_rows": nnz, "graph_build_s": build_s, "gate": gate, "construct": construct, "readout": results})
    print("%-48s %10s %12s" % ("arm", "ms", "peak MiB"), file=sys.stderr)
    for k, v in results.items():
        print("%-48s %10.3f %12.1f" % (k, v["ms_median"], v["peak_alloc_MiB"]), file=sys.stderr)
    for k, v in construct.items():
        print("%-48s %10.3f" % (k, v), file=sys.stderr)


if __name__ == "__main__":
    main(parse())
