#!/usr/bin/env python
"""The unsupervised skip-gram step on one H100: the fused op (ops.skipgram_xent_loss) against the torch composition a user
writes today (unsupervised.composed_skipgram_loss: three embedding lookups, matmul, BCE with logits and a sort-based rank).

    python benchmarks/skipgram_loss.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E] [--dims 32,128]

Ids: BASELINE's C3 walk on its R-MAT (10M nodes / 100M edges): node2vec p = 0.5, q = 2, walk_len 80 from 4096 walkers,
gen_pair with windows 1 / 1 (160 pairs per walk, 655 360 pairs), and K = 5 negatives per pair from sample_node; drawn once.
Tables f32[n + 2, dim] (ShallowEncoder's rows), dim 32 and 128.  Arms, alternating round by round in one process after a
GATE against float64 over the touched rows (the fused loss within 1e-6, its dense gradients within 1e-5 of the largest
entry, the metric within 1e-4 of the composition's; the composition's own error is reported beside):
  fwd           the loss and mrr (no gradient)
  fwd_bwd       forward + backward, dense table gradients (nn.Embedding's default)
  fwd_bwd_sparse  forward + backward, sparse COO gradients (nn.Embedding(sparse=True) for the composition)
Memory, per arm in a fresh process on the same ids: torch's allocator peak above the inputs, plus the device memory the
library's ctx scratch took (the growth of the device's used memory outside torch's reserve).  Then one whole DeepWalk step
(walk -> pairs -> negatives -> loss -> backward -> SGD) is timed fused and composed.  The card's name, power limit and SM
clock are read in the same run.  One JSON line on stdout."""
import argparse
import os
import shutil
import tempfile
import time

import harness
from bench import GRAPH_SEED

ARMS = ("fwd", "fwd_bwd", "fwd_bwd_sparse")


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=4096)
    p.add_argument("--walk-len", type=int, default=80)
    p.add_argument("--negs", type=int, default=5)
    p.add_argument("--dims", default="32,128")
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--mem-arm", default=None, help=argparse.SUPPRESS)   # internal: one arm's memory, in a fresh process
    p.add_argument("--ids", default=None, help=argparse.SUPPRESS)
    return p.parse_args(argv)


def tables(n_rows, dim, requires_grad):
    import torch
    g = torch.Generator(device="cuda").manual_seed(dim)
    t = (torch.randn(n_rows, dim, device="cuda", generator=g) * 0.1).requires_grad_(requires_grad)
    c = (torch.randn(n_rows, dim, device="cuda", generator=g) * 0.1).requires_grad_(requires_grad)
    return t, c


def run_arm(kind, arm, ids, t, c):
    """one call of an arm: (loss, metric); the gradients land in t.grad / c.grad"""
    import torch
    import torch.nn.functional as F
    import euler_b200 as eb
    from euler_b200.unsupervised import composed_skipgram_loss
    src, pos, negs = ids
    sparse = arm == "fwd_bwd_sparse"
    with torch.set_grad_enabled(arm != "fwd"):
        if kind == "fused":
            loss, m = eb.skipgram_xent_loss(src, pos, negs, t, c, metric="mrr", sparse_grad=sparse)
        else:
            loss, m = composed_skipgram_loss(F.embedding(src, t, sparse=sparse), F.embedding(pos, c, sparse=sparse),
                                             F.embedding(negs, c, sparse=sparse), "mrr")
        if arm != "fwd":
            t.grad = c.grad = None
            loss.backward()
    return loss, m


def float64_step(ids, t, c):
    """(loss, (grad_target, grad_context, rows)) of the composition in float64 over the rows the ids touch"""
    import torch
    import torch.nn.functional as F
    from euler_b200.unsupervised import composed_skipgram_loss
    flat = torch.cat([x.reshape(-1) for x in ids])
    rows, inv = torch.unique(flat, return_inverse=True)
    sizes = [x.numel() for x in ids]
    s_, p_, n_ = (v.reshape(x.shape) for v, x in zip(torch.split(inv, sizes), ids))
    T = t.detach()[rows].double().requires_grad_(True)
    Cx = c.detach()[rows].double().requires_grad_(True)
    loss, _ = composed_skipgram_loss(F.embedding(s_, T), F.embedding(p_, Cx), F.embedding(n_, Cx), "mrr")
    loss.backward()
    return float(loss.detach()), (T.grad, Cx.grad, rows)


def mem_arm(args):
    """torch's peak and the library's scratch growth of one arm, in this fresh process"""
    import torch
    import euler_b200 as eb
    kind, arm, dim = args.mem_arm.split(":")
    saved = torch.load(args.ids)
    ids = tuple(x.cuda() for x in saved["ids"])
    eb.set_graph(eb.Graph.rmat(1000, 5000, seed=1), rng="minstd", seed=1)   # a ctx; the ids index the tables only
    t, c = tables(saved["n_rows"], int(dim), arm != "fwd")
    peak, outside = harness.memory_of(lambda: run_arm(kind, arm, ids, t, c))
    harness.emit({"torch_peak_bytes": peak, "ctx_scratch_bytes": max(outside, 0)})


def main(args):
    import numpy as np
    import torch
    import euler_b200 as eb
    from euler_b200 import unsupervised as un
    g = eb.Graph.rmat(args.nodes, args.edges, seed=GRAPH_SEED)
    eb.set_graph(g, rng="philox", seed=7)
    n_rows = args.nodes + 2
    starts = torch.as_tensor(np.random.RandomState(3).randint(1, args.nodes + 1, size=args.batch), dtype=torch.int64).cuda()
    path = eb.random_walk(starts, [[0]] * args.walk_len, p=0.5, q=2.0, default_node=args.nodes + 1)
    pair = eb.gen_pair(path, 1, 1)
    n = pair.shape[0] * pair.shape[1]
    ids = (pair[:, :, 0].reshape(n, 1).contiguous(), pair[:, :, 1].reshape(n, 1).contiguous(),
           eb.sample_node(n * args.negs, 0).reshape(n, args.negs))
    out = {"what": "skip-gram step (loss + mrr), fused eu_skipgram_loss vs torch composition", "gpu": harness.gpu_info(0),
           "pairs": n, "K": args.negs, "nodes": args.nodes, "rows_touched": int(torch.unique(torch.cat([x.reshape(-1) for x in ids])).numel()),
           "results": {}}
    tmp = tempfile.mkdtemp(prefix="skipgram_bench_")
    ids_path = os.path.join(tmp, "ids.pt")
    torch.save({"ids": [x.cpu() for x in ids], "n_rows": n_rows}, ids_path)
    for dim in (int(d) for d in args.dims.split(",")):
        t, c = tables(n_rows, dim, True)
        # GATE: the fused and the composed loss and gradients against float64 over the rows the batch touches
        lf, mf = run_arm("fused", "fwd_bwd", ids, t, c)
        gtf, gcf = t.grad.clone(), c.grad.clone()
        lc, mc = run_arm("composed", "fwd_bwd", ids, t, c)
        l64, g64 = float64_step(ids, t, c)
        gate = {"loss_f64": l64, "loss_fused": float(lf), "loss_composed": float(lc), "mrr_fused": float(mf), "mrr_composed": float(mc)}
        for name, (gf, gc_, w) in (("target", (gtf, t.grad, g64[0])), ("context", (gcf, c.grad, g64[1]))):
            scale = float(w.abs().max())
            gate["grad_%s_fused_err" % name] = float((gf[g64[2]].double() - w).abs().max()) / scale
            gate["grad_%s_composed_err" % name] = float((gc_[g64[2]].double() - w).abs().max()) / scale
            assert gate["grad_%s_fused_err" % name] <= 1e-5, ("gradient gate", dim, gate)
        assert abs(float(lf) - l64) <= 1e-6 * l64, ("loss gate", dim, gate)
        assert abs(float(mf) - float(mc)) <= 1e-4, ("metric gate", dim, gate)
        del gtf, gcf
        ms = harness.time_arms({(k, a): (lambda k=k, a=a: run_arm(k, a, ids, t, c)) for k in ("fused", "composed") for a in ARMS},
                               args.steps, args.warmup)
        t.grad = c.grad = None
        del t, c
        torch.cuda.empty_cache()
        res = {}
        for (k, a), v in ms.items():
            try:
                m = harness.in_fresh_process(__file__, ["--mem-arm", "%s:%s:%d" % (k, a, dim), "--ids", ids_path])
            except SystemExit as e:
                m = {"error": str(e)[-500:]}
            res["%s_%s" % (k, a)] = {"ms_median": float(np.median(v)), "ms_min": float(np.min(v)), "ms_max": float(np.max(v)), **m}
        for a in ARMS:
            res["speedup_" + a] = res["composed_" + a]["ms_median"] / res["fused_" + a]["ms_median"]
        res["gate"] = gate
        out["results"]["dim%d" % dim] = res
    # one whole DeepWalk step: walk -> pairs -> negatives -> loss -> backward -> SGD, fused and composed
    step = {}
    for fused in (True, False):
        torch.manual_seed(0)
        model = un.DeepWalk(0, [0], args.nodes, 128, walk_len=args.walk_len, walk_p=0.5, walk_q=2.0, num_negs=args.negs,
                            fused=fused, device="cuda")
        times = []
        for r in range(args.warmup + 3):
            torch.cuda.synchronize()
            h0 = time.perf_counter()
            _, loss, _, _ = model(starts)
            model.zero_grad()
            loss.backward()
            with torch.no_grad():
                for p in model.parameters():
                    p.add_(p.grad, alpha=-0.01)
            torch.cuda.synchronize()
            if r >= args.warmup:
                times.append((time.perf_counter() - h0) * 1e3)
        step["fused" if fused else "composed"] = {"ms_median": float(np.median(times)), "ms_all": times}
        del model
        torch.cuda.empty_cache()
    out["deepwalk_step_dim128"] = step
    shutil.rmtree(tmp, ignore_errors=True)
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    a = parse()
    if a.mem_arm:
        mem_arm(a)
    else:
        main(a)
