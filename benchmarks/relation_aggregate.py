#!/usr/bin/env python
"""RelationConv's typed mean aggregation on one H100: the fused op (ops.relation_mean_aggregate) against the literal
composition (convolution.relation_aggregate: gather, unique, one [D, F] matrix per edge, batched matvec, scatter_mean),
forward and forward + backward.

    python benchmarks/relation_aggregate.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Workload = the deepest block of the rgcn example's dataflow: a 2-hop RelationDataFlow over all 5 edge types of the
heterogeneous R-MAT graph of BASELINE configs[4] (Graph.rmat_hetero, 10M nodes / 100M edges, 3 node types, seed 44), batch
2048.  Two relation modes: rel = e_id (the listed edge type, R = 5; the keys arrive sorted) and a seeded per-edge relation in
[0, 18) as in wn18 (R = 18; the keys are unsorted, so the op sorts).  Two shapes (F, D) = (16, 32) (the example's
embedding_dim and hidden_dim) and (128, 128).  x_src, the matrices and the output gradient are seeded random tensors.

The composition materialises an [E, D, F] f32 matrix per call.  Its footprint is computed from the block's shape before
anything runs; where it does not fit 80 % of the free device memory the composition is skipped on the batch-2048 block and
both arms run on the largest smaller block (batch 1024, 512, ...) where it fits.

Before anything is timed a PARITY GATE checks, on every block timed: the fused forward within 1e-5 (floor 1e-5 x largest)
of a float64 restatement (x_src summed per (target, relation) in float64, then the matrices), the fused gradients within 1e-4
of the float64 gradients, and, where the composition runs, the fused forward within 1e-4 of it; a mismatch aborts.  The arms
alternate in rounds in one process.  metric = block edges per second of the fused forward at (16, 32), rel = e_id.  Also
reported per block: E, P (the distinct (target, relation) pairs), targets, the largest target, ms per call, per-kernel times
(eu_ctx_profile), the device memory one call needs above its inputs per arm (torch's allocator peak plus the library's
scratch, measured in a fresh process per arm), and the card's name and power limit read in the same run.  One JSON line on
stdout; nothing is written to the tree."""
import argparse
import time

import harness
import numpy as np

from bench import C5_ETYPES, C5_NTYPES, C5_SEED

SHAPES = [(16, 32), (128, 128)]
MODES = {"e_id": C5_ETYPES, "wn18": 18}
SMALLER = (1024, 512, 256, 128, 64)
FIT = 0.8          # the share of the free device memory the composition may take (a child process holds its own graph)
ARMS = ("fused_fwd", "composition_fwd", "fused_fwd_bwd", "composition_fwd_bwd")


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--memory-arm", default=None, help=argparse.SUPPRESS)    # mode,F,D,batch,arm: one measurement (internal)
    return p.parse_args(argv)


_GRAPH = {}


def block(args, batch, mode):
    """the deepest block at `batch`: (dst, src, rel) int32 on the device, n_dst, n_src, each target's edge count"""
    import torch
    import euler_b200 as eb
    from euler_b200.dataflow import RelationDataFlow
    if "g" not in _GRAPH:
        _GRAPH["g"] = eb.Graph.rmat_hetero(args.nodes, args.edges, C5_ETYPES, C5_NTYPES, seed=C5_SEED, device=0)
        eb.set_graph(_GRAPH["g"])
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=batch).astype(np.int64)).cuda()
    types = list(range(C5_ETYPES))
    blk = RelationDataFlow([10, 10], [types, types])(seeds)[0]
    ei = blk.edge_index.to(torch.int32)
    n_dst, n_src = blk.size
    dst, src = ei[0].contiguous(), ei[1].contiguous()
    if mode == "e_id":
        rel = blk.e_id.to(torch.int32).contiguous()
    else:
        rel = torch.from_numpy(np.random.RandomState(18).randint(0, 18, size=dst.numel()).astype(np.int32)).cuda()
    return dst, src, rel, n_dst, n_src, torch.bincount(dst.long(), minlength=n_dst)


def composition_bytes(E, F, D, bwd):
    """the composition's peak from shapes: the [E, D, F] matrices (and, with backward, their gradient), x_j and its gradient,
    the [E, D] messages and their gradient, plus one [E, D] margin"""
    return 4 * ((2 * E * D * F + 2 * E * F + 3 * E * D) if bwd else (E * D * F + E * F + 3 * E * D))


def shape_inputs(n_dst, n_src, R, F, D):
    import torch
    rs = np.random.RandomState(F * 1000 + D + R)
    return tuple(torch.from_numpy(a.astype(np.float32)).cuda() for a in
                 (rs.randn(n_src, F), rs.randn(R, D, F) / np.sqrt(F), rs.randn(n_dst, D)))


def make_arms(x, W, g, dst, src, rel, n_dst, n_src):
    import torch
    from euler_b200 import ops
    from euler_b200 import convolution as conv
    edge_index = torch.stack([dst, src])

    def fused(a, b):
        return ops.relation_mean_aggregate(a, b, rel, edge_index, (n_dst, n_src))

    def comp(a, b):
        return conv.relation_aggregate((None, a), edge_index, (n_dst, n_src), rel, b)

    def fwd(fn):
        def run():
            with torch.no_grad():
                return fn(x, W)
        return run

    def fb(fn):
        def run():
            leaves = [t.clone().requires_grad_(True) for t in (x, W)]
            fn(*leaves).backward(g)
            return [t.grad for t in leaves]
        return run

    return dict(zip(ARMS, (fwd(fused), fwd(comp), fb(fused), fb(comp))))


def reference64(x, W, g, dst, src, rel, n_dst, R):
    """float64 on the device: S[i, r] = sum of x_src rows per (target, relation), out = sum_r W[r] S[i, r] / (cnt + 1e-7); the
    gradients gm = g / (cnt + 1e-7), grad_x_src[j] = sum over j's edges of W[rel]^T gm[dst], grad_W[r] = sum_i gm[i] (x) S[i, r]"""
    import torch
    x64, W64, g64 = x.double(), W.double(), g.double()
    key = dst.long() * R + rel.long()
    S = torch.zeros((n_dst * R, x.shape[1]), dtype=torch.float64, device=x.device)
    step = 1 << 20
    for b in range(0, dst.numel(), step):
        S.index_add_(0, key[b:b + step], x64[src[b:b + step].long()])
    S = S.view(n_dst, R, -1)
    den = torch.bincount(dst.long(), minlength=n_dst).double()[:, None] + 1e-7
    out = torch.einsum("rdf,irf->id", W64, S) / den
    gm = g64 / den
    gS = torch.einsum("rdf,id->irf", W64, gm).reshape(n_dst * R, -1)
    gx = torch.zeros_like(x64)
    for b in range(0, dst.numel(), step):
        gx.index_add_(0, src[b:b + step].long(), gS[key[b:b + step]])
    gW = torch.einsum("id,irf->rdf", gm, S)
    return out, gx, gW


def within(a, b, rtol):
    floor = rtol * float(b.abs().max())
    return bool(((a.double() - b.double()).abs() <= floor + rtol * b.double().abs()).all()), float((a.double() - b.double()).abs().max())


def gate(arms, x, W, g, dst, src, rel, n_dst, R, with_comp, what):
    import torch
    out64, gx64, gW64 = reference64(x, W, g, dst, src, rel, n_dst, R)
    out = arms["fused_fwd"]()
    ok, d = within(out, out64, 1e-5)
    if not ok:
        raise SystemExit("PARITY GATE FAILED: fused forward vs float64 at %s: max abs diff %g" % (what, d))
    report = {"fwd_vs_float64_max_abs_diff": d}
    if with_comp:
        ok, d = within(out, arms["composition_fwd"](), 1e-4)
        if not ok:
            raise SystemExit("PARITY GATE FAILED: fused forward vs relation_aggregate at %s: max abs diff %g" % (what, d))
        report["fwd_vs_composition_max_abs_diff"] = d
    del out
    for nm, a, b in zip(("grad_x_src", "grad_matrix"), arms["fused_fwd_bwd"](), (gx64, gW64)):
        ok, d = within(a, b, 1e-4)
        if not ok:
            raise SystemExit("PARITY GATE FAILED: fused %s vs float64 at %s: max abs diff %g" % (nm, what, d))
        report[nm + "_vs_float64_max_abs_diff"] = d
    del out64, gx64, gW64
    torch.cuda.empty_cache()
    return report


def memory_of_arm(args, mode, F, D, batch, arm):
    """In a process of its own: the device memory one call of `arm` needs above its inputs, as gat_aggregate.py
    measures it (torch's allocator peak + the device memory allocated outside it, i.e. the library's ctx scratch, on Contexts
    that have done nothing else; the kernels and Contexts are set up first by every arm on a tiny block)."""
    import gc
    import torch
    import euler_b200 as eb
    R = MODES[mode]
    dst, src, rel, n_dst, n_src, _ = block(args, batch, mode)
    eb.set_graph(eb.get_graph())
    gc.collect()
    x, W, g = shape_inputs(n_dst, n_src, R, F, D)
    t = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    for fn in make_arms(x[:8], W, g[:2], t([1, 0]), t([3, 5]), t([0, R - 1]), 2, 8).values():
        fn()
    fn = make_arms(x, W, g, dst, src, rel, n_dst, n_src)[arm]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    peak, scratch = harness.memory_of(fn)
    return {"torch_peak_bytes": peak, "op_scratch_bytes": scratch, "total_bytes": peak + scratch}


def measure_memory(args, mode, F, D, batch, arm):
    return harness.in_fresh_process(__file__, ["--memory-arm", "%s,%d,%d,%d,%s" % (mode, F, D, batch, arm),
                                               "--nodes", str(args.nodes), "--edges", str(args.edges)])


def kernel_times(x, W, g, dst, src, rel, n_dst, n_src, R):
    """per-kernel times of the fused op in a separate pass (events bracket every kernel), both entry points called directly
    on this thread's Context (autograd would run the backward on another)"""
    import torch
    from euler_b200 import _lib, ops
    lib = _lib.load()
    torch.cuda.synchronize()
    ctx = ops._ctx_on_stream()
    gx, gW = torch.empty_like(x), torch.empty_like(W)
    F, D = x.shape[1], W.shape[1]

    def fused_passes():
        for _ in range(3):
            ops._raw_relation(x, W, rel, dst, src, n_dst)
            _lib.check(lib.eu_relation_aggregate_backward(ctx._h, g.data_ptr(), x.data_ptr(), W.data_ptr(), rel.data_ptr(),
                                                          dst.data_ptr(), src.data_ptr(), dst.numel(), n_dst, n_src, R, D, F,
                                                          gx.data_ptr(), gW.data_ptr()))
    return harness.kernel_times(lib, ctx, "rel_", fused_passes)


def run_block(args, mode, F, D, batch, with_comp, memory):
    import torch
    R = MODES[mode]
    dst, src, rel, n_dst, n_src, indeg = block(args, batch, mode)
    E = dst.numel()
    key = dst.long() * R + rel.long()
    info = {"batch": batch, "edges": E, "pairs": int(torch.unique(key).numel()), "targets": n_dst, "sources": n_src,
            "relations": R, "max_edges_per_target": int(indeg.max()), "sorted_keys": bool((key[1:] >= key[:-1]).all()),
            "composition_fwd_estimate_bytes": composition_bytes(E, F, D, False),
            "composition_fwd_bwd_estimate_bytes": composition_bytes(E, F, D, True)}
    del key
    x, W, g = shape_inputs(n_dst, n_src, R, F, D)
    arms = make_arms(x, W, g, dst, src, rel, n_dst, n_src)
    what = "%s (F, D) = (%d, %d) batch %d" % (mode, F, D, batch)
    info["gate"] = gate(arms, x, W, g, dst, src, rel, n_dst, R, with_comp, what)
    names = list(ARMS) if with_comp else ["fused_fwd", "fused_fwd_bwd"]
    rounds, per = harness.rounds_of(args.steps)
    ms = {k: float(np.mean(v)) for k, v in harness.time_arms({k: arms[k] for k in names}, rounds, args.warmup, per).items()}
    info["arms"] = {k: {"ms_per_call": ms[k], "edges_per_sec": E / (ms[k] * 1e-3),
                        "memory": memory.get((mode, F, D, batch, k))} for k in names}
    info["kernels"] = kernel_times(x, W, g, dst, src, rel, n_dst, n_src, R)
    del x, W, g, arms, dst, src, rel, indeg
    torch.cuda.empty_cache()
    return info


def plan(args):
    """per (mode, shape): whether the composition fits at --batch, else the batch where it does (fwd + bwd estimate)"""
    import torch
    out = {}
    sizes = {}
    for b in (args.batch,) + tuple(s for s in SMALLER if s < args.batch):
        dst = block(args, b, "e_id")[0]          # the block's edges do not depend on the relation mode
        sizes[b] = dst.numel()
        del dst
        torch.cuda.empty_cache()
        if composition_bytes(sizes[b], *SHAPES[-1], True) <= FIT * torch.cuda.mem_get_info()[0]:
            break
    free = torch.cuda.mem_get_info()[0]
    for mode in MODES:
        for F, D in SHAPES:
            fits = [b for b in sizes if composition_bytes(sizes[b], F, D, True) <= FIT * free]
            out[(mode, F, D)] = {"main": args.batch, "composition_at": max(fits) if fits else None}
    return out, free


def run(args):
    import torch
    torch.cuda.set_device(0)
    t0 = time.time()
    todo, free = plan(args)
    t_plan = time.time() - t0
    memory = {}
    for (mode, F, D), p in todo.items():
        for arm in ("fused_fwd", "fused_fwd_bwd"):
            memory[(mode, F, D, p["main"], arm)] = measure_memory(args, mode, F, D, p["main"], arm)
        if p["composition_at"] is not None and (mode == "e_id" or p["composition_at"] == p["main"]):
            for arm in ARMS:     # on a smaller block, for rel = e_id only (the composition's memory does not depend on the mode)
                key = (mode, F, D, p["composition_at"], arm)
                if key not in memory:
                    memory[key] = measure_memory(args, mode, F, D, p["composition_at"], arm)
    results = []
    for (mode, F, D), p in todo.items():
        blocks = [run_block(args, mode, F, D, p["main"], p["composition_at"] == p["main"], memory)]
        if p["composition_at"] is not None and p["composition_at"] != p["main"]:
            blocks.append(run_block(args, mode, F, D, p["composition_at"], True, memory))
        r = {"mode": mode, "fea_dim": F, "dim": D, "blocks": blocks}
        if p["composition_at"] != p["main"]:
            r["composition_skipped_at_batch_%d" % p["main"]] = (
                "the composition's estimated forward + backward footprint, %.1f GB, exceeds %d%% of the %.1f GB free"
                % (blocks[0]["composition_fwd_bwd_estimate_bytes"] / 1e9, round(FIT * 100), free / 1e9))
        for b in blocks:
            if "composition_fwd" in b["arms"]:
                b["speedup_fwd"] = b["arms"]["composition_fwd"]["ms_per_call"] / b["arms"]["fused_fwd"]["ms_per_call"]
                b["speedup_fwd_bwd"] = b["arms"]["composition_fwd_bwd"]["ms_per_call"] / b["arms"]["fused_fwd_bwd"]["ms_per_call"]
        results.append(r)
    head = results[0]["blocks"][0]["arms"]["fused_fwd"]
    out = {"metric": "relation_block_edges_per_sec", "value": head["edges_per_sec"], "unit": "edges/s", "n_gpus": 1,
           "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "data": "synthetic",
           "config": {"workload": "deepest block of a 2-hop RelationDataFlow over all %d edge types, batch=%d, heterogeneous R-MAT "
                                  "%dM nodes / %dM edges; RelationConv mean aggregation at (F, D) = %s, rel = e_id and wn18-like"
                                  % (C5_ETYPES, args.batch, args.nodes // 10**6, args.edges // 10**6, SHAPES),
                      "nodes": args.nodes, "edges": args.edges, "batch": args.batch},
           "results": results,
           "parity_gate": {"passed": True, "what": "per block timed: fused forward within 1e-5 (floor 1e-5 x largest) of float64, "
                                                   "within 1e-4 of relation_aggregate where it runs; fused gradients within 1e-4 "
                                                   "of float64"},
           "gpu": harness.gpu_info(0), "plan_s": round(t_plan, 2)}
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    a = parse()
    if a.memory_arm:
        mode, F, D, batch, arm = a.memory_arm.split(",")
        harness.emit(memory_of_arm(a, mode, int(F), int(D), int(batch), arm))
    else:
        run(a)
