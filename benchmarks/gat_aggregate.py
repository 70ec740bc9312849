#!/usr/bin/env python
"""GATConv's attention aggregation on one H100: the fused op (ops.gat_attention_aggregate) against the same aggregation
composed from the mp ops (gather, leaky_relu, scatter_softmax, multiply, scatter_add), forward and forward + backward.

    python benchmarks/gat_aggregate.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Workload = the deepest block of the gat example's 'full' dataflow: 2-hop GCNDataFlow [[0],[0]] without self loops
(examples/gat/gat.py runs GATConv with add_self_loops=False), batch 2048, on the R-MAT graph of BASELINE configs[1] (10M nodes /
100M edges).  That block has 12.6M edges into 14.7K targets from 2.05M sources.  h_src and the scores are seeded random
tensors; (H, C) = (1, 32), the example's default, and (8, 8).

Before anything is timed a PARITY GATE checks, per (H, C), the fused forward bit for bit against the composition and the
fused gradients within 1e-4 of autograd through the composition; a mismatch aborts.  The arms then alternate in rounds in
one process.  metric = block edges per second of the fused forward at (1, 32).  Also reported: ms per call, edges/s and
the device memory one call needs above its inputs per arm (torch's allocator peak plus the library's own scratch, measured
in a fresh process per arm), the per-kernel times of the fused op (eu_ctx_profile), both
forward arms on the same block without its largest target (what that one target costs), and the card's name and power
limit read in the same run.  One JSON line on stdout; nothing is written to the tree."""
import argparse
import time

import harness
import numpy as np

from harness import block_edges

SHAPES = [(1, 32), (8, 8)]


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--memory-arm", default=None, help=argparse.SUPPRESS)    # H,C,arm: one memory measurement (internal)
    return p.parse_args(argv)


def composition(ops, F, h, sd, ss, dst, src, n_dst):
    E, H = dst.numel(), sd.shape[1]
    Cd = h.shape[1] // H
    u = F.leaky_relu(ops.gather(sd, dst) + ops.gather(ss, src), 0.2)
    alpha = ops.scatter_softmax(u, dst, n_dst)
    return ops.scatter_add((ops.gather(h, src).view(E, H, Cd) * alpha.view(E, H, 1)).view(E, H * Cd), dst, n_dst)


ARMS = ("fused_fwd", "composition_fwd", "fused_fwd_bwd", "composition_fwd_bwd")


def shape_inputs(n_dst, n_src, H, Cd):
    """seeded h_src, s_dst, s_src and the output gradient"""
    import torch
    rs = np.random.RandomState(H * 1000 + Cd)
    return tuple(torch.from_numpy(rs.randn(*shape).astype(np.float32)).cuda()
                 for shape in ((n_src, H * Cd), (n_dst, H), (n_src, H), (n_dst, H * Cd)))


def make_arms(ops, F, h, sd, ss, g, dst, src, n_dst, n_src):
    import torch
    edge_index = torch.stack([dst, src])

    def fused_fwd():
        with torch.no_grad():
            return ops.gat_attention_aggregate(h, sd, ss, edge_index, (n_dst, n_src))

    def comp_fwd():
        with torch.no_grad():
            return composition(ops, F, h, sd, ss, dst, src, n_dst)

    def grads(fn):
        leaves = [x.clone().requires_grad_(True) for x in (h, sd, ss)]
        out = fn(*leaves)
        out.backward(g)
        return [x.grad for x in leaves]

    def fused_fb():
        return grads(lambda a, b, c: ops.gat_attention_aggregate(a, b, c, edge_index, (n_dst, n_src)))

    def comp_fb():
        return grads(lambda a, b, c: composition(ops, F, a, b, c, dst, src, n_dst))

    return dict(zip(ARMS, (fused_fwd, comp_fwd, fused_fb, comp_fb)))


def memory_of_arm(args, hc, arm):
    """In a process of its own: the device memory one call of `arm` needs above its inputs.  torch_peak = the torch caching
    allocator's peak (torch.cuda.max_memory_allocated); op_scratch = device memory allocated outside torch's allocator, which is
    where the library's ctx scratch lives (cudaMalloc), on every Context the call uses (autograd runs the backward pass on
    its own thread, with its own Context).  The calls run on Contexts that have done nothing else: in a training step the
    Context has usually grown its scratch for the dataflow already, and the op reuses it.  The kernels and both Contexts are
    set up first by one call of every arm on a tiny block, so neither module loading nor a Context's fixed state is counted."""
    import torch
    import torch.nn.functional as F
    from euler_b200 import ops
    import gc
    import euler_b200 as eb
    H, Cd = hc
    dst, src, n_dst, n_src, _ = block_edges(args)
    eb.set_graph(eb.get_graph())       # a fresh Context: the dataflow's (larger) scratch would hide the op's
    gc.collect()
    h, sd, ss, g = shape_inputs(n_dst, n_src, H, Cd)
    tiny = make_arms(ops, F, h[:8], sd[:2], ss[:8], g[:2], torch.tensor([0, 1], dtype=torch.int32, device="cuda"),
                     torch.tensor([3, 5], dtype=torch.int32, device="cuda"), 2, 8)
    for fn in tiny.values():
        fn()
    fn = make_arms(ops, F, h, sd, ss, g, dst, src, n_dst, n_src)[arm]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    peak, scratch = harness.memory_of(fn)
    return {"torch_peak_bytes": peak, "op_scratch_bytes": scratch, "total_bytes": peak + scratch}


def measure_memory(args, hc, arm):
    """memory_of_arm in a fresh process (scratch only grows, so each arm needs its own)"""
    return harness.in_fresh_process(__file__, ["--memory-arm", "%d,%d,%s" % (hc[0], hc[1], arm), "--nodes", str(args.nodes),
                                               "--edges", str(args.edges), "--batch", str(args.batch)])


def run(args):
    import torch
    import torch.nn.functional as F
    from euler_b200 import _lib, ops
    torch.cuda.set_device(0)
    memory = {"%d,%d" % hc: {arm: measure_memory(args, hc, arm) for arm in ARMS} for hc in SHAPES}
    t0 = time.time()
    dst, src, n_dst, n_src, indeg = block_edges(args)
    E = dst.numel()
    torch.cuda.synchronize()
    t_setup = time.time() - t0
    block = {"edges": E, "targets": n_dst, "sources": n_src, "max_edges_per_target": int(indeg.max()),
             "sorted_targets": bool((dst[1:] >= dst[:-1]).all()) if E > 1 else True}
    lib = _lib.load()
    results = []
    for H, Cd in SHAPES:
        h, sd, ss, g = shape_inputs(n_dst, n_src, H, Cd)
        arms = make_arms(ops, F, h, sd, ss, g, dst, src, n_dst, n_src)
        fused_fwd, comp_fwd, fused_fb, comp_fb = (arms[k] for k in ARMS)

        # gate
        a, b = fused_fwd(), comp_fwd()
        if not torch.equal(a.view(torch.int32), b.view(torch.int32)):
            raise SystemExit("PARITY GATE FAILED: fused forward differs from the composition at (H, C) = (%d, %d)" % (H, Cd))
        del a, b
        fg, cg = fused_fb(), comp_fb()
        for nm, x, y in zip(("grad_h_src", "grad_s_dst", "grad_s_src"), fg, cg):
            floor = 1e-4 * float(y.abs().max())
            if not torch.allclose(x, y, rtol=1e-4, atol=floor):
                raise SystemExit("PARITY GATE FAILED: fused %s differs from autograd through the composition at (H, C) = (%d, %d): "
                                 "max abs diff %g" % (nm, H, Cd, float((x - y).abs().max())))
        del fg, cg

        rounds, per = harness.rounds_of(args.steps)
        ms = harness.time_arms(arms, rounds, args.warmup, per)
        arm_out = {k: {"ms_per_call": float(np.mean(v)), "edges_per_sec": E / (float(np.mean(v)) * 1e-3), "calls": rounds * per,
                       "memory": memory["%d,%d" % (H, Cd)][k]} for k, v in ms.items()}
        # per-kernel times of the fused op, in a separate pass (the events bracket every kernel).  Autograd runs the backward
        # pass on its own thread, hence on another Context: both entry points are called here directly, on this thread's.
        torch.cuda.synchronize()
        ctx = ops._ctx_on_stream()
        gh, gsd, gss = torch.empty_like(h), torch.empty_like(sd), torch.empty_like(ss)

        def fused_passes():
            for _ in range(3):
                _, alpha = ops._raw_gat(h, sd, ss, dst, src, n_dst, True)
                _lib.check(lib.eu_gat_aggregate_backward(ctx._h, g.data_ptr(), h.data_ptr(), alpha.data_ptr(), sd.data_ptr(),
                                                         ss.data_ptr(), dst.data_ptr(), src.data_ptr(), E, n_dst, n_src, H, Cd,
                                                         gh.data_ptr(), gsd.data_ptr(), gss.data_ptr()))
        kern = harness.kernel_times(lib, ctx, "gat_", fused_passes)
        del gh, gsd, gss
        # what the largest target costs: it stays on one lane group (its sums run in edge order), so it sets the kernel's
        # critical path; the same block without that target's edges, forward only
        keep = dst != int(indeg.argmax())
        kd, ks = dst[keep].contiguous(), src[keep].contiguous()
        kei = torch.stack([kd, ks])
        no_hub = {}
        for k, fn in (("fused_fwd", lambda: ops.gat_attention_aggregate(h, sd, ss, kei, (n_dst, n_src))),
                      ("composition_fwd", lambda: composition(ops, F, h, sd, ss, kd, ks, n_dst))):
            with torch.no_grad():
                ms = harness.time_arms({k: fn}, 1, args.warmup, args.steps)[k][0]
            no_hub[k] = {"ms_per_call": ms, "edges": kd.numel()}
        del kd, ks, kei, keep
        results.append({"heads": H, "head_dim": Cd, "arms": arm_out, "kernels": kern, "without_largest_target": no_hub,
                        "speedup_fwd": arm_out["composition_fwd"]["ms_per_call"] / arm_out["fused_fwd"]["ms_per_call"],
                        "speedup_fwd_bwd": arm_out["composition_fwd_bwd"]["ms_per_call"] / arm_out["fused_fwd_bwd"]["ms_per_call"]})
        del h, sd, ss, g, arms, fused_fwd, comp_fwd, fused_fb, comp_fb
        torch.cuda.empty_cache()
    head = results[0]["arms"]["fused_fwd"]
    out = {"metric": "gat_block_edges_per_sec", "value": head["edges_per_sec"], "unit": "edges/s", "n_gpus": 1,
           "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "data": "synthetic",
           "config": {"workload": "deepest block of a 2-hop GCNDataFlow [[0],[0]] without self loops, batch=%d, R-MAT %dM nodes / "
                                  "%dM edges; GAT attention aggregation at (H, C) = %s" % (args.batch, args.nodes // 10**6,
                                                                                         args.edges // 10**6, SHAPES),
                      "nodes": args.nodes, "edges": args.edges, "batch": args.batch},
           "block": block, "shapes": results,
           "parity_gate": {"passed": True, "what": "per (H, C): fused forward bit-exact vs the composition; fused gradients within "
                                                   "1e-4 (floor 1e-4 x largest) of autograd through the composition"},
           "gpu": harness.gpu_info(0), "setup_s": round(t_setup, 2)}
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    a = parse()
    if a.memory_arm:
        H, Cd, arm = a.memory_arm.split(",")
        harness.emit(memory_of_arm(a, (int(H), int(Cd)), arm))
    else:
        run(a)
