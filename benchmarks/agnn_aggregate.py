#!/usr/bin/env python
"""AGNNConv's cosine-attention aggregation on one H100: the fused op (ops.agnn_attention_aggregate) against the same
aggregation composed from the mp ops (gather, multiply, beta *, sum, scatter_softmax, multiply, scatter_add), forward and
forward + backward.

    python benchmarks/agnn_aggregate.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Workload = the deepest block of the agnn example's 'full' dataflow: 2-hop GCNDataFlow [[0],[0]] WITH self loops (BaseGNNNet's
default, so the targets arrive unsorted), on the R-MAT graph of BASELINE configs[1] (10M nodes / 100M edges).  AGNN has no
`fc`, so its width is the raw feature width: D = 32 at batch 2048, and D = 128 at the largest batch of 2048, 1024, 512, 256
whose composition forward + backward fits the free device memory by an estimate from shapes (composition_peak_bytes),
computed before anything runs.  x_src, the normalized rows and the output gradient are seeded random tensors; beta = 1.

Before anything is timed a PARITY GATE checks, per D, the fused forward bit for bit against the composition fed the op's
own cos on the stably sorted edge list (the fused op on unsorted targets gives the sorted list's bits; the composition's
scatters take their atomic path on unsorted ones), and the fused gradients within 1e-4 of autograd through the composition
(grad_beta within 1e-4 of the magnitude of its terms du * cos); a mismatch aborts.  The arms then alternate in rounds in
one process.  metric = block edges per second of the fused forward at D = 32.  Also reported: ms per call, edges/s and the
device memory one call needs above its inputs per arm (torch's allocator peak plus the library's own scratch, measured in a
fresh process per arm), the per-kernel times of the fused op (eu_ctx_profile), and the card's name and power limit read in
the same run.  One JSON line on stdout; nothing is written to the tree."""
import argparse
import time

import harness
import numpy as np
from harness import block_edges


DIMS = (32, 128)
BATCHES_128 = (2048, 1024, 512, 256)
ARMS = ("fused_fwd", "composition_fwd", "fused_fwd_bwd", "composition_fwd_bwd")


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--memory-arm", default=None, help=argparse.SUPPRESS)    # D,batch,arm: one memory measurement (internal)
    p.add_argument("--choose-batch", type=int, default=None, help=argparse.SUPPRESS)   # D: batch_for (internal)
    return p.parse_args(argv)


def composition(ops, x, nd, ns, beta, dst, src, n_dst):
    u = (beta * (ops.gather(nd, dst) * ops.gather(ns, src))).sum(-1, keepdim=True)
    alpha = ops.scatter_softmax(u, dst, n_dst)
    return ops.scatter_add(ops.gather(x, src) * alpha, dst, n_dst)


def composition_peak_bytes(E, n_dst, n_src, D):
    """The composition's forward + backward at its peak, from shapes.  In the backward of x_j * alpha autograd holds 7
    [E, D] f32 tensors at once: gather(nrm_dst), gather(nrm_src), their product and x_j (saved by the forward), the
    messages' gradient, x_j's gradient and the product of the gradient with x_j (for alpha's).  One more is counted as
    margin for the allocator's rounding and the [E]-sized softmax tensors are added; then the three inputs, their gradients
    and the output and its gradient."""
    return 4 * (8 * E * D + 16 * E + 6 * n_src * D + 2 * n_dst * D)


def block_at(args, batch):
    return block_edges(argparse.Namespace(**dict(vars(args), batch=batch)), self_loops=True)


def batch_for(args, D):
    """D = 32: --batch.  D = 128: the largest of BATCHES_128 (<= --batch) whose composition_peak_bytes fits 90% of the
    free device memory once its block is built.  Returns the batch, the estimate and the free bytes it was held to."""
    import torch
    for b in ([args.batch] if D == 32 else [b for b in BATCHES_128 if b <= args.batch] or [args.batch]):
        dst, src, n_dst, n_src, _ = block_at(args, b)
        torch.cuda.synchronize()
        est = composition_peak_bytes(dst.numel(), n_dst, n_src, D)
        free = torch.cuda.mem_get_info()[0]
        del dst, src
        torch.cuda.empty_cache()
        if D == 32 or est <= 0.9 * free:
            return {"batch": b, "composition_peak_estimate_bytes": est, "free_bytes_at_choice": int(free)}
    raise SystemExit("no batch of %s fits the composition at D = %d" % (BATCHES_128, D))


def in_child(args, flag, value):
    """this script with `flag value` in a fresh process: its one JSON line"""
    return harness.in_fresh_process(__file__, [flag, value, "--nodes", str(args.nodes), "--edges", str(args.edges),
                                               "--batch", str(args.batch)])


def dim_inputs(n_dst, n_src, D):
    """seeded x_src, row-normalized nrm_dst and nrm_src, beta = 1 and the output gradient"""
    import torch
    rs = np.random.RandomState(D)

    def unit(n):
        x = rs.randn(n, D).astype(np.float32)
        return x / np.linalg.norm(x, axis=1, keepdims=True)

    t = [torch.from_numpy(a).cuda() for a in (rs.randn(n_src, D).astype(np.float32), unit(n_dst), unit(n_src),
                                              np.ones(1, np.float32), rs.randn(n_dst, D).astype(np.float32))]
    return tuple(t)


def make_arms(ops, x, nd, ns, beta, g, dst, src, n_dst, n_src):
    import torch
    edge_index = torch.stack([dst, src])

    def fused_fwd():
        with torch.no_grad():
            return ops.agnn_attention_aggregate(x, nd, ns, beta, edge_index, (n_dst, n_src))

    def comp_fwd():
        with torch.no_grad():
            return composition(ops, x, nd, ns, beta, dst, src, n_dst)

    def grads(fn):
        leaves = [t.clone().requires_grad_(True) for t in (x, nd, ns, beta)]
        out = fn(*leaves)
        out.backward(g)
        return [t.grad for t in leaves]

    def fused_fb():
        return grads(lambda a, b, c, d: ops.agnn_attention_aggregate(a, b, c, d, edge_index, (n_dst, n_src)))

    def comp_fb():
        return grads(lambda a, b, c, d: composition(ops, a, b, c, d, dst, src, n_dst))

    return dict(zip(ARMS, (fused_fwd, comp_fwd, fused_fb, comp_fb)))


def memory_of_arm(args, D, batch, arm):
    """In a process of its own: the device memory one call of `arm` needs above its inputs, as gat_aggregate.py
    measures it (torch's allocator peak + the device memory allocated outside it, i.e. the library's ctx scratch, on
    Contexts that have done nothing else; kernels and Contexts set up first by every arm on a tiny block)."""
    import gc
    import torch
    import euler_b200 as eb
    from euler_b200 import ops
    dst, src, n_dst, n_src, _ = block_at(args, batch)
    eb.set_graph(eb.get_graph())       # a fresh Context: the dataflow's (larger) scratch would hide the op's
    gc.collect()
    x, nd, ns, beta, g = dim_inputs(n_dst, n_src, D)
    tiny = make_arms(ops, x[:8], nd[:2], ns[:8], beta, g[:2], torch.tensor([1, 0], dtype=torch.int32, device="cuda"),
                     torch.tensor([3, 5], dtype=torch.int32, device="cuda"), 2, 8)
    for fn in tiny.values():
        fn()
    fn = make_arms(ops, x, nd, ns, beta, g, dst, src, n_dst, n_src)[arm]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    peak, scratch = harness.memory_of(fn)
    return {"torch_peak_bytes": peak, "op_scratch_bytes": scratch, "total_bytes": peak + scratch}


def gate(ops, arms, x, nd, ns, beta, g, dst, src, n_dst, D):
    """the parity gate of the module docstring; returns the largest relative gradient difference seen"""
    import torch
    out, alpha, cos = ops._raw_agnn(x, nd, ns, beta, dst, src, n_dst, True)
    order = torch.sort(dst, stable=True)[1]
    sd, ss = dst[order].contiguous(), src[order].contiguous()
    a = ops.scatter_softmax((beta * cos[order]).view(-1, 1), sd, n_dst)
    want = ops.scatter_add(ops.gather(x, ss) * a, sd, n_dst)
    if not (torch.equal(out.view(torch.int32), want.view(torch.int32)) and
            torch.equal(alpha[order].view(torch.int32), a.view(-1).view(torch.int32))):
        raise SystemExit("PARITY GATE FAILED: fused forward differs from the composition fed its cos at D = %d" % D)
    da = (ops.gather(g, dst) * ops.gather(x, src)).sum(-1)
    du = alpha * (da - ops.gather(ops.scatter_add((alpha * da).view(-1, 1), dst, n_dst), dst).view(-1))
    beta_terms = float((du * cos).abs().sum())
    del out, alpha, cos, order, sd, ss, a, want, da, du
    fg = arms["fused_fwd_bwd"]()
    cg = arms["composition_fwd_bwd"]()
    worst = 0.0
    for nm, p, q in zip(("grad_x_src", "grad_nrm_dst", "grad_nrm_src", "grad_beta"), fg, cg):
        floor = 1e-4 * (beta_terms if nm == "grad_beta" else float(q.abs().max()))
        diff = float((p - q).abs().max())
        if not torch.allclose(p, q, rtol=1e-4, atol=floor):
            raise SystemExit("PARITY GATE FAILED: fused %s differs from autograd through the composition at D = %d: max abs diff %g"
                             % (nm, D, diff))
        worst = max(worst, diff / max(floor / 1e-4, 1e-30))
    return worst


def run(args):
    import torch
    from euler_b200 import _lib, ops
    torch.cuda.set_device(0)
    lib = _lib.load()
    # the batches, then the memory per arm, each in a fresh process before this one holds any device memory
    choice = {D: in_child(args, "--choose-batch", str(D)) for D in DIMS}
    memory = {D: {k: in_child(args, "--memory-arm", "%d,%d,%s" % (D, choice[D]["batch"], k)) for k in ARMS} for D in DIMS}
    results = []
    for D in DIMS:
        t0 = time.time()
        batch = choice[D]["batch"]
        dst, src, n_dst, n_src, indeg = block_at(args, batch)
        E = dst.numel()
        torch.cuda.synchronize()
        t_setup = time.time() - t0
        block = {"batch": batch, "edges": E, "targets": n_dst, "sources": n_src, "max_edges_per_target": int(indeg.max()),
                 "sorted_targets": bool((dst[1:] >= dst[:-1]).all()) if E > 1 else True}
        x, nd, ns, beta, g = dim_inputs(n_dst, n_src, D)
        arms = make_arms(ops, x, nd, ns, beta, g, dst, src, n_dst, n_src)
        worst = gate(ops, arms, x, nd, ns, beta, g, dst, src, n_dst, D)

        rounds, per = harness.rounds_of(args.steps)
        ms = harness.time_arms(arms, rounds, args.warmup, per)
        arm_out = {k: {"ms_per_call": float(np.mean(v)), "edges_per_sec": E / (float(np.mean(v)) * 1e-3), "calls": rounds * per,
                       "memory": memory[D][k]} for k, v in ms.items()}
        # per-kernel times of the fused op, in a separate pass (the events bracket every kernel).  Autograd runs the backward
        # pass on its own thread, hence on another Context: both entry points are called here directly, on this thread's.
        torch.cuda.synchronize()
        ctx = ops._ctx_on_stream()
        gx, gnd, gns, gb = (torch.empty_like(t) for t in (x, nd, ns, beta))

        def fused_passes():
            for _ in range(3):
                _, alpha, cos = ops._raw_agnn(x, nd, ns, beta, dst, src, n_dst, True)
                _lib.check(lib.eu_agnn_aggregate_backward(ctx._h, g.data_ptr(), x.data_ptr(), nd.data_ptr(), ns.data_ptr(),
                                                          beta.data_ptr(), alpha.data_ptr(), cos.data_ptr(), dst.data_ptr(),
                                                          src.data_ptr(), E, n_dst, n_src, D, gx.data_ptr(), gnd.data_ptr(),
                                                          gns.data_ptr(), gb.data_ptr()))
        kern = harness.kernel_times(lib, ctx, "agnn_", fused_passes)
        del gx, gnd, gns, gb
        results.append({"dim": D, "block": block, "arms": arm_out, "kernels": kern, "setup_s": round(t_setup, 2),
                        "composition_peak_estimate_bytes": choice[D]["composition_peak_estimate_bytes"],
                        "free_bytes_at_choice": choice[D]["free_bytes_at_choice"],
                        "gate_worst_grad_diff_over_floor": worst,
                        "speedup_fwd": arm_out["composition_fwd"]["ms_per_call"] / arm_out["fused_fwd"]["ms_per_call"],
                        "speedup_fwd_bwd": arm_out["composition_fwd_bwd"]["ms_per_call"] / arm_out["fused_fwd_bwd"]["ms_per_call"]})
        del x, nd, ns, beta, g, arms, dst, src, indeg
        torch.cuda.empty_cache()
    head = results[0]["arms"]["fused_fwd"]
    out = {"metric": "agnn_block_edges_per_sec", "value": head["edges_per_sec"], "unit": "edges/s", "n_gpus": 1,
           "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "data": "synthetic",
           "config": {"workload": "deepest block of a 2-hop GCNDataFlow [[0],[0]] with self loops, R-MAT %dM nodes / %dM edges; "
                                  "AGNN attention aggregation at D = 32 (batch %d) and D = 128 (batch %d)"
                                  % (args.nodes // 10**6, args.edges // 10**6, results[0]["block"]["batch"],
                                     results[1]["block"]["batch"]),
                      "nodes": args.nodes, "edges": args.edges},
           "dims": results,
           "parity_gate": {"passed": True, "what": "per D: fused forward bit-exact vs the composition fed the op's cos on the "
                                                   "stably sorted edge list; fused gradients within 1e-4 (floor 1e-4 x largest; "
                                                   "grad_beta: 1e-4 x sum |du * cos|) of autograd through the composition"},
           "gpu": harness.gpu_info(0)}
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    a = parse()
    if a.memory_arm:
        D, batch, arm = a.memory_arm.split(",")
        harness.emit(memory_of_arm(a, int(D), int(batch), arm))
    elif a.choose_batch:
        harness.emit(batch_for(a, a.choose_batch))
    else:
        run(a)
