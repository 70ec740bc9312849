#!/usr/bin/env python
"""DNAConv's attention aggregation on one H100: the fused path (convolution.dna_aggregate: group_dense once per node, gcn_norm,
ops.dna_attention_aggregate) against a literal per-edge restatement of dna_conv.py over the mp ops (gather both sides,
lin_q / lin_k / lin_v on the E gathered rows, the reshapes and transposes of multi_head, restricted_softmax, the second
matmul, the norm product, scatter_mean), forward and forward + backward.  Both arms start from the in_fc outputs.

    python benchmarks/dna_aggregate.py [--steps K] [--warmup W] [--batch B] [--nodes N --edges E]

Workload = the deepest block of the dna example's 'full' dataflow: 2-hop GCNDataFlow [[0],[0]] WITH self loops (so the
targets arrive unsorted), on the R-MAT graph of BASELINE configs[1] (10M nodes / 100M edges), at (dim, heads) = (32, 1),
(128, 1) and (128, 4), groups = 8 ((32, 1) is the example's default).  The fused arms run at --batch.  The composition runs at
the largest batch of 2048, 1024, 512, 256 (<= --batch) whose forward + backward fits 90% of the free device memory by an
estimate from shapes (composition_peak_bytes), and the fused arms are timed at that batch as well for the comparison; if no
batch fits, the composition is reported as "not run" with its estimate.  Inputs are seeded random tensors.

Before anything is timed a PARITY GATE checks, per configuration and at the comparison batch, the fused forward within 1e-4
of the composition (floor 1e-4 x the largest magnitude) and the fused gradients of the in_fc outputs and the GroupDense
kernels and biases within 1e-3 of autograd through the composition; a mismatch aborts.  The arms then alternate in rounds in
one process.  metric = block edges per second of the fused forward at (32, 1) at --batch.  Also reported: ms per call,
edges/s and the device memory one call needs above its inputs per arm (torch's allocator peak plus the library's own
scratch, measured in a fresh process per arm), the per-kernel times of the fused op (eu_ctx_profile), and the card's name,
power limit and SM clock read in the same run.  One JSON line on stdout; nothing is written to the tree."""
import argparse
import time

import harness
import numpy as np
from harness import block_edges


CONFIGS = ((32, 1), (128, 1), (128, 4))
GROUPS = 8
BATCHES = (2048, 1024, 512, 256)
ARMS = ("fused_fwd", "composition_fwd", "fused_fwd_bwd", "composition_fwd_bwd")


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--batch", type=int, default=2048)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--memory-arm", default=None, help=argparse.SUPPRESS)    # dim,heads,batch,arm: one measurement (internal)
    p.add_argument("--choose-batch", default=None, help=argparse.SUPPRESS)  # dim,heads: batch_for (internal)
    return p.parse_args(argv)


def composition(ops, conv, xt, xs, lins, dst, src, n_dst, n_src, H):
    """dna_conv.py:149-170 literally over the mp ops, from the in_fc outputs"""
    import torch
    dim = xt.shape[1]
    c = dim // H
    n0, n1 = conv.gcn_norm(torch.stack([dst, src]), (n_dst, n_src))
    x_i, x_j = ops.gather(xt, dst), ops.gather(xs, src)
    q, k, v = (conv.group_dense(x, *p) for x, p in ((x_i, lins[0]), (x_j, lins[1]), (x_j, lins[2])))
    q, k, v = (t.reshape(-1, 1, H, c).permute(1, 0, 2, 3) for t in (q, k, v))
    score = torch.matmul(q, k.permute(0, 1, 3, 2)) / torch.sqrt(torch.tensor(float(c), device=xt.device))
    m = score.max(dim=-1, keepdim=True).values[0].clamp(0, torch.finfo(torch.float32).max)
    score = torch.exp(score - m)
    score = score / (score.sum(-1, keepdim=True) + torch.exp(0 - m))
    out = torch.matmul(score, v).permute(1, 0, 2, 3).reshape(-1, q.shape[1], dim).squeeze(0)
    return ops.scatter_mean(ops.gather(n0, dst) * ops.gather(n1, src) * out, dst, n_dst)


def composition_peak_bytes(E, n_dst, n_src, dim, H):
    """The composition's forward + backward at its peak, from shapes: about 18 [E, dim] f32 tensors (the two gathers, the
    three per-edge GroupDense outputs and their group-major copies, the attention output and its transposed copy, the
    messages, and their gradients in the backward pass, plus margin for the allocator), 8 [E, H, H] score tensors and 6
    [E]-sized ones; then the inputs, their gradients and the output."""
    return 4 * (18 * E * dim + 8 * E * H * H + 6 * E + 4 * (n_dst + n_src) * dim)


def block_at(args, batch):
    return block_edges(argparse.Namespace(**dict(vars(args), batch=batch)), self_loops=True)


def batch_for(args, dim, H):
    """the largest of BATCHES (<= --batch) whose composition_peak_bytes fits 90% of the free device memory once its block
    is built; None when none does"""
    import torch
    est = None
    for b in [b for b in BATCHES if b <= args.batch] or [args.batch]:
        dst, src, n_dst, n_src, _ = block_at(args, b)
        torch.cuda.synchronize()
        est = composition_peak_bytes(dst.numel(), n_dst, n_src, dim, H)
        free = torch.cuda.mem_get_info()[0]
        del dst, src
        torch.cuda.empty_cache()
        if est <= 0.9 * free:
            return {"batch": b, "composition_peak_estimate_bytes": est, "free_bytes_at_choice": int(free)}
    return {"batch": None, "composition_peak_estimate_bytes": est, "free_bytes_at_choice": int(free)}


def in_child(args, flag, value):
    """this script with `flag value` in a fresh process: its one JSON line"""
    return harness.in_fresh_process(__file__, [flag, value, "--nodes", str(args.nodes), "--edges", str(args.edges),
                                               "--batch", str(args.batch)])


def inputs(n_dst, n_src, dim, H):
    """seeded in_fc outputs of both sides, GroupDense (kernel, bias) for lin_q, lin_k, lin_v, and the output gradient"""
    import torch
    rs = np.random.RandomState(dim + H)

    def t(*shape, scale=1.0):
        return torch.from_numpy((rs.randn(*shape) * scale).astype(np.float32)).cuda()

    lins = [(t(GROUPS, dim // GROUPS, dim // GROUPS, scale=(GROUPS / dim) ** 0.5), t(dim, scale=0.1)) for _ in range(3)]
    return t(n_dst, dim), t(n_src, dim), lins, t(n_dst, dim)


def make_arms(ops, conv, xt, xs, lins, g, dst, src, n_dst, n_src, H):
    import torch
    edge_index = torch.stack([dst, src])

    def fused(a, b, ls):
        return conv.dna_aggregate((a, b), edge_index, (n_dst, n_src), *ls, H)

    def comp(a, b, ls):
        return composition(ops, conv, a, b, ls, dst, src, n_dst, n_src, H)

    def fwd(fn):
        with torch.no_grad():
            return fn(xt, xs, lins)

    def grads(fn):
        leaves = [xt.clone().requires_grad_(True), xs.clone().requires_grad_(True)]
        ls = [tuple(p.clone().requires_grad_(True) for p in pair) for pair in lins]
        fn(leaves[0], leaves[1], ls).backward(g)
        return [leaves[0].grad, leaves[1].grad] + [p.grad for pair in ls for p in pair]

    return dict(zip(ARMS, (lambda: fwd(fused), lambda: fwd(comp), lambda: grads(fused), lambda: grads(comp))))


def memory_of_arm(args, dim, H, batch, arm):
    """In a process of its own: the device memory one call of `arm` needs above its inputs (torch's allocator peak + the
    device memory allocated outside it, i.e. the library's ctx scratch, on a Context that has done nothing else; kernels
    set up first by every arm on a tiny block)."""
    import gc
    import torch
    import euler_b200 as eb
    from euler_b200 import convolution as conv
    from euler_b200 import ops
    dst, src, n_dst, n_src, _ = block_at(args, batch)
    eb.set_graph(eb.get_graph())       # a fresh Context: the dataflow's (larger) scratch would hide the op's
    gc.collect()
    xt, xs, lins, g = inputs(n_dst, n_src, dim, H)
    tiny = make_arms(ops, conv, xt[:2], xs[:8], lins, g[:2], torch.tensor([1, 0], dtype=torch.int32, device="cuda"),
                     torch.tensor([3, 5], dtype=torch.int32, device="cuda"), 2, 8, H)
    for fn in tiny.values():
        fn()
    fn = make_arms(ops, conv, xt, xs, lins, g, dst, src, n_dst, n_src, H)[arm]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    peak, scratch = harness.memory_of(fn)
    return {"torch_peak_bytes": peak, "op_scratch_bytes": scratch, "total_bytes": peak + scratch}


def gate(arms, dim, H):
    """the parity gate of the module docstring; returns the largest relative gradient difference seen"""
    import torch
    f, c = arms["fused_fwd"](), arms["composition_fwd"]()
    if not torch.allclose(f, c, rtol=1e-4, atol=1e-4 * float(c.abs().max())):
        raise SystemExit("PARITY GATE FAILED: fused forward differs from the composition at (%d, %d): max abs diff %g"
                         % (dim, H, float((f - c).abs().max())))
    del f, c
    fg = arms["fused_fwd_bwd"]()
    cg = arms["composition_fwd_bwd"]()
    worst = 0.0
    names = ("grad_x_target", "grad_x_source") + tuple("grad_%s_%s" % (a, b) for a in ("lin_q", "lin_k", "lin_v")
                                                       for b in ("kernel", "bias"))
    for nm, p, q in zip(names, fg, cg):
        floor = 1e-3 * float(q.abs().max())
        diff = float((p - q).abs().max())
        if not torch.allclose(p, q, rtol=1e-3, atol=floor):
            raise SystemExit("PARITY GATE FAILED: fused %s differs from autograd through the composition at (%d, %d): "
                             "max abs diff %g" % (nm, dim, H, diff))
        worst = max(worst, diff / max(floor / 1e-3, 1e-30))
    return worst


def kernel_times(lib, ops, xt, xs, lins, g, dst, src, n_dst, n_src, H):
    """per-kernel times of the fused op on this thread's Context (autograd's backward runs on another thread: both entry
    points are called here directly)"""
    import torch
    from euler_b200 import _lib
    from euler_b200 import convolution as conv
    q = conv.group_dense(xt, *lins[0])
    k, v = conv.group_dense(xs, *lins[1]), conv.group_dense(xs, *lins[2])
    n0, n1 = (t.reshape(-1).contiguous() for t in conv.gcn_norm(torch.stack([dst, src]), (n_dst, n_src)))
    torch.cuda.synchronize()
    ctx = ops._ctx_on_stream()
    gq, gk, gv = (torch.empty_like(t) for t in (q, k, v))
    E, dim = dst.numel(), q.shape[1]

    def fused_passes():
        for _ in range(3):
            _, alpha = ops._raw_dna(q, k, v, n0, n1, dst, src, n_dst, H, True)
            _lib.check(lib.eu_dna_aggregate_backward(ctx._h, g.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), n0.data_ptr(),
                                                     n1.data_ptr(), alpha.data_ptr(), dst.data_ptr(), src.data_ptr(), E, n_dst,
                                                     n_src, H, dim // H, gq.data_ptr(), gk.data_ptr(), gv.data_ptr()))
        torch.cuda.synchronize()
    return harness.kernel_times(lib, ctx, "dna_", fused_passes)


def block_info(dst, n_dst, n_src, indeg, batch):
    E = dst.numel()
    return {"batch": batch, "edges": E, "targets": n_dst, "sources": n_src, "max_edges_per_target": int(indeg.max()),
            "sorted_targets": bool((dst[1:] >= dst[:-1]).all()) if E > 1 else True}


def run(args):
    import torch
    from euler_b200 import _lib, ops
    from euler_b200 import convolution as conv
    torch.cuda.set_device(0)
    lib = _lib.load()
    # the batches, then the memory per arm, each in a fresh process before this one holds any device memory
    choice = {cf: in_child(args, "--choose-batch", "%d,%d" % cf) for cf in CONFIGS}
    memory = {}
    for cf in CONFIGS:
        b = choice[cf]["batch"]
        memory[cf] = {k: in_child(args, "--memory-arm", "%d,%d,%d,%s" % (cf[0], cf[1], b if b else args.batch, k))
                      for k in ARMS if b or k.startswith("fused")}
    results = []
    for dim, H in CONFIGS:
        b = choice[(dim, H)]["batch"]
        res = {"dim": dim, "heads": H, "groups": GROUPS,
               "composition_peak_estimate_bytes": choice[(dim, H)]["composition_peak_estimate_bytes"],
               "free_bytes_at_choice": choice[(dim, H)]["free_bytes_at_choice"]}
        for batch in sorted({args.batch, b or args.batch}, reverse=True):
            t0 = time.time()
            dst, src, n_dst, n_src, indeg = block_at(args, batch)
            torch.cuda.synchronize()
            t_setup = time.time() - t0
            E = dst.numel()
            xt, xs, lins, g = inputs(n_dst, n_src, dim, H)
            arms = make_arms(ops, conv, xt, xs, lins, g, dst, src, n_dst, n_src, H)
            with_comp = batch == b
            if with_comp:
                res["gate_worst_grad_diff_over_floor"] = gate(arms, dim, H)
            else:
                arms = {k: fn for k, fn in arms.items() if k.startswith("fused")}
            rounds, per = harness.rounds_of(args.steps)
            times = {k: float(np.mean(v)) for k, v in harness.time_arms(arms, rounds, args.warmup, per).items()}
            arm_out = {k: {"ms_per_call": ms, "edges_per_sec": E / (ms * 1e-3), "calls": rounds * per,
                           "memory": memory[(dim, H)].get(k) if batch == (b or args.batch) else None}
                       for k, ms in times.items()}
            entry = {"block": block_info(dst, n_dst, n_src, indeg, batch), "arms": arm_out, "setup_s": round(t_setup, 2)}
            if with_comp:
                entry["speedup_fwd"] = arm_out["composition_fwd"]["ms_per_call"] / arm_out["fused_fwd"]["ms_per_call"]
                entry["speedup_fwd_bwd"] = arm_out["composition_fwd_bwd"]["ms_per_call"] / arm_out["fused_fwd_bwd"]["ms_per_call"]
            if batch == args.batch:
                entry["kernels"] = kernel_times(lib, ops, xt, xs, lins, g, dst, src, n_dst, n_src, H)
            res["at_batch_%d" % batch] = entry
            del xt, xs, lins, g, arms, dst, src, indeg
            torch.cuda.empty_cache()
        if not b:
            res["composition"] = "not run: its estimated peak does not fit at any batch of %s" % (BATCHES,)
        results.append(res)
    head = results[0]["at_batch_%d" % args.batch]["arms"]["fused_fwd"]
    out = {"metric": "dna_block_edges_per_sec", "value": head["edges_per_sec"], "unit": "edges/s", "n_gpus": 1,
           "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "data": "synthetic",
           "config": {"workload": "deepest block of a 2-hop GCNDataFlow [[0],[0]] with self loops, R-MAT %dM nodes / %dM edges; "
                                  "DNA attention aggregation at (dim, heads) in %s, groups = %d, batch %d"
                                  % (args.nodes // 10**6, args.edges // 10**6, list(CONFIGS), GROUPS, args.batch),
                      "nodes": args.nodes, "edges": args.edges},
           "configs": results,
           "parity_gate": {"passed": True, "what": "per configuration at the comparison batch: fused forward within 1e-4 (floor "
                                                   "1e-4 x largest) of the composition; fused gradients within 1e-3 (floor 1e-3 "
                                                   "x largest) of autograd through the composition"},
           "gpu": harness.gpu_info(0)}
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    a = parse()
    if a.memory_arm:
        d, h, batch, arm = a.memory_arm.split(",")
        harness.emit(memory_of_arm(a, int(d), int(h), int(batch), arm))
    elif a.choose_batch:
        d, h = a.choose_batch.split(",")
        harness.emit(batch_for(a, int(d), int(h)))
    else:
        run(a)
