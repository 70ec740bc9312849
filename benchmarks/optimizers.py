#!/usr/bin/env python
"""tf_euler's optimizers (euler_b200/optimizers.py) on one H100: the fused step (one device op per parameter) against the
fused=False step, TF 1.x's op sequence written out in torch, one torch op per TF op.

    python benchmarks/optimizers.py [--steps K] [--warmup W]

Workloads:
  - sparse Adam, Momentum and Adagrad on id tables of 10M x 128 and 20M x 64 float32, the sizes of table the project is for.
    The gradient's rows are those of a DeepWalk batch (512 sources, walks of 3 steps, windows of 1, 5 negatives a pair):
    the distinct ids among 512 x 4 walk nodes and 3,072 x 5 negatives, drawn uniformly, with unit-normal values.
  - the dense Adam step of the Dense layers of SageEncoder([[0], [0]], [10, 10], 128) over 128 features.
A GATE first: from the same parameters and slots, one step of each arm leaves bit-identical parameters and slots, else it
aborts.  Then the arms alternate round by round, each stepping its own state, timed with device events.
Reported per arm: ms per step and torch's allocator peak above the inputs; for sparse Adam the achieved GB/s of the fused
pass from its algorithmic bytes 24 N D + 4 R (D + 2) (var, m and v read and written once, the gradient rows and their ids
read once) and that rate over the H100 SXM's 3.35 TB/s; the card's name, power limit and max SM clock read in the same run.
One JSON line on stdout.  It needs a GPU: without one it fails rather than measure anything else."""
import argparse

import harness
from harness import timed

TABLES = [(10_000_000, 128), (20_000_000, 64)]
HBM_BYTES_PER_S = 3.35e12


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    return p.parse_args(argv)


def deepwalk_rows(N, gen):
    """the sorted distinct rows a DeepWalk batch touches: 512 walks of 4 nodes, 512 x 6 pairs with 5 negatives each"""
    ids = torch.randint(0, N, (512 * 4 + 512 * 6 * 5,), generator=gen, device="cuda")
    return torch.unique(ids)


def make_arm(name, params, grads, fused):
    from euler_b200 import optimizers
    opt = optimizers.get(name)(params, 0.01, fused=fused)
    for p, g in zip(params, grads):
        p.grad = g

    def step():
        opt.step()
    return opt, step


def bits_equal(a, b):
    return bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))


def gate(name, opts, params_per_arm):
    """after one step from identical states the arms agree bit for bit on every parameter and slot"""
    (o0, p0), (o1, p1) = zip(opts, params_per_arm)
    for a, b in zip(p0, p1):
        if not bits_equal(a.detach(), b.detach()):
            raise SystemExit("GATE FAILED: %s parameters differ" % name)
        for k in o0.state[a]:
            if not bits_equal(o0.state[a][k], o1.state[b][k]):
                raise SystemExit("GATE FAILED: %s slot %s differs" % (name, k))
    if name == 'adam' and not bits_equal(o0.beta_powers, o1.beta_powers):
        raise SystemExit("GATE FAILED: adam powers differ")


def compare(name, make_params, grads, args):
    """fused and fused=False arms of optimizer `name`, from identical parameters: gate, then time"""
    arms, opts, plist = {}, [], []
    for fused in (True, False):
        params = make_params()
        opt, step = make_arm(name, params, grads, fused)
        step()
        opts.append(opt)
        plist.append(params)
        arms["fused" if fused else "literal"] = step
    torch.cuda.synchronize()
    gate(name, opts, plist)
    res = timed(arms, args.steps, args.warmup)
    del arms, opts, plist
    torch.cuda.empty_cache()
    return res


def run(args):
    import euler_b200 as eb
    from euler_b200 import encoders
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/optimizers.py needs a GPU")
    eb.set_graph(eb.Graph.rmat(1000, 5000, seed=1), rng="minstd", seed=1)
    gen = torch.Generator(device="cuda").manual_seed(0)
    out = {"metric": "ms_per_step", "gpu": harness.gpu_info(0), "steps": args.steps, "warmup": args.warmup, "sparse": [], "dense": {}}
    for N, D in TABLES:
        rows = deepwalk_rows(N, gen)
        R = rows.numel()
        vals = torch.randn(R, D, generator=gen, device="cuda")
        grad = torch.sparse_coo_tensor(rows[None], vals, (N, D), is_coalesced=True)
        base = torch.randn(N, D, generator=gen, device="cuda")
        rec = {"N": N, "D": D, "R": int(R)}
        for name in ('adam', 'momentum', 'adagrad'):
            res = compare(name, lambda: [torch.nn.Parameter(base.clone())], [grad], args)
            if name == 'adam':
                nbytes = 24 * N * D + 4 * R * (D + 2)
                for arm in res.values():
                    arm["algorithmic_GBps"] = nbytes / (arm["ms_per_call"] * 1e-3) / 1e9
                res["fused"]["share_of_3.35TBps"] = res["fused"]["algorithmic_GBps"] * 1e9 / HBM_BYTES_PER_S
                rec["adam_bytes"] = int(nbytes)
            rec[name] = res
        out["sparse"].append(rec)
        del base, grad, vals, rows
        torch.cuda.empty_cache()
    torch.manual_seed(0)
    enc = encoders.SageEncoder([[0], [0]], [10, 10], 128, 'mean', feature_idx=0, feature_dim=128, device="cuda")
    dense = [p.detach().clone() for p in enc.parameters()]
    dgrads = [torch.randn(p.shape, generator=gen, device="cuda") for p in dense]
    out["dense"] = {"params": len(dense), "elements": int(sum(p.numel() for p in dense)),
                    "adam": compare('adam', lambda: [torch.nn.Parameter(p.clone()) for p in dense], dgrads, args)}
    harness.emit(out)


if __name__ == "__main__":
    import torch
    harness.divert_stdout()
    run(parse())
