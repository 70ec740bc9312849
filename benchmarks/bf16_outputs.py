#!/usr/bin/env python
"""bfloat16 outputs of the headline step on one H100: the step's features and SAGE means written as bf16 by the ops
themselves (out_dtype=), against f32 outputs and against f32 outputs cast to bf16 afterwards.

    python benchmarks/bf16_outputs.py [--rounds R] [--iters K] [--host-iters H]

Workload: the headline step's shape -- R-MAT 10M nodes / 100M edges, D = 256, batch 8192, fanout [15, 10]: sample the
hops, then for each hop l the features of its 8192 / 122,880 source rows and the SAGE means of their neighbours (131,072
feature rows and 131,072 mean rows per step).  Run on an f32 and on a bf16 feature table.  Three arms alternate round by
round in one process:
  f32       the ops' f32 outputs;
  f32+cast  the f32 outputs, then .to(torch.bfloat16) of each (what a mixed-precision user does without out_dtype=);
  bf16      out_dtype=torch.bfloat16.
A PARITY GATE runs first and aborts on failure: on one step under one seed, every bf16 output equals the f32 output
converted on the device, bit for bit, and the host-buffer twins' bf16 outputs equal the device ones.
Reported per table and arm:
  device_ms   ms per step through the Python ops (sampling + features + means on one stream), each arm's step captured
              once in a CUDA graph and replayed --iters times between device events, so the host's launch time is not in
              it; min / median / max over the rounds (the spread);
  e2e_ms      ms per step through the _host C ABI (eu_sample_fanout_batched_host, eu_get_dense_feature_host[_out_dtype],
              eu_sage_mean_aggregate_host[_out_dtype]) into pinned host buffers, host clock, each call returning once its
              results have landed; f32+cast adds torch's host cast of the pinned f32 outputs;
  output_bytes  the bytes of the step's feature and mean outputs, from their shapes (f32+cast: both copies);
  peak_alloc_bytes  torch's allocator peak over one device step, above what was allocated before it.
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout; it needs a GPU."""
import argparse
import ctypes
import time

import harness
import numpy as np
import torch


NODES, EDGES, D, BATCH, COUNTS = 10_000_000, 100_000_000, 256, 8192, [15, 10]
ARMS = ("f32", "f32+cast", "bf16")
BF = torch.bfloat16


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=10)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--host-iters", type=int, default=3)
    return p.parse_args(argv)


def device_step(eb, seeds, arm):
    """one headline step through the Python ops; returns its feature and mean outputs, hop-major"""
    ids, _, _ = eb.sample_fanout(seeds, [[0], [0]], COUNTS)
    dt = BF if arm == "bf16" else torch.float32
    outs = []
    for l, c in enumerate(COUNTS):
        outs.append(eb.get_dense_feature(ids[l], [0], [D], out_dtype=dt)[0])
        outs.append(eb.sage_mean_aggregate(ids[l + 1], c, D, out_dtype=dt))
    if arm == "f32+cast":
        outs = [x.to(BF) for x in outs]
    return outs


class HostStep:
    """the same step through the _host C ABI into pinned buffers"""

    def __init__(self, eb, seeds):
        from euler_b200 import _lib
        self.lib, self.ctx = _lib.load(), eb.Context(eb.get_graph(), seed=3)
        self.rows = [BATCH]
        for c in COUNTS:
            self.rows.append(self.rows[-1] * c)
        self.h_seeds = seeds.cpu().pin_memory()
        self.h_ids = [torch.empty(r, dtype=torch.int64, pin_memory=True) for r in self.rows[1:]]
        self.h_w = [torch.empty(r, dtype=torch.float32, pin_memory=True) for r in self.rows[1:]]
        self.h_t = [torch.empty(r, dtype=torch.int32, pin_memory=True) for r in self.rows[1:]]
        self.out = {dt: [torch.empty((self.rows[l], D), dtype=dt, pin_memory=True) for l in range(len(COUNTS)) for _ in range(2)]
                    for dt in (torch.float32, BF)}
        self.et = np.zeros((len(COUNTS), 1), np.int32)
        self.cs = np.asarray(COUNTS, np.int32)

    def __call__(self, arm):
        lib, h, L = self.lib, self.ctx._h, len(COUNTS)
        P = ctypes.c_void_p * L
        rc = lib.eu_sample_fanout_batched_host(h, self.h_seeds.data_ptr(), 1, BATCH, self.et.ctypes.data, 1, self.cs.ctypes.data, L, -1,
                                               P(*[x.data_ptr() for x in self.h_ids]), P(*[x.data_ptr() for x in self.h_w]),
                                               P(*[x.data_ptr() for x in self.h_t]))
        dt = BF if arm == "bf16" else torch.float32
        out = self.out[dt]
        for l, c in enumerate(COUNTS):
            src = self.h_seeds if l == 0 else self.h_ids[l - 1]
            x, agg = out[2 * l].data_ptr(), out[2 * l + 1].data_ptr()
            if arm == "bf16":
                rc |= lib.eu_get_dense_feature_host_out_dtype(h, src.data_ptr(), self.rows[l], 0, D, 1, x)
                rc |= lib.eu_sage_mean_aggregate_host_out_dtype(h, self.h_ids[l].data_ptr(), self.rows[l], c, D, 1, agg)
            else:
                rc |= lib.eu_get_dense_feature_host(h, src.data_ptr(), self.rows[l], 0, D, x)
                rc |= lib.eu_sage_mean_aggregate_host(h, self.h_ids[l].data_ptr(), self.rows[l], c, D, agg)
        if rc:
            raise RuntimeError("euler_b200: " + lib.eu_last_error().decode())
        return [x.to(BF) for x in out] if arm == "f32+cast" else out


def gate(eb, seeds, host):
    eb.seed(11)
    f32 = device_step(eb, seeds, "f32")
    eb.seed(11)
    bf = device_step(eb, seeds, "bf16")
    for a, b in zip(f32, bf):
        if b.dtype != BF or not torch.equal(b.view(torch.int16), a.to(BF).view(torch.int16)):
            raise SystemExit("PARITY GATE FAILED: a bf16 output differs from the f32 output converted on the device")
    host.ctx.seed(11)
    hf = [x.clone() for x in host("f32")]
    host.ctx.seed(11)
    hb = host("bf16")
    for a, b in zip(hf, hb):
        if not torch.equal(b.view(torch.int16), a.cuda().to(BF).view(torch.int16).cpu()):
            raise SystemExit("PARITY GATE FAILED: a bf16 host output differs from the f32 host output converted on the device")
    return "bit-exact"


def spread(v):
    return {"min": round(min(v), 4), "median": round(float(np.median(v)), 4), "max": round(max(v), 4)}


def run_table(eb, dtype, args):
    g = eb.Graph.rmat(NODES, EDGES, seed=42, feat_dim=D, feat_seed=7, feat_dtype=dtype)
    eb.set_graph(g, rng="philox", seed=1)
    seeds = torch.randint(1, NODES + 1, (BATCH,), generator=torch.Generator().manual_seed(5)).cuda()
    host = HostStep(eb, seeds)
    res = {"table": dtype, "gate": gate(eb, seeds, host)}
    feat_rows = sum(host.rows[:-1])
    graphs = {}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    for arm in ARMS:
        esz = 2 if arm == "bf16" else 4
        res.setdefault(arm, {})["output_bytes"] = 2 * feat_rows * D * esz + (2 * feat_rows * D * 2 if arm == "f32+cast" else 0)
        host(arm)
        with torch.cuda.stream(s):
            device_step(eb, seeds, arm)
            graphs[arm] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[arm], stream=s):
                device_step(eb, seeds, arm)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    dev = {a: [] for a in ARMS}
    e2e = {a: [] for a in ARMS}
    for _ in range(args.rounds):
        for arm in ARMS:
            dev[arm] += harness.time_arms({arm: graphs[arm].replay}, 1, 0, args.iters)[arm]
            t0 = time.perf_counter()
            for _ in range(args.host_iters):
                host(arm)
            e2e[arm].append((time.perf_counter() - t0) * 1e3 / args.host_iters)
    for arm in ARMS:
        res[arm].update(device_ms=spread(dev[arm]), e2e_ms=spread(e2e[arm]),
                        peak_alloc_bytes=harness.memory_of(lambda: device_step(eb, seeds, arm))[0])
    del graphs
    for key in ("device_ms", "e2e_ms"):
        res["bf16_over_f32_" + key] = round(res["bf16"][key]["median"] / res["f32"][key]["median"], 3)
    host.ctx.close()
    eb.set_graph(None)
    g.close()
    torch.cuda.empty_cache()
    return res


def main():
    args = parse()
    if not torch.cuda.is_available():
        raise SystemExit("bf16_outputs.py needs a GPU")
    import euler_b200 as eb
    out = {"benchmark": "bf16_outputs", "gpu": harness.gpu_info(torch.cuda.current_device()),
           "workload": "rmat %d nodes / %d edges, D = %d, batch %d, fanout %s" % (NODES, EDGES, D, BATCH, COUNTS),
           "rounds": args.rounds, "iters": args.iters, "host_iters": args.host_iters, "tables": []}
    for dtype in ("float32", "bfloat16"):
        out["tables"].append(run_table(eb, dtype, args))
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    main()
