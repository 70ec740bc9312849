"""What the scripts under benchmarks/ share: the one JSON line on stdout, the card's data, the device-event timer, the memory
probe, the fresh-process runner, and the workload parts more than one script measures.  A library, not a script: a script
imports it first, and no script imports another.

Importing it puts the repository root (the package and bench.py) and tests/ (the numpy restatements some gates compare
against) on sys.path, so every script still runs as `python benchmarks/<name>.py`."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

_REAL_STDOUT = None


def divert_stdout():
    """Keep the process's real stdout for emit() and send fd 1 to stderr, so whatever a library prints stays out of the one
    JSON line.  Called once, at the start of __main__."""
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)


def emit(out):
    """the ONE JSON line goes to the process's real stdout; everything else any library printed went to stderr"""
    os.write(_REAL_STDOUT if _REAL_STDOUT is not None else 1, (json.dumps(out) + "\n").encode())


def gpu_info(index):
    """card name, power limit and max SM clock, read in the measuring run"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, mhz = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as e:                      # noqa: BLE001
        return {"unavailable": str(e)}


def rounds_of(steps):
    """--steps calls split into at most 5 alternating rounds: (rounds, calls per round)"""
    rounds = max(1, min(5, steps))
    return rounds, -(-steps // rounds)


def time_arms(arms, rounds, warmup=0, calls=1):
    """arms: ordered name -> thunk.  `warmup` times every arm in turn, untimed; then each round times every arm in turn, `calls`
    calls between two device events with the device idle before and after.  Returns each arm's ms per call, one per round."""
    import torch
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / calls)
    return ms


def memory_of(fn):
    """Run fn once.  Returns (torch's allocator peak above what was allocated before the call, the device bytes allocated
    outside torch's reserve during the call -- where the library's ctx scratch lives)."""
    import torch
    torch.cuda.synchronize()
    alloc0, free0, reserved0 = torch.cuda.memory_allocated(), torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    outside = (free0 - torch.cuda.mem_get_info()[0]) - (torch.cuda.memory_reserved() - reserved0)
    del r
    return int(torch.cuda.max_memory_allocated() - alloc0), int(outside)


def timed(arms, steps, warmup):
    """Each arm warmed up on its own and its allocator peak taken over one more call; then --steps calls per arm, the arms
    alternating in rounds.  {arm: {ms_per_call (the mean), calls, torch_peak_bytes}}"""
    peak = {}
    for k, fn in arms.items():
        for _ in range(warmup):
            fn()
        peak[k] = memory_of(fn)[0]
    rounds, per = rounds_of(steps)
    ms = time_arms(arms, rounds, 0, per)
    return {k: {"ms_per_call": float(np.mean(v)), "calls": rounds * per, "torch_peak_bytes": peak[k]} for k, v in ms.items()}


def in_fresh_process(script, argv):
    """`python script argv...` in a process of its own: its last stdout line, parsed as JSON"""
    r = subprocess.run([sys.executable, script] + list(argv), capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit("%s %s failed:\n%s" % (os.path.basename(script), " ".join(argv), r.stderr[-2000:]))
    return json.loads(r.stdout.strip().splitlines()[-1])


def kernel_times(lib, ctx, prefix, run):
    """The library's per-kernel times on `ctx` while run() executes (its events bracket every kernel, so this is a pass of
    its own): {kernel: {launches, ms_per_launch}} for the kernels whose names start with `prefix`."""
    lib.eu_ctx_profile(ctx._h, 1)
    run()
    buf = ctypes.create_string_buffer(1 << 16)
    lib.eu_ctx_profile_read(ctx._h, buf, len(buf))
    lib.eu_ctx_profile(ctx._h, 0)
    kern = {}
    for line in buf.value.decode().splitlines():
        parts = line.split(",")
        if len(parts) == 4 and parts[0].startswith(prefix):
            kern[parts[0]] = {"launches": int(parts[2]), "ms_per_launch": float(parts[3]) / max(int(parts[2]), 1)}
    return kern


# ---- workload parts measured by more than one script

DENSE_DIM, DIM = 128, 16                               # the dense slot's width; the id and slot tables' dim
SLOTS = (("u64_0", 10 ** 6), ("u64_1", 10 ** 7))       # name, max_id + 1 (the default value; the table has one more row)


def slot_arrays(n, seed=2024):
    """u64_ptr [n * 2 + 1] and u64_val of the two seeded slots"""
    rng = np.random.RandomState(seed)
    la = rng.randint(1, 9, size=n)
    la[rng.rand(n) < 0.2] = 0
    big = rng.rand(n) < 0.001
    la[big] = rng.randint(300, 2001, size=int(big.sum()))
    lb = rng.randint(1, 5, size=n)
    lens = np.stack([la, lb], axis=1).reshape(-1).astype(np.int64)
    ptr = np.zeros(2 * n + 1, np.int64)
    np.cumsum(lens, out=ptr[1:])
    slot = np.repeat(np.tile(np.arange(2, dtype=np.int8), n), lens)
    vals = np.empty(int(ptr[-1]), np.uint64)
    na, nb = int((slot == 0).sum()), int((slot == 1).sum())
    vals[slot == 0] = (rng.zipf(1.2, size=na) - 1) % SLOTS[0][1]
    vals[slot == 1] = rng.randint(0, SLOTS[1][1], size=nb)
    return ptr, vals


def build_graph(args):
    """the R-MAT of --nodes / --edges with a dense slot of DENSE_DIM columns and the two seeded uint64 slots, installed"""
    import euler_b200 as eb
    from bench import GRAPH_SEED
    g0 = eb.Graph.rmat(args.nodes, args.edges, seed=GRAPH_SEED, feat_dim=DENSE_DIM, device=0)
    csr = g0.export(with_feat=True)
    g0.close()
    ptr, vals = slot_arrays(args.nodes)
    g = eb.Graph.from_csr(csr["ids"], csr["grp_ptr"], csr["nbr"], n_edge_types=csr["T"], cum_w=csr["cum_w"], grp_cum=csr["grp_cum"],
                          node_type=csr["node_type"], node_w=csr["node_w"], feat=csr["feat"], feat_slot_dims=[DENSE_DIM],
                          u64_ptr=ptr, u64_val=vals, n_u64_slots=2)
    del csr
    eb.set_graph(g, rng="philox", seed=5)
    return g


def block_edges(args, self_loops=False):
    """the deepest block of a 2-hop GCNDataFlow [[0],[0]] at --batch on the R-MAT of --nodes / --edges: (dst, src) int32 on
    the device, its sizes and each target's edge count"""
    import torch
    import euler_b200 as eb
    from bench import GRAPH_SEED
    from euler_b200.dataflow import GCNDataFlow
    graph = eb.Graph.rmat(args.nodes, args.edges, seed=GRAPH_SEED, device=0)
    eb.set_graph(graph)
    seeds = torch.from_numpy(np.random.RandomState(7000).randint(1, args.nodes + 1, size=args.batch).astype(np.int64)).cuda()
    blk = GCNDataFlow([[0], [0]], add_self_loops=self_loops)(seeds)[0]
    ei = blk.edge_index.to(torch.int32)
    n_dst, n_src = blk.size
    dst, src = ei[0].contiguous(), ei[1].contiguous()
    return dst, src, n_dst, n_src, torch.bincount(dst.long(), minlength=n_dst)
