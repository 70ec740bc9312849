#!/usr/bin/env python
"""A training step on float32 against bfloat16 id tables, at one shape, in one run on one GPU: DeepWalk's
(unsupervised.DeepWalk(table_dtype=...), train_step; the default), a knowledge-graph model's (knowledge.TransE, TransR,
TransD or DistMult(table_dtype=...), train_step), a supervised SageEncoder's (encoders.SageEncoder(table_dtype=...),
optimizers.minimize) or a ScalableSageEncoder's over f32 against bf16 embedding stores (store_dtype=..., train_step).

    python benchmarks/bf16_tables.py [--model deepwalk] [--nodes N] [--edges E] [--dim D] [--batch B] [--optimizer NAME]
                                     [--steps K] [--warmup W]
    python benchmarks/bf16_tables.py --model {transe,transr,transd,distmult} [--nodes N] [--triples T] [--relations R]
                                     [--dim D] [--rel-dim D] [--batch B] [--negs K] [--lr LR] [--optimizer NAME] [--steps K]
                                     [--warmup W]
    python benchmarks/bf16_tables.py --model sage [--nodes N] [--edges E] [--dim D] [--batch B] [--lr LR] [--optimizer NAME]
                                     [--steps K] [--warmup W]
    python benchmarks/bf16_tables.py --model scalable [--nodes N] [--edges E] [--dim D] [--batch B] [--lr LR] [--steps K]
                                     [--warmup W] [--no-part-b]

DeepWalk: a step is train_step: the walks, pairs and negatives drawn on the device, the fused skip-gram forward, its sparse
backward, and the optimizer's fused update of both tables and their slots (bf16: stochastic rounding on every store), on an
R-MAT graph.  A knowledge-graph step is train_step on B triples from sample_edge: the relation ids from the edge feature
'id', K negatives per triple from sample_node, the fused margin loss ('both' corruptions, L1) and its sparse backward, and
the optimizer's update of every table and slot.  Its graph is built from a seed: N entities and T triples, uniform
endpoints, relations of Zipf-like frequency (exponent 1.1) over R relation ids (Graph.from_csr + set_edges).  Defaults:
10M entities, 10M triples, 1 000 relations, B = 8192, K = 64, dim 128 (TransR 128 x 32), Adam at lr 0.001.
SageEncoder: a step is optimizers.minimize of a SuperviseModel over SageEncoder on the graph of benchmarks/sage_encoder.py
(the 10M-node R-MAT with a 128-column dense slot and its two seeded uint64 slots): use_id at dim 128 and both slots at dim
128 (tables of N + 2, 10^6 + 2 and 10^7 + 2 rows), fanout [15, 10], 'mean' (so the deepest hop is pooled), dim 128, and a
label of 8 columns taken from the dense slot (each column's sign) -- the fanout, both encoder passes with the tables' sparse
backward, and the optimizer's update of the dense parameters and every table and slot.  Defaults: B = 512, Adam at lr 0.001.
Both arms draw the same ids (the sampler is reseeded before each step of each arm) and start from the same tables (the
f32 arm holds the bf16 arm's widened values).  The arms alternate round by round, timed with device events.  Reported per
arm: ms per step, the tables' and slots' bytes, and the mean loss of the timed steps; the card's name, power limit and max
SM clock are read in the same run.  One JSON line on stdout.  It needs a GPU: without one it fails.

ScalableSageEncoder (--model scalable), part A: the configuration of benchmarks/scalable_encoder.py -- the 10M-node /
100M-edge R-MAT with its 128-column dense slot, 2 layers at dim 128, fanout 10, 'mean', batch 8192, a Linear(128, 16) head
on seeded labels and SGD at lr 0.01 -- with f32 stores against bf16 stores (store_dtype=torch.bfloat16).  A step is
forward(training=True), the loss and train_step; the f32 arm starts from the bf16 arm's widened stores, both arms draw the
same seeds and the sampler is reseeded per step.  Reported per arm: ms per step, the two store ops alone (store_exchange over
the batch, store_accumulate over the hop with count 10 and 'mean'), the store pair's bytes and the mean loss; all timed
arms alternate round by round.  Part B: the headline graph, the 50M-node / 500M-edge R-MAT with bf16 features of 256
columns, and the same 2-layer encoder over them.  The store pair's bytes, and the f32 initialisation each bf16 store is rounded from, are computed from the
shapes and compared with the free device memory after the graph is built: each arm that fits runs on its own, and an arm that
does not is reported as not fitting from that arithmetic, never by attempting the allocation."""
import argparse

import harness
KG_MODELS = {"transe": "TransE", "transr": "TransR", "transd": "TransD", "distmult": "DistMult"}


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="deepwalk", choices=["deepwalk", "sage", "scalable"] + sorted(KG_MODELS))
    p.add_argument("--nodes", type=int, default=10_000_000)
    p.add_argument("--edges", type=int, default=100_000_000)
    p.add_argument("--triples", type=int, default=10_000_000)
    p.add_argument("--relations", type=int, default=1000)
    p.add_argument("--dim", type=int, default=128)
    p.add_argument("--rel-dim", type=int, default=32, help="TransR's relation dim")
    p.add_argument("--batch", type=int, default=None, help="default 512 (DeepWalk), 8192 (knowledge graph)")
    p.add_argument("--negs", type=int, default=64)
    p.add_argument("--lr", type=float, default=None, help="default 0.01 (DeepWalk), 0.001 (knowledge graph)")
    p.add_argument("--optimizer", default="adam")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--no-part-b", action="store_true", help="--model scalable: skip the 50M-node part")
    args = p.parse_args(argv)
    kg = args.model not in ("deepwalk", "sage", "scalable")
    if args.batch is None:
        args.batch = 8192 if kg or args.model == "scalable" else 512
    if args.lr is None:
        args.lr = 0.01 if args.model in ("deepwalk", "scalable") else 0.001
    return args


def kg_graph(n_ent, n_tri, n_rel, seed=11):
    """the knowledge graph of the module docstring: entities of node type 0, triples of edge type 0 whose relation id is
    the dense edge feature 'id'"""
    import numpy as np
    import euler_b200 as eb
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_rel + 1) ** 1.1
    rel = rng.choice(n_rel, size=n_tri, p=p / p.sum())
    src, dst = rng.randint(0, n_ent, n_tri), rng.randint(0, n_ent, n_tri)
    order = np.lexsort((dst, src))
    src, dst, rel = src[order], dst[order], rel[order]
    ptr = np.zeros(n_ent + 1, np.int64)
    np.add.at(ptr, src + 1, 1)
    g = eb.Graph.from_csr(np.arange(n_ent), np.cumsum(ptr), dst, w=np.ones(n_tri, np.float32))
    g.set_edges(src, dst, np.zeros(n_tri, np.int32), dense=rel.reshape(-1, 1).astype(np.float32), dense_names=['id'])
    return g


def sage_model(args, dt):
    """the supervised SageEncoder of the module docstring (f32 tables take sparse gradients, as the bf16 proxies do)"""
    import torch
    import torch.nn.functional as F
    import euler_b200 as eb
    from harness import DENSE_DIM, SLOTS
    from euler_b200.encoders import SageEncoder
    from euler_b200.supervised import SuperviseModel

    class SupervisedSage(SuperviseModel):
        def __init__(self):
            super().__init__("feat0", 8, dim=args.dim, device="cuda")
            self.encoder = SageEncoder([[0], [0]], [15, 10], args.dim, aggregator="mean", feature_idx="feat0",
                                       feature_dim=DENSE_DIM, max_id=args.nodes, use_id=True,
                                       sparse_feature_idx=[n for n, _ in SLOTS], sparse_feature_max_id=[m - 1 for _, m in SLOTS],
                                       embedding_dim=args.dim, sparse_grad=dt == torch.float32, device="cuda", table_dtype=dt)

        def embed(self, n_id):
            return self.encoder(n_id)

        def forward(self, inputs):
            """SuperviseModel's loss, its labels in {0, 1}: the signs of the slot's first 8 columns"""
            label = (eb.get_dense_feature(inputs, ["feat0"], [8])[0] > 0).float()
            return F.binary_cross_entropy_with_logits(self.out_fc(self.embed(inputs)), label)

    return SupervisedSage()


SCALABLE_LABELS = 16
SCALABLE_FANOUT = 10


def store_pair_bytes(n_nodes, dim, dt):
    """one layer's store and gradient store, [n_nodes + 2, dim] each"""
    return 2 * (n_nodes + 2) * dim * (2 if dt == "bf16" else 4)


def init_peak_bytes(n_nodes, dim, dt):
    """the most the stores of a 2-layer encoder hold while they are built: a bf16 store is rounded from an f32 one, which
    lives until the bf16 copy exists, and its gradient store comes after"""
    row = (n_nodes + 2) * dim
    return 4 * row + 2 * row if dt == "bf16" else 2 * 4 * row


def scalable_arms(args, n_nodes, feature, dts, steps, warmup, store_ops=True):
    """ScalableSageEncoder train steps (and the store ops alone) for each store dtype of dts on the installed graph, the f32
    arm from the bf16 arm's widened stores; {dt: {...}} of ms per step, store-op ms, store bytes and mean loss"""
    import numpy as np
    import torch
    import euler_b200 as eb
    from euler_b200.encoders import ScalableSageEncoder
    fid, fdim = feature
    labels = (torch.rand(args.batch, SCALABLE_LABELS, generator=torch.Generator().manual_seed(3)) < 0.5).float().cuda()
    encs, heads, opts = {}, {}, {}
    for k in dts:
        torch.manual_seed(0)
        encs[k] = ScalableSageEncoder([0], SCALABLE_FANOUT, 2, args.dim, aggregator="mean", feature_idx=[fid], feature_dim=[fdim],
                                      max_id=n_nodes, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1),
                                      store_dtype=torch.bfloat16 if k == "bf16" else torch.float32, store_seed=5)
        heads[k] = torch.nn.Linear(args.dim, SCALABLE_LABELS).cuda()
        opts[k] = torch.optim.SGD(list(encs[k].parameters()) + list(heads[k].parameters()), lr=args.lr)
    if "bf16" in encs and "f32" in encs:
        with torch.no_grad():
            for a, b in zip(encs["f32"].stores, encs["bf16"].stores):
                a.copy_(b.float())
    torch.cuda.empty_cache()
    batches = [torch.from_numpy(np.random.RandomState(100 + i).randint(1, n_nodes + 1, size=args.batch)).cuda()
               for i in range(warmup + steps)]
    losses = {k: [] for k in encs}
    nxt = {k: 0 for k in encs}

    def train(k):
        i = nxt[k] % len(batches)
        nxt[k] += 1
        eb.seed(1000 + i)                      # the sampler reseeded per step: both arms draw the same hop
        enc = encs[k]
        loss = torch.nn.functional.binary_cross_entropy_with_logits(heads[k](enc(batches[i], training=True)), labels)
        enc.train_step(loss, opts[k])
        losses[k].append(loss.detach())

    eb.seed(7)
    node, neighbor = eb.sample_fanout(batches[0], [[0]], [SCALABLE_FANOUT], default_node=n_nodes + 1)[0]
    gen = torch.Generator(device="cuda").manual_seed(4)
    rows = torch.randn(node.numel(), args.dim, device="cuda", generator=gen)
    grad = torch.randn(node.numel(), args.dim, device="cuda", generator=gen)
    counter = torch.zeros((), dtype=torch.int64, device="cuda")

    def ops_of(k):
        store, gs = encs[k].stores[0], encs[k].gradient_stores[0]
        sr = dict(seed=5, step=counter, tensor=0) if k == "bf16" else {}

        def run():
            eb.store_exchange(store, gs, node, rows)
            eb.store_accumulate(gs, neighbor, grad, SCALABLE_FANOUT, "mean", **sr)
        return run

    arms = {("step", k): (lambda k=k: train(k)) for k in encs}
    if store_ops:
        arms.update({("store_ops", k): ops_of(k) for k in encs})
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    for k in losses:
        losses[k].clear()
    rounds, per = harness.rounds_of(steps)
    ms = harness.time_arms(arms, rounds, 0, per)
    out = {}
    for k in encs:
        out[k] = {"ms_per_step": float(np.mean(ms[("step", k)])), "steps": rounds * per,
                  "store_pair_bytes": sum(t.numel() * t.element_size() for t in encs[k].stores + encs[k].gradient_stores),
                  "mean_loss": float(np.mean([float(x) for x in losses[k]]))}
        if store_ops:
            out[k]["store_ops_ms"] = float(np.mean(ms[("store_ops", k)]))
    return out


def run_scalable(args):
    import torch
    import euler_b200 as eb
    torch.cuda.set_device(0)
    from harness import DENSE_DIM
    out = {"workload": "scalable_sage_train_step", "gpu": harness.gpu_info(0), "dim": args.dim, "fanout": SCALABLE_FANOUT, "layers": 2,
           "aggregator": "mean", "batch": args.batch, "optimizer": "sgd", "lr": args.lr}
    g = harness.build_graph(args)
    a = scalable_arms(args, args.nodes, ("feat0", DENSE_DIM), ("bf16", "f32"), args.steps, args.warmup)
    a["bf16_over_f32_time"] = a["bf16"]["ms_per_step"] / a["f32"]["ms_per_step"]
    a["bf16_over_f32_store_ops_time"] = a["bf16"]["store_ops_ms"] / a["f32"]["store_ops_ms"]
    out["part_a"] = dict(graph="rmat %d nodes / %d edges, feat_dim %d f32" % (args.nodes, args.edges, DENSE_DIM), **a)
    g.close()
    del g
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    if not args.no_part_b:
        out["part_b"] = scalable_part_b(args)
    harness.emit(out)


def scalable_part_b(args):
    """the headline graph: fit from the arithmetic, then the arms that fit"""
    import gc
    import time
    import torch
    import euler_b200 as eb
    n, E = 50_000_000, 500_000_000
    D = 256
    res = {"graph": "rmat %d nodes / %d edges, feat_dim %d bf16" % (n, E, D)}
    t0 = time.time()
    g = eb.Graph.rmat(n, E, seed=11, feat_dim=D, feat_dtype="bfloat16")
    torch.cuda.synchronize()
    eb.set_graph(g, rng="philox", seed=5)
    free, total = torch.cuda.mem_get_info()
    spare = 2 << 30                      # the step's own buffers: batch, hop, plan scratch, the head
    res.update(build_s=round(time.time() - t0, 1), graph_hbm_bytes=g.hbm_bytes, free_after_graph_bytes=free, device_bytes=total)
    fits = []
    for dt in ("bf16", "f32"):
        need = max(store_pair_bytes(n, args.dim, dt), init_peak_bytes(n, args.dim, dt)) + spare
        ok = need <= free
        res[dt] = {"store_pair_bytes": store_pair_bytes(n, args.dim, dt), "init_peak_bytes": init_peak_bytes(n, args.dim, dt),
                   "needed_bytes": need, "fits": ok}
        if ok:
            fits.append(dt)
        else:
            res[dt]["result"] = "does not fit: %.1f GB needed beside the graph, %.1f GB free" % (need / 1e9, free / 1e9)
    for dt in fits:                      # one arm at a time: the two pairs together are not the question here
        r = scalable_arms(args, n, (0, D), (dt,), max(1, args.steps // 2), min(args.warmup, 2), store_ops=False)[dt]
        res[dt].update(r)
        gc.collect()
        torch.cuda.empty_cache()
    g.close()
    return res


def run(args):
    import numpy as np
    import torch
    import euler_b200 as eb
    from euler_b200 import knowledge, optimizers, unsupervised as un
    torch.cuda.set_device(0)
    if args.model == "scalable":
        return run_scalable(args)
    kg = args.model not in ("deepwalk", "sage")
    sage = args.model == "sage"
    if kg:
        eb.set_graph(kg_graph(args.nodes, args.triples, args.relations), rng="philox", seed=1)
    elif sage:
        harness.build_graph(args)
    else:
        eb.set_graph(eb.Graph.rmat(args.nodes, args.edges, seed=11), rng="philox", seed=1)
    models = {}
    for name, dt in (("bf16", torch.bfloat16), ("f32", torch.float32)):
        torch.manual_seed(3)
        if sage:
            models[name] = sage_model(args, dt)
        elif kg:
            rel_dim = args.rel_dim if args.model == "transr" else args.dim
            models[name] = getattr(knowledge, KG_MODELS[args.model])(
                0, 0, args.nodes - 1, args.relations - 1, args.dim, rel_dim, num_negs=args.negs, margin=1.0, l1=True,
                corrupt='both', device="cuda", table_dtype=dt)
        else:
            models[name] = un.DeepWalk(0, [0], args.nodes, args.dim, walk_len=3, num_negs=5, device="cuda", table_dtype=dt)
    with torch.no_grad():
        for p16, p32 in zip(models["bf16"].parameters(), models["f32"].parameters()):
            p32.copy_(p16.float())
    torch.cuda.empty_cache()
    opts = {k: optimizers.get(args.optimizer)(list(m.parameters()), args.lr, **({"seed": 5} if k == "bf16" else {}))
            for k, m in models.items()}
    if kg:   # the triples of each step, drawn once: both arms train on the same edges
        batches = []
        for i in range(args.warmup + args.steps):
            eb.seed(100 + i)
            batches.append(eb.sample_edge(args.batch, 0))
    else:
        batches = [torch.from_numpy(np.random.RandomState(100 + i).randint(1, args.nodes + 1, size=args.batch)).cuda()
                   for i in range(args.warmup + args.steps)]
    losses = {k: [] for k in models}

    def step(k, i):
        eb.seed(1000 + i)
        if sage:
            losses[k].append(optimizers.minimize(opts[k], models[k](batches[i]), models[k]).detach())
            return
        out = models[k].train_step(batches[i], opts[k])
        losses[k].append(out.loss if kg else out[0])

    for i in range(args.warmup):
        for k in models:
            step(k, i)
    torch.cuda.synchronize()
    for k in losses:
        losses[k].clear()
    rounds, per = harness.rounds_of(args.steps)
    tot = {k: [0.0, 0] for k in models}
    i = args.warmup
    for _ in range(rounds):
        n = min(per, args.warmup + args.steps - i)
        if n <= 0:
            break
        ms = harness.time_arms({k: (lambda k=k, seq=iter(range(i, i + n)): step(k, next(seq))) for k in models}, 1, 0, n)
        for k, v in ms.items():
            tot[k][0] += v[0] * n
            tot[k][1] += n
        i += n

    def state_bytes(k):
        ps = [p for p in models[k].parameters() if p.dim() == 2 and p.shape[0] > 10 ** 5] if sage else list(models[k].parameters())
        return sum(p.numel() * p.element_size() for p in ps) + sum(
            t.numel() * t.element_size() for p in ps for t in opts[k].state[p].values() if torch.is_tensor(t))

    if kg:
        out = {"workload": "%s_train_step" % args.model, "entities": args.nodes, "triples": args.triples,
               "relations": args.relations, "dim": args.dim, "rel_dim": args.rel_dim if args.model == "transr" else args.dim,
               "batch": args.batch, "negs": args.negs, "optimizer": args.optimizer, "lr": args.lr, "gpu": harness.gpu_info(0)}
    elif sage:
        out = {"workload": "supervised_sage_minimize_step", "nodes": args.nodes, "edges": args.edges, "dim": args.dim,
               "fanout": [15, 10], "aggregator": "mean", "batch": args.batch, "optimizer": args.optimizer, "lr": args.lr,
               "gpu": harness.gpu_info(0)}
    else:
        out = {"workload": "deepwalk_train_step", "nodes": args.nodes, "edges": args.edges, "dim": args.dim, "batch": args.batch,
               "optimizer": args.optimizer, "gpu": harness.gpu_info(0)}
    for k, (ms, n) in tot.items():
        out[k] = {"ms_per_step": ms / n, "steps": n, "table_and_slot_bytes": state_bytes(k),
                  "mean_loss": float(np.mean([float(x) for x in losses[k]]))}
    out["bf16_over_f32_time"] = out["bf16"]["ms_per_step"] / out["f32"]["ms_per_step"]
    harness.emit(out)


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
