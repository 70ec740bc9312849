#!/usr/bin/env python
"""The streaming AUC update (ops.metric_auc_update: tf.metrics.auc's per-batch counts added to the state, and the value) on
one H100, against two torch formulations of the same step, and the metric's share of a supervised training step.

    python benchmarks/streaming_metrics.py [--steps K] [--warmup W]

Arms, alternating round by round in one process, each adding the batch to its own state and computing the value:
    fused      ops.metric_auc_update: each prediction bucketed once, integer histograms, prefix sums, the value
    literal    TF 1.x metrics_impl's [T, N] comparison predictions > thresholds, summed per threshold in float32 (run only
               where T N <= 4e8)
    composed   torch.searchsorted + torch.bincount + cumsum, the counts rounded to float32 and added
Workloads: N = 61,952 (PPI: batch 512 x 121 labels), 20,480 (examples/gae: batch 1024, K = 10, 2K logits a row) and 2^20,
each at T = 5000 (upstream's default) and T = 200.  Predictions are sigmoid(sigmoid(logit)) of unit-normal logits, as
SuperviseModel feeds auc_score; labels are Bernoulli of the prediction.
A GATE first: from a zero state, every arm's four state vectors after one batch are bit-identical, else it aborts.
Then one SuperviseModel step (forward, backward, SGD) over SageEncoder([[0], [0]], [10, 10], 128) with a 121-wide label, on a
1M-node / 10M-edge R-MAT, at batch 512 with streaming=True ('auc') and with streaming=False (the per-batch f1).
Reported per arm: us per call and torch's allocator peak above the inputs; the card's name, power limit and max SM clock read
in the same run.  One JSON line on stdout.  It needs a GPU: without one it fails rather than measure anything else."""
import argparse

import harness
from harness import timed

WORKLOADS = [(61952, 5000), (61952, 200), (20480, 5000), (20480, 200), (1 << 20, 5000), (1 << 20, 200)]
LITERAL_MAX = 400_000_000


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--nodes", type=int, default=1_000_000)
    p.add_argument("--edges", type=int, default=10_000_000)
    p.add_argument("--model-steps", type=int, default=20)
    return p.parse_args(argv)


def thresholds(T, dev):
    """metrics_impl.auc's thresholds: Python doubles rounded once to float32"""
    t = [0.0 - 1e-7] + [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)] + [1.0 + 1e-7]
    return torch.tensor(t, dtype=torch.float64, device=dev).float()


def torch_value(tp, fn, tn, fp):
    eps = 1e-6
    rec = (tp + eps) / ((tp + fn) + eps)
    fpr = fp / ((fp + tn) + eps)
    return ((fpr[:-1] - fpr[1:]) * ((rec[:-1] + rec[1:]) / 2.0)).sum()


def literal_update(lab, p, thr, st):
    above = p[None, :] > thr[:, None]
    pos = (lab != 0)[None, :]
    st[0] += (above & pos).float().sum(1)
    st[1] += (~above & pos).float().sum(1)
    st[2] += (~above & ~pos).float().sum(1)
    st[3] += (above & ~pos).float().sum(1)
    return torch_value(*st)


def composed_update(lab, p, thr, st):
    T = thr.numel()
    pos = (lab != 0).long()
    b = torch.searchsorted(thr, p)                                 # #{i : t[i] < p}
    h = torch.bincount(b + (T + 1) * pos, minlength=2 * (T + 1)).view(2, T + 1)
    c = torch.cumsum(h, 1)[:, :T]                                  # at or below threshold i
    tot = h.sum(1, keepdim=True)
    st[0] += (tot[1] - c[1]).float()
    st[1] += c[1].float()
    st[2] += c[0].float()
    st[3] += (tot[0] - c[0]).float()
    return torch_value(*st)


def run(args):
    global torch
    import torch
    assert torch.cuda.is_available(), "streaming_metrics.py needs a GPU"
    import euler_b200 as eb
    from euler_b200 import ops
    dev = torch.device("cuda", 0)
    g = eb.Graph.rmat(args.nodes, args.edges, seed=42, feat_dim=128, device=0)
    eb.set_graph(g, rng="minstd", seed=5)
    out = {"gpu": harness.gpu_info(0), "workloads": []}
    gen = torch.Generator(device=dev).manual_seed(1)
    for N, T in WORKLOADS:
        x = torch.randn(N, generator=gen, device=dev)
        p = torch.sigmoid(torch.sigmoid(x))
        lab = (torch.rand(N, generator=gen, device=dev) < p).float()
        thr = thresholds(T, dev)
        arms, states = {}, {}

        def fused_arm(st):
            return lambda: ops.metric_auc_update(lab, p, *st)

        def torch_arm(fn, st):
            return lambda: fn(lab, p, thr, st)

        names = ["fused", "composed"] + (["literal"] if N * T <= LITERAL_MAX else [])
        for name in names:
            st = [torch.zeros(T, device=dev) for _ in range(4)]
            if name == "fused":
                st += [torch.zeros((), dtype=torch.int64, device=dev), torch.zeros((), device=dev)]
                arms[name] = fused_arm(st)
            else:
                arms[name] = torch_arm(literal_update if name == "literal" else composed_update, st)
            arms[name]()
            states[name] = torch.stack([s.clone() for s in st[:4]])
        for name in names:   # the gate: one batch from zero, every arm's state bit for bit
            if not torch.equal(states[name].view(torch.int32), states["fused"].view(torch.int32)):
                raise SystemExit("GATE FAILED: N=%d T=%d: the %s state differs from the fused one" % (N, T, name))
        res = timed(arms, args.steps, args.warmup)
        for r in res.values():
            r["us_per_call"] = r.pop("ms_per_call") * 1000.0
        out["workloads"].append({"N": N, "T": T, "arms": res, "literal_skipped": "literal" not in names})
    out["supervise_step"] = model_step(args, eb, dev)
    harness.emit(out)


def model_step(args, eb, dev):
    from euler_b200 import encoders
    from euler_b200.supervised import SuperviseModel

    def make(streaming):
        torch.manual_seed(0)
        enc = encoders.SageEncoder([[0], [0]], [10, 10], 128, 'mean', feature_idx=0, feature_dim=128, max_id=args.nodes,
                                   device="cuda")

        class Model(SuperviseModel):
            def __init__(self):
                super().__init__(0, 121, 'auc' if streaming else 'f1', dim=128, device="cuda", streaming=streaming)
                self.enc = enc

            def embed(self, n_id):
                return self.enc(n_id)

        m = Model()
        return m, torch.optim.SGD(m.parameters(), lr=0.01)

    models = {"streaming_auc": make(True), "per_batch_f1": make(False)}
    ids = torch.randint(1, args.nodes + 1, (512,), generator=torch.Generator(device=dev).manual_seed(3), device=dev)

    def step(pair):
        m, opt = pair
        opt.zero_grad()
        _, loss, _, metric = m(ids)
        loss.backward()
        opt.step()
        return metric

    res = timed({k: (lambda pr=pr: step(pr)) for k, pr in models.items()}, args.model_steps, 3)
    return {"batch": 512, "label_dim": 121, "arms": res}


if __name__ == "__main__":
    harness.divert_stdout()
    run(parse())
