"""Rows of every length class of the fanout sampler, bit-exact against the oracle.  k_sample keeps a row of at most SG edges in
its lane group's registers, stages a row of at most kStageF * SG cumulative weights (counted from the 16-byte boundary below the
row) in shared memory, and bisects every longer row in global memory.  The graph has hub rows of more than 2^16 edges and rows
at each class boundary, with both 16-byte alignments of the row start; the seeds include placeholders and absent ids.  Modes
0, 1 and 2; plain and batched; deep hops below and above kRepeatMinRows; hops whose live rows are all hubs or hold none; and
the 48-register build of the sampler (EU_SAMPLE_CTAS=5, the grid the benchmark runs) in a process of its own."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cases
import graphs
from oracle import pyoracle as po
from test_gpu_parity import _oracle_fanout

pytestmark = pytest.mark.gpu

REPEAT_MIN_ROWS = 1 << 17   # kRepeatMinRows
SG, STAGE_F = 16, 16        # lanes per row at fanout 10 (and T = 3), floats per lane of a staged tile
CAP = SG * STAGE_F          # a staged row holds at most CAP floats from the 16-byte boundary below it
HUB_DEG = 140_000           # > 2^16, and so is the half of it in edge type 0
T = 3
ETS = {0: [0], 1: [0, 2], 2: [0, 1, 2]}   # K == 1, 1 < K < T, every type


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def class_graph(seed=71, n=6000, n_hubs=3):
    """Rows of every class in random order (so row starts take every alignment), each row's edges split over T types;
    a tenth of all edges lead to a hub, so the deep hop's frontier is degree-biased as on a power-law graph."""
    rs = np.random.RandomState(seed)
    boundary = [SG - 1, SG, SG + 1, SG + 2] + list(range(CAP - 6, CAP + 3))
    lens = [HUB_DEG + k for k in range(n_hubs)] + boundary * 32 + [2 * CAP, 5000]
    rest = n - len(lens)
    lens += list(np.where(rs.rand(rest) < 0.15, 0, rs.geometric(1 / 40, size=rest)))
    lens = np.asarray(lens, np.int64)[rs.permutation(n)]
    deg = np.stack([rs.multinomial(L, [0.5, 0.3, 0.2]) for L in lens]).astype(np.int64)
    grp_ptr = np.zeros(n * T + 1, np.int64)
    grp_ptr[1:] = np.cumsum(deg.reshape(-1))
    E = int(grp_ptr[-1])
    ids = (1 + np.arange(n)).astype(np.uint64)
    hubs = ids[lens >= HUB_DEG]
    nbr = np.where(rs.rand(E) < 0.1, hubs[rs.randint(0, len(hubs), size=E)], ids[rs.randint(0, n, size=E)]).astype(np.uint64)
    for k in range(n * T):
        nbr[grp_ptr[k]:grp_ptr[k + 1]].sort()
    w = (1 + rs.randint(0, 100, size=E)).astype(np.float32) / np.float32(10)
    cum_w, grp_cum = po.build_cum(grp_ptr, w, n, T)
    g = dict(ids=ids, node_type=np.zeros(n, np.int32), node_w=np.ones(n, np.float32), T=T, grp_ptr=grp_ptr, nbr=nbr, w=w,
             cum_w=cum_w, grp_cum=grp_cum, feat=None, n_node_types=1)
    # the staged-tile boundary is met from both alignments of the row start (cum_w is allocated 16-byte aligned)
    base = grp_ptr[:-1:T][:n]
    for L in range(CAP - 2, CAP + 1):
        fits = (base % 4 + L <= CAP)[lens == L]
        assert fits.any() and not fits.all(), L
    return g, lens


def seeds_for(g, lens, B, seed, which="mixed"):
    rs = np.random.RandomState(seed)
    ids = g["ids"]
    if which == "hubs":
        pool = ids[lens >= HUB_DEG]
    elif which == "no_hubs":
        pool = ids[(lens > 0) & (lens <= CAP)]
    else:
        pool = ids
    s = pool[rs.randint(0, len(pool), size=B)].astype(np.int64)
    if which == "mixed":
        s[::5] = ids[lens >= HUB_DEG][rs.randint(0, 3, size=len(s[::5]))].astype(np.int64)
        s[3::11] = 0              # placeholder
        s[7::13] = 987654321      # absent
    return s


def _eq(ids, ws, ts, o, counts, what, b=None):
    o_ids, o_ws, o_ts = o
    for l in range(len(counts)):
        sel = (lambda x: x[b]) if b is not None else (lambda x: x)
        cases.eq(sel(ids[l + 1]).cpu().numpy(), o_ids[l], "%s ids hop %d" % (what, l))
        cases.eq(sel(ws[l]).cpu().numpy(), o_ws[l], "%s w hop %d" % (what, l))
        cases.eq(sel(ts[l]).cpu().numpy(), o_ts[l], "%s t hop %d" % (what, l))


_G = {}


def _graph():
    if "g" not in _G:
        g, lens = class_graph()
        _G["g"] = (g, lens, graphs.cuda_graph(g), graphs.oracle_graph(g))
    return _G["g"]


def run_plain(mode, deep_rows_above, seed=5):
    import euler_b200
    g, lens, gr, og = _graph()
    B = 9000 if deep_rows_above else 1500
    counts = [15, 10]
    assert (B * counts[0] >= REPEAT_MIN_ROWS) == deep_rows_above
    ets = [ETS[mode]] * 2
    seeds = seeds_for(g, lens, B, seed=mode)
    euler_b200.set_graph(gr, rng="minstd", seed=seed)
    ids, ws, ts = euler_b200.sample_fanout(seeds, ets, counts, -1)
    po.seed(seed)
    _eq(ids, ws, ts, _oracle_fanout(og, seeds, ets, counts), counts, "mode %d" % mode)


@pytest.mark.parametrize("deep_rows_above", [False, True])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_row_classes_plain(mode, deep_rows_above):
    run_plain(mode, deep_rows_above)


@pytest.mark.parametrize("mode", [0, 2])
def test_row_classes_batched(mode):
    """Three batches, each its own engine and dedup scope; the deep hop (3 x 3000 x 15 seeds) copies its duplicates."""
    import euler_b200
    g, lens, gr, og = _graph()
    nb, B, counts = 3, 3000, [15, 10]
    assert nb * B * counts[0] >= REPEAT_MIN_ROWS
    ets = [ETS[mode]] * 2
    euler_b200.set_graph(gr)
    ctx = euler_b200.Context(gr, "minstd", 1)
    seeds_e = [300 + 7 * b for b in range(nb)]
    ctx.set_engines(nb, seeds_e)
    nodes = np.stack([seeds_for(g, lens, B, seed=40 + b) for b in range(nb)])
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    ids, ws, ts = euler_b200.sample_fanout_batched(nodes, ets, counts, -1, ctx=ctx)
    for b in range(nb):
        po.seed(seeds_e[b])
        _eq(ids, ws, ts, _oracle_fanout(og, nodes[b], ets, counts), counts, "batch %d" % b, b=b)


@pytest.mark.parametrize("which", ["hubs", "no_hubs"])
@pytest.mark.parametrize("mode", [0, 2])
def test_hop_of_hubs_only_or_none(mode, which):
    """One hop whose rows that draw are all hubs of more than 2^16 edges, or all at most a staged tile long."""
    import euler_b200
    g, lens, gr, og = _graph()
    seeds = seeds_for(g, lens, 4000, seed=9, which=which)
    ets, counts = [ETS[mode]], [10]
    euler_b200.set_graph(gr, rng="minstd", seed=11)
    ids, ws, ts = euler_b200.sample_fanout(seeds, ets, counts, -1)
    po.seed(11)
    _eq(ids, ws, ts, _oracle_fanout(og, seeds, ets, counts), counts, which)


def test_row_classes_five_ctas_per_sm():
    """EU_SAMPLE_CTAS is read once per process: the 48-register build runs in a child process."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_sample_row_class_gpu as t\n"
            "for mode in (0, 1, 2):\n"
            "    t.run_plain(mode, True)\n"
            "print('ok')\n") % (here, os.path.dirname(here))
    env = dict(os.environ, EU_SAMPLE_CTAS="5")
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
