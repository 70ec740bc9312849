"""Exact-mode node2vec (random_walk with p, q != 1, euler_b200/csrc/walk.cu) against the oracle's op_random_walk, bit for
bit, with the engine's draw count checked after every call.  The rows are built (tests/walk_rows.py) so that the
sequential f32 prefix of CompactWeightedCollection::Init ties, rounds, changes binade, starts from zero or stays
subnormal after the serial head, at every row length where the step switches kernels: the warp chain (<= 512), the
CTA-256 and CTA-1024 exact prefixes (block_exact_prefix), the self-contained warp path for rows that do not fit in the
weight scratch V, and the sequential k_walk_step (unsorted adjacency or several edge types per step)."""
import functools

import numpy as np
import pytest
import torch

import cases
import walk_rows as wr
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

V_BIG = 1 << 28         # EU_WALK_V_ELEMS for the tests that keep every walker in V (1 GiB)
I63 = 2 ** 63 - 1
ABSENT = 987654321012   # ids without a row
EMPTY = 424242          # a node with a row and no neighbors


@pytest.fixture(autouse=True)
def _sync_after():
    yield
    torch.cuda.synchronize()


def _backends(g, monkeypatch, v_elems):
    """Device and oracle on g; the device context is created fresh, so its weight scratch V holds v_elems floats."""
    monkeypatch.setenv("EU_WALK_V_ELEMS", str(v_elems))
    return cases.CudaBackend(g, g["ids"]), cases.OracleBackend(g, g["ids"])


def _walk(be, ob, seeds, wet, p, q, seed, what):
    wet = np.asarray(wet, np.int32)
    be.seed(seed)
    ob.seed(seed)
    got = be.op_random_walk(seeds, wet, p, q, -1)
    cases.eq(got, ob.op_random_walk(seeds, wet, p, q, -1), what)
    assert be.draws() == ob.draws(), what
    return got


def _both_kernels(be, ob, seeds, L, p, q, seed, what):
    """[[0]] per step takes the parallel kernels; [[0, 8]] lists the same neighbors (type 8 does not exist and is skipped)
    but K = 2 takes the sequential k_walk_step.  Both against the oracle and so against each other."""
    a = _walk(be, ob, seeds, [[0]] * L, p, q, seed, what + " parallel")
    b = _walk(be, ob, seeds, [[0, 8]] * L, p, q, seed, what + " sequential")
    cases.eq(a, b, what + " parallel vs sequential")
    return a


def _starts(hg, per, rng, dead=()):
    """per walkers at every hub's start node, with the dead ids spread among them, shuffled"""
    seeds = np.concatenate([np.repeat([h["start"] for h in hg.hubs], per), np.asarray(dead, np.int64)]).astype(np.int64)
    rng.shuffle(seeds)
    return seeds


def _step1_classes(hg, seeds, cap_v):
    """k_walk_plan's class of every walker at step 1, when the walkers started at a hub's start node sit at the hub"""
    deg = {h["start"]: h["n"] for h in hg.hubs}
    return wr.walker_classes([deg.get(int(s), 0) for s in seeds], cap_v)


def _family_graph(family, lengths, seed=0):
    rows = [wr.family_row(family, n) for n in lengths]
    hg = wr.hub_graph([(w, sh) for w, sh, _, _ in rows], seed=seed)
    p, q = rows[0][2], rows[0][3]
    for h, (w, _, _, _) in zip(hg.hubs, rows):
        if h["n"] in wr.FAMILY_LENGTHS[family]:
            wr.check_events(family, w, hg.step1_row(h, p, q))
    hg.add_row(EMPTY, [], [])
    return hg, p, q


@functools.lru_cache(maxsize=None)
def _boundary_graph(family):
    hg, p, q = _family_graph(family, wr.BOUNDARY_LENGTHS, seed=5)
    return hg, hg.build(), p, q


# ------------------------------------------------------------------------------------------------------- families
@pytest.mark.parametrize("family", sorted(wr.FAMILY_LENGTHS))
def test_rounding_rows_vs_oracle(family, monkeypatch):
    """Tie-heavy, zero-laden, wide-exponent, subnormal and randomly rounding rows past the serial head, in the CTA-256
    and CTA-1024 prefixes and in k_walk_step."""
    hg, p, q = _family_graph(family, wr.FAMILY_LENGTHS[family], seed=1)
    be, ob = _backends(hg.build(), monkeypatch, V_BIG)
    seeds = _starts(hg, 40, np.random.RandomState(2), dead=[ABSENT, EMPTY, -1])
    want = {"small" if n <= wr.K_WALK_BIG else "big" if n <= wr.K_WALK_HUGE else "huge" for n in wr.FAMILY_LENGTHS[family]}
    assert set(_step1_classes(hg, seeds, V_BIG)) - {"dead"} == want
    got = _both_kernels(be, ob, seeds, 4, p, q, 3, family)
    other = (2.0, 0.5) if (p, q) != (2.0, 0.5) else (0.7, 3.0)
    _both_kernels(be, ob, seeds, 4, *other, 4, family + " p=%s q=%s" % other)
    if family != "all_zero":   # the walks reach different entries of every row (wide rows: mostly their last jump)
        for h in hg.hubs:
            assert len(np.unique(got[seeds == h["start"], 2])) > (1 if family == "wide_exponent" else 5)
    else:                      # a zero row falls through to its last entry
        for h in hg.hubs:
            assert (got[seeds == h["start"], 2] == h["nbr"][-1]).all()


@pytest.mark.parametrize("family", ["tie_heavy", "random_rounding"])
def test_boundary_row_lengths_vs_oracle(family, monkeypatch):
    """Row lengths 1 .. 70K at every boundary of the step kernels: 32-wide warp chunks, warp / CTA-256 / CTA-1024, the
    768-entry serial head and one CTA-256 / CTA-1024 iteration after it."""
    hg, g, p, q = _boundary_graph(family)
    be, ob = _backends(g, monkeypatch, V_BIG)
    seeds = _starts(hg, 12, np.random.RandomState(6), dead=[ABSENT, EMPTY, -1, 0] * 3)
    assert {"small", "big", "huge", "dead"} == set(_step1_classes(hg, seeds, V_BIG))
    for p2, q2 in [(p, q), (0.7, 3.0) if (p, q) != (0.7, 3.0) else (2.0, 0.5)]:
        _both_kernels(be, ob, seeds, 4, p2, q2, 7, "%s boundaries p=%s q=%s" % (family, p2, q2))


def test_600k_tie_heavy_row_runs_out_of_checkpoints(monkeypatch):
    """A 600K-entry tie-heavy row: checkpoint stride 2 and more than 512 iterations, so the select pass resumes from the
    last of the 256 checkpoints; a few hundred walkers draw on it at once, all in V."""
    w, sh, p, q = wr.family_row("tie_heavy", 600_000)
    hg = wr.hub_graph([(w, sh)], seed=8)
    v = hg.step1_row(hg.hubs[0], p, q)
    wr.check_events("tie_heavy", w, v)
    assert wr.prefix_iterations(v, 1024) > 2 * 256
    be, ob = _backends(hg.build(), monkeypatch, V_BIG)
    seeds = np.full(300, hg.hubs[0]["start"], np.int64)
    assert (_step1_classes(hg, seeds, V_BIG) == "huge").all()
    got = _walk(be, ob, seeds, [[0]] * 4, p, q, 9, "600K tie-heavy")
    assert len(np.unique(got[:, 2])) > 100
    _walk(be, ob, seeds, [[0]] * 4, 0.7, 3.0, 10, "600K p=0.7 q=3")


# ------------------------------------------------------------------------------------------- overflow and batches
def _mixed_graph():
    rows = [wr.family_row("random_rounding", 100), wr.family_row("tie_heavy", 3000), wr.family_row("tie_heavy", 20000),
            wr.family_row("zero_head", 5000)]
    hg = wr.hub_graph([(w, sh) for w, sh, _, _ in rows], seed=11)
    hg.add_row(EMPTY, [], [])
    return hg


@functools.lru_cache(maxsize=None)
def _mixed():
    hg = _mixed_graph()
    return hg, hg.build()


@pytest.mark.parametrize("B", [1, 1023, 1025, 5000])
def test_overflow_path_and_batch_bookkeeping(B, monkeypatch):
    """V ends mid-batch: the walkers before the boundary take the three V kernels, every live one after it the
    self-contained warp path, whatever its row length; dead walkers, absent ids and empty rows are interleaved.
    B around the 1024 threads of k_walk_plan."""
    hg, g = _mixed()
    rng = np.random.RandomState(B)
    starts = np.asarray([h["start"] for h in hg.hubs], np.int64)
    pool = np.concatenate([np.repeat(starts, 3), [ABSENT, EMPTY, -1]]).astype(np.int64)
    seeds = rng.choice(pool, B)
    seeds[0] = starts[2]
    deg = {h["start"]: h["n"] for h in hg.hubs}
    d1 = np.asarray([deg.get(int(s), 0) for s in seeds])
    cap = max(1, int(d1[:B // 2 + 1].sum()) - (1 if B == 1 else 0))
    cls = _step1_classes(hg, seeds, cap)
    if B == 1:
        assert list(cls) == ["ovf"]
    else:
        assert {"small", "big", "huge", "ovf", "dead"} == set(cls)
        assert set(d1[cls == "ovf"]) == {h["n"] for h in hg.hubs}     # every row length overflows too
    be, ob = _backends(g, monkeypatch, cap)
    for p, q, s in [(0.7, 3.0, 12), (2.0, 0.5, 13)]:
        _walk(be, ob, seeds, [[0]] * 4, p, q, s, "B=%d cap=%d p=%s q=%s" % (B, cap, p, q))


# --------------------------------------------------------------------------------------------------------- id edges
def _i63_graph():
    """Hubs whose lists end with id 2^63-1 (several copies), biased against parent lists whose last 32-entry chunk is
    partial and that do not hold 2^63-1, weighted so that dividing those entries by q or not moves half the draws."""
    rng = np.random.RandomState(14)
    hg = wr.HubGraph(15)
    specs = [(60, 3, 36, ()), (39, 1, 1, (10 ** 7 + 100,)), (2000, 4, 500, ()), (20000, 2, 5001, ())]
    for k, (n, copies, n_shared, extra) in enumerate(specs):
        lo = (k + 1) * 10 ** 7
        body = np.arange(lo + 1, lo + n + 1, dtype=np.int64) if k == 1 else wr.hub_neighbors(n, rng, lo)
        nbr = np.concatenate([body, np.full(copies, I63, np.int64)])
        w = np.concatenate([1 + rng.randint(0, 10, size=n), np.zeros(copies)]).astype(np.float32)
        shared = np.zeros(n + copies, bool)
        shared[np.sort(rng.choice(n, n_shared, replace=False)) if k != 1 else [n - 1]] = True
        start = 10 ** 9 + 2 * k + 1
        others = wr.build_weights(body, w[:n], np.sort(body[shared[:n]]), start, 2.0, 3.0).sum()
        w[n:] = np.float32(max(1, int(3 * others / copies)))
        hg.add_hub(10 ** 9 + 2 * k, start, nbr, w, shared, extra_parent=extra)
        pn = hg.hubs[-1]["pn"]
        assert len(pn) % 32 != 0 and I63 not in pn
    return hg


@pytest.mark.parametrize("v_elems", [V_BIG, 1], ids=["in_V", "overflow"])
def test_max_int64_neighbor_id(v_elems, monkeypatch):
    """A neighbor id 2^63-1 is biased like any other: the parent's list does not hold it, so it is divided by q."""
    hg = _i63_graph()
    be, ob = _backends(hg.build(), monkeypatch, v_elems)
    seeds = _starts(hg, 400, np.random.RandomState(16), dead=[ABSENT, -1])
    cls = set(_step1_classes(hg, seeds, v_elems)) - {"dead"}
    assert cls == ({"ovf"} if v_elems == 1 else {"small", "big", "huge"})
    for p, q, s in [(2.0, 3.0, 17), (0.7, 0.25, 18)]:
        got = _walk(be, ob, seeds, [[0]] * 3, p, q, s, "2^63-1 p=%s q=%s v=%d" % (p, q, v_elems))
        if q == 3.0:   # the weights were chosen for this q: about half the step-1 draws land on 2^63-1
            assert 0.2 < (got[:, 2] == I63).mean() < 0.8


@pytest.mark.parametrize("order", ["int64", "uint64"])
def test_ids_at_and_above_2_63(order, monkeypatch):
    """Ids >= 2^63 (negative as int64) among positive ones.  Adjacency in int64 order is what the parallel kernels
    merge; adjacency in uint64 order is not sorted for them and goes to k_walk_step, whose merge compares as int64
    like BuildWeights."""
    rng = np.random.RandomState(19)
    hg = wr.HubGraph(20)
    for k, n in enumerate([300, 3000, 20000]):
        w, sh, _, _ = wr.family_row("random_rounding", n)
        nbr = np.sort(np.concatenate([wr.hub_neighbors(n // 2, rng, -2 ** 62 + (k + 1) * 10 ** 7),
                                      wr.hub_neighbors(n - n // 2, rng, (k + 1) * 10 ** 7)]))
        nbr[-1] = I63
        nbr[0] = -2 ** 63
        hg.add_hub(-2 ** 61 + 2 * k, -2 ** 61 + 2 * k + 1, nbr, w, sh)
    g = hg.build(sort_u64=order == "uint64")
    nb = g["nbr"].view(np.int64)
    in_order = all((np.diff(nb[b:e]) >= 0).all() for b, e in zip(g["grp_ptr"][:-1], g["grp_ptr"][1:]))
    assert in_order == (order == "int64")
    be, ob = _backends(g, monkeypatch, V_BIG)
    seeds = _starts(hg, 100, np.random.RandomState(21), dead=[ABSENT, 2 ** 63 - 2, -2])
    for p, q, s in [(0.7, 3.0, 22), (2.0, 0.5, 23)]:
        got = _walk(be, ob, seeds, [[0]] * 4, p, q, s, "ids >= 2^63 %s order p=%s q=%s" % (order, p, q))
        assert (got[:, 2] < 0).mean() > 0.2 and (got[:, 2] > 0).mean() > 0.2


# ------------------------------------------------------------------------------------------------------- philox
def test_philox_exact_mode_parallel_kernels_equal_the_sequential_one(monkeypatch):
    """EU_RNG_PHILOX with the rejection mode switched off: the parallel kernels and k_walk_step draw the same
    philox_uniform2(walker, step) and must pick the same entries (the oracle has no counter-based stream)."""
    import euler_b200
    hg, g, _, _ = _boundary_graph("tie_heavy")
    monkeypatch.setenv("EU_WALK_FAST_OFF", "1")
    monkeypatch.setenv("EU_WALK_V_ELEMS", str(V_BIG))
    be = cases.CudaBackend(g, g["ids"])
    euler_b200.set_graph(be.graph, rng="philox", seed=31)
    seeds = _starts(hg, 12, np.random.RandomState(32), dead=[ABSENT, EMPTY, -1])
    for p, q in [(2.0, 0.5), (0.7, 3.0)]:
        be.seed(33)
        a = be.op_random_walk(seeds, [[0]] * 4, p, q, -1)
        be.seed(33)
        b = be.op_random_walk(seeds, [[0, 8]] * 4, p, q, -1)
        cases.eq(a, b, "philox exact p=%s q=%s parallel vs sequential" % (p, q))
        assert len(np.unique(a[:, 2])) > 50


# ----------------------------------------------------------------------------------------------------------- R-MAT
def test_rmat_hubs_vs_oracle():
    """R-MAT 2M nodes / 20M edges: walkers at the highest-degree rows (over 16384 entries: the CTA-1024 prefix) and at
    random nodes, p = 0.7, q = 3, against the oracle on the exported graph."""
    import euler_b200
    n, E = 2_000_000, 20_000_000
    gr = euler_b200.Graph.rmat(n, E)
    ex = gr.export(with_feat=False)
    deg = np.diff(ex["grp_ptr"])
    assert deg.max() > wr.K_WALK_HUGE
    og = po.OracleGraph(ex["ids"], ex["node_type"], ex["node_w"], 1, ex["grp_ptr"], ex["nbr"], ex["cum_w"],
                        np.zeros(n, np.float32))
    top = ex["ids"][np.argsort(-deg, kind="stable")[:64]].astype(np.int64)
    seeds = np.concatenate([top, np.random.RandomState(40).randint(1, n + 1, size=1000)]).astype(np.int64)
    euler_b200.set_graph(gr, rng="minstd", seed=41)
    euler_b200.seed(42)
    po.seed(42)
    got = euler_b200.random_walk(seeds, [[0]] * 4, 0.7, 3.0, -1).cpu().numpy()
    cases.eq(got, og.op_random_walk(seeds, np.asarray([[0]] * 4, np.int32), 0.7, 3.0, -1), "R-MAT node2vec")
    assert euler_b200.context().draws() == po.draws()
