"""CPU checks of the row builders behind tests/test_walk_prefix_gpu.py (tests/walk_rows.py): the numpy replays equal the
literal sequential forms, and every family causes the prefix events it is built for, so that a generator cannot quietly
stop testing anything."""
import numpy as np
import pytest

import walk_rows as wr

F32 = np.float32


def test_prefix_is_the_sequential_f32_sum():
    rng = np.random.RandomState(0)
    v = (rng.rand(5000) * np.exp2(rng.randint(-30, 30, size=5000))).astype(F32)
    S, want = F32(0), np.empty(5000, F32)
    for k in range(5000):
        S = F32(S + v[k])
        want[k] = S
    assert np.array_equal(wr.prefix(v).view(np.uint32), want.view(np.uint32))


def test_build_weights_rule_equals_the_literal_merge():
    """The per-element multiset rule (used to replay the device's rows) against BuildWeights' two-pointer merge, on sorted
    multisets with repeats, the parent id among the children, and ids at both ends of int64."""
    rng = np.random.RandomState(1)
    edge = np.asarray([-2 ** 63, -2 ** 63 + 1, -1, 0, 1, 2 ** 63 - 2, 2 ** 63 - 1], np.int64)
    for it in range(300):
        pool = np.concatenate([edge, rng.randint(-20, 20, size=6)]).astype(np.int64)
        cn = np.sort(rng.choice(pool, rng.randint(0, 60)))
        pn = np.sort(rng.choice(pool, rng.randint(0, 45)))
        w = (1 + rng.randint(0, 50, size=len(cn))).astype(F32)
        parent = int(rng.choice(pool))
        p, q = (0.7, 3.0) if it % 2 else (2.0, 0.25)
        a = wr.build_weights(cn, w, pn, parent, p, q)
        b = wr.build_weights_literal(cn, w, pn, parent, p, q)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (cn, pn, parent)


def test_event_counter_on_hand_made_rows():
    t24 = F32(2 ** 24)
    ev = wr.prefix_events(np.asarray([t24, 1, 1, 3, 2], F32), start=1)
    assert ev["tie"] == 3 and ev["inexact"] == 3 and ev["binade"] == 0          # 2^24 + odd: halfway between evens
    ev = wr.prefix_events(np.asarray([1, 1, 8, 0, 0, 0, 2 ** -30], F32), start=1)
    assert ev["above"] == 1 and ev["binade"] == 2 and ev["zero_run"] == 3 and ev["inexact"] == 1 and ev["tie"] == 0
    ev = wr.prefix_events(np.asarray([0, 0, 1e-45, 1e-45, 1], F32), start=1)
    assert ev["tiny_S"] == 3 and ev["S_start"] == 0
    # iterations of the total pass: the head, then one per stretch of 1024 (CTA-256) / 4096 (CTA-1024) elements, or up
    # to the first exception and 96 more
    clean = np.concatenate([np.full(768, 1000, F32), np.full(8192, F32(2 ** -4))])    # S stays in [2^19, 2^20)
    assert wr.prefix_iterations(clean, 1024) == 3 and wr.prefix_iterations(clean, 256) == 9
    # S = k + 1 steps binade at 1024 and 2048: [768, 1119) ends 96 after the first, [1119, 2143) holds the second
    assert wr.prefix_iterations(np.ones(768 + 3000, F32), 256) == 5


@pytest.mark.parametrize("family,n", [(f, n) for f, ns in sorted(wr.FAMILY_LENGTHS.items()) for n in ns])
def test_family_causes_its_events(family, n):
    w, shared, p, q = wr.family_row(family, n)
    assert len(w) == n and w.dtype == F32 and (w >= 0).all()
    cum = wr.prefix(w)
    assert np.array_equal(wr.stored_weights(cum), w), "the chosen weights are not what the device reads back"
    if family in ("tie_heavy", "random_rounding", "zero_runs", "zero_head"):
        assert cum[-1] < 2 ** 24 and (w == np.round(w)).all()
    hg = wr.hub_graph([(w, shared)])
    wr.check_events(family, w, hg.step1_row(hg.hubs[0], p, q))


def test_tie_heavy_600k_row_reaches_the_checkpoint_cap():
    """The 600K-entry row: checkpoint stride 2 in the CTA-1024 kernel (1 + (n / 4096) / 128), and more than 2 * 256
    iterations of the total pass, so that the 256 checkpoints run out before the row does."""
    n = 600_000
    w, shared, p, q = wr.family_row("tie_heavy", n)
    assert wr.prefix(w)[-1] < 2 ** 24
    hg = wr.hub_graph([(w, shared)])
    v = hg.step1_row(hg.hubs[0], p, q)
    wr.check_events("tie_heavy", w, v)
    assert 1 + (n // 4096) // 128 == 2
    assert wr.prefix_iterations(v, 1024) > 2 * 256


def test_hub_graph_walkers_reach_their_hub_and_keep_the_subset():
    w, shared, p, q = wr.family_row("random_rounding", 2000)
    hg = wr.hub_graph([(w, shared)], extra_parent=[5, 2 ** 63 - 1])
    g = hg.build()
    h = hg.hubs[0]
    ids = g["ids"].view(np.int64)
    row = {int(i): r for r, i in enumerate(ids)}
    a = row[h["start"]]
    b, e = g["grp_ptr"][a], g["grp_ptr"][a + 1]
    an, aw = g["nbr"][b:e].view(np.int64), wr.stored_weights(g["cum_w"][b:e])
    assert (np.diff(an) >= 0).all() and aw[an == h["hub"]].tolist() == [1] and aw[an != h["hub"]].sum() == 0
    assert len(an) == 1 + shared.sum() + 2
    v = hg.step1_row(h, p, q)
    assert (v == w).sum() == shared.sum()          # multi-edges: the parent's copies keep as many entries, maybe others
    ua = hg.build(sort_u64=True)["nbr"][b:e]
    assert (ua[1:] >= ua[:-1]).all() and np.array_equal(np.sort(ua), np.sort(an.view(np.uint64)))


def test_walker_classes_follow_k_walk_plan():
    deg = [3, 0, 600, 20000, 512, 513, 16384, 16385, 10, 0, 7]
    cap = sum(deg[:6])
    assert list(wr.walker_classes(deg, cap)) == ["small", "dead", "big", "huge", "small", "big", "ovf", "ovf", "ovf",
                                                 "dead", "ovf"]
    assert list(wr.walker_classes(deg, 10 ** 9)) == ["small", "dead", "big", "huge", "small", "big", "big", "huge",
                                                     "small", "dead", "small"]
