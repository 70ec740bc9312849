"""The numpy restatements of tests/mp_ops_reference.py that test_mp_ops_gpu.py compares the kernels with, checked against
hand-worked vectors of tf_euler/kernels/scatter_op.cc (zero / -1e9 fill, then `out[idx[i]] += upd[i]` or
`if (upd > out) out = upd` for i ascending) and against that loop written out element by element."""
import numpy as np

import cases
import mp_ops_reference as ref

F = np.float32
NAN, INF = F(np.nan), F(np.inf)


def _col(*v):
    return np.asarray(v, np.float32).reshape(-1, 1)


def _loop(op, upd, idx, size):
    """scatter_op.cc's loop, one float32 element at a time"""
    out = np.full((size, upd.shape[1]), F(-1e9) if op == "max" else F(0), np.float32)
    for i in range(len(idx)):
        for j in range(upd.shape[1]):
            o, u = out[idx[i], j], upd[i, j]
            out[idx[i], j] = (u if u > o else o) if op == "max" else F(o + u)
    return out


def test_max_nan_never_wins():
    got = ref.scatter_max(_col(NAN, 1.5, NAN, NAN, -INF), [0, 0, 0, 1, 1], 3)
    cases.eq(got, _col(1.5, -1e9, -1e9), "NaN never wins")


def test_max_floor_is_minus_1e9():
    # -999999936 is the float32 just above -1e9
    got = ref.scatter_max(_col(-2e9, -INF, -1e9, -1e10, -999999936.0), [0, 0, 1, 2, 2], 4)
    cases.eq(got, _col(-1e9, -1e9, -999999936.0, -1e9), "values at or below -1e9 leave -1e9; empty rows hold it")


def test_max_keeps_the_first_of_equal_values():
    got = ref.scatter_max(_col(0.0, -0.0, -0.0, 0.0, 2.0, 2.0), [0, 0, 1, 1, 2, 2], 3)
    cases.eq(got, _col(0.0, -0.0, 2.0), "the first of +0.0 / -0.0 stays")
    assert not np.signbit(got[0, 0]) and np.signbit(got[1, 0])


def test_max_minus_zero_beats_negative_values():
    got = ref.scatter_max(_col(-0.0, -3.0, -1e-45, -0.0, -0.0), [0, 0, 1, 1, 2], 3)
    cases.eq(got, _col(-0.0, -0.0, -0.0), "-0.0 over negatives, subnormal ones included, and over -1e9")


def test_order_free_max_prefers_plus_zero_only_among_zeros():
    upd = _col(-0.0, 0.0, -0.0, -1.0, 0.0, -0.0, 3.0, -0.0)
    idx = [0, 0, 1, 1, 2, 2, 3, 3]
    cases.eq(ref.scatter_max(upd, idx, 4), _col(-0.0, -0.0, 0.0, 3.0), "reference")
    cases.eq(ref.scatter_max_order_free(upd, idx, 4), _col(0.0, -0.0, 0.0, 3.0), "order-free")


def test_add_and_mean():
    upd = _col(-0.0, 1.0, 2.0 ** -24, 2.0 ** -24, 1e-45, NAN, INF, -INF, INF, 1.0)
    idx = [0, 1, 1, 1, 2, 3, 4, 4, 5, 5]
    with np.errstate(invalid="ignore"):
        got = ref.scatter_add(upd, idx, 7)
    # 0 + -0.0 = +0.0; 1 + 2^-24 rounds to 1 twice (ties to even), where 2^-24 + 2^-24 first would not
    cases.eq(got[[0, 1, 2, 5, 6]], _col(0.0, 1.0, 1e-45, INF, 0.0), "add")
    assert np.isnan(got[3, 0]) and np.isnan(got[4, 0])
    mean = ref.scatter_mean(_col(1.0, 3.0, 5.0), [0, 1, 1], 3)
    # count 1: 1 + 1e-7 rounds up to 1 + 2^-23 in float32, so 1 / that rounds to 1 - 2^-23 (0x3f7ffffe), not to 1
    assert mean[0, 0].view(np.uint32) == 0x3f7ffffe
    cases.eq(mean[1:], _col(4.0, 0.0), "mean: count 2 + 1e-7 rounds to 2; an empty row is 0 / 1e-7 = +0.0")


def test_restatements_equal_the_element_loop():
    rs = np.random.RandomState(5)
    E, D, size = 300, 3, 23
    upd = (rs.randint(-4, 5, size=(E, D)) * 0.5).astype(np.float32)
    pool = np.asarray([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, -2e9, 1e7, 1e-3], np.float32)
    m = rs.rand(E, D) < 0.3
    upd[m] = rs.choice(pool, m.sum())
    for idx in (rs.randint(0, size - 3, size=E), np.sort(rs.randint(0, size, size=E)), np.zeros(E, np.int64)):
        with np.errstate(invalid="ignore"):
            for op in ("add", "max"):
                want = _loop(op, upd, idx, size)
                got = getattr(ref, "scatter_" + op)(upd, idx, size)
                assert np.array_equal(np.isnan(got), np.isnan(want)), op
                cases.eq(np.where(np.isnan(want), F(0), got), np.where(np.isnan(want), F(0), want), op)
            cases.eq(ref.scatter_mean(upd, idx, size), ref.scatter_add(upd, idx, size) / (_loop("add", np.ones((E, 1), np.float32), idx, size) + F(1e-7)), "mean")


def test_rank_in_row():
    assert ref.rank_in_row([3, 1, 3, 3, 0, 1]).tolist() == [0, 0, 1, 2, 0, 1]
    assert ref.rank_in_row([]).tolist() == []


def test_max_gradient_splits_ties():
    """mp_ops_test.py's 3x3 case: column 2 of rows 0 and 2 tie at 7"""
    upd = np.asarray([[1, 2, 7], [3, 4, 8], [5, 6, 7]], np.float32)
    idx = [1, 0, 1]
    out = ref.scatter_max(upd, idx, 2)
    g = ref.scatter_max_grad64(upd, idx, out, np.ones((2, 3)))
    assert g.tolist() == [[0, 0, .5], [1, 1, 1], [1, 1, .5]]


def test_fanout_aggregate_equals_whole_rows_then_scatter():
    rs = np.random.RandomState(8)
    feat = rs.uniform(-1, 1, size=(40, 11)).astype(np.float32)
    feat[::5, ::2] = -0.0
    rows = rs.randint(-1, 40, size=(17, 6))
    rows[3] = -1
    flat = rows.reshape(-1)
    seg = np.repeat(np.arange(17), 6)
    for dim in (1, 8, 11, 15):
        x = ref.whole_rows(feat, flat, dim)
        cases.eq(ref.fanout_aggregate(feat, rows, dim, True), ref.scatter_mean(x, seg, 17), "mean dim %d" % dim)
        cases.eq(ref.fanout_aggregate(feat, rows, dim, False), ref.scatter_add(x, seg, 17), "add dim %d" % dim)
    # two slots [3, 8]: get_dense_feature of slot 0 stops at column 3, the whole row does not
    x = ref.whole_rows(feat, flat, 8)
    d0 = ref.dense_feature(feat, [3, 8], flat, 0, 8)
    have = flat >= 0
    cases.eq(d0[:, :3], x[:, :3], "slot 0")
    assert not d0[:, 3:].any() and np.array_equal(x[have, 3:], feat[flat[have], 3:8])
    cases.eq(ref.dense_feature(feat, [3, 8], flat, 1, 10)[have], np.pad(feat[flat[have], 3:11], ((0, 0), (0, 2))), "slot 1")
    assert not ref.dense_feature(feat, [3, 8], flat, 2, 4).any()
