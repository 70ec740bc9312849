"""CPU: the numpy restatements of embedding_lookup_sparse that the sparse-embedding GPU tests compare against."""
import numpy as np
import pytest

import embedding_reference as er


@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_f32_order_is_within_rounding_of_f64(combiner):
    rng = np.random.RandomState(0)
    table = rng.standard_normal((50, 7)).astype(np.float32)
    bl = [list(rng.randint(0, 50, size=rng.randint(1, 40))) for _ in range(100)]
    a, b = er.lookup_f32(table, bl, combiner), er.lookup_f64(table, bl, combiner)
    assert a.dtype == np.float32
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-5)


def test_f32_order_is_left_to_right_from_the_first_row():
    table = np.asarray([[1.0], [2.0 ** -24], [2.0 ** -24]], np.float32)
    # (1 + 2^-24) + 2^-24 rounds to 1 twice (ties to even); the other order would give 1 + 2^-23
    assert er.lookup_f32(table, [[0, 1, 2]], "sum")[0, 0] == np.float32(1.0)
    assert er.lookup_f32(table, [[1, 2, 0]], "sum")[0, 0] == np.float32(1.0) + np.float32(2.0 ** -23)


def test_one_entry_bag_keeps_negative_zero():
    table = np.asarray([[-0.0, 0.0, 3.0]], np.float32)
    for c in er.COMBINERS:
        out = er.lookup_f32(table, [[0]], c)
        assert np.signbit(out[0, 0]) and not np.signbit(out[0, 1]), c   # -0 / 1 = -0; a sum from +0 would give +0
    assert np.signbit(er.lookup_f32(np.asarray([[-0.0]], np.float32), [[0, 0]], "sum")[0, 0])   # -0 + -0 = -0


def test_mean_and_sqrtn_divide_once():
    table = np.asarray([[1.0], [1.0], [1.0]], np.float32)
    assert er.lookup_f32(table, [[0, 1, 2]], "mean")[0, 0] == np.float32(3.0) / np.float32(3.0)
    assert er.lookup_f32(table, [[0, 1, 2]], "sqrtn")[0, 0] == np.float32(3.0) / np.sqrt(np.float32(3.0))


def test_bags_default_entry_rules():
    ids = np.asarray([0, 5, 9], np.uint64)
    S = 2
    # node 0: slot 0 = [4, 1], slot 1 empty; node 5: slot 0 empty, slot 1 = [2]; node 9: both empty
    ptr = np.asarray([0, 2, 2, 2, 3, 3, 3], np.int64)
    val = np.asarray([4, 1, 2], np.uint64)
    got = er.bags(ids, ptr, val, S, [0, 5, 9, 77, 0], 0, 8)
    assert got == [[4, 1], [8], [8], [8], [4, 1]]             # stored order; empty slot, absent id -> the default
    assert er.bags(ids, ptr, val, S, [5, 0], 1, 8) == [[2], [8]]
    assert er.bags(ids, ptr, val, S, [0], 3, 8) == [[8]]       # unknown slot


def test_grad_f64_scales_by_the_combiner():
    g = np.asarray([[1.0, 2.0], [4.0, 8.0]])
    bl = [[0, 1, 1, 1], [1]]
    np.testing.assert_allclose(er.grad_f64(g, bl, 3, "sum"), [[1, 2], [7, 14], [0, 0]])
    np.testing.assert_allclose(er.grad_f64(g, bl, 3, "mean"), [[0.25, 0.5], [4.75, 9.5], [0, 0]])
    np.testing.assert_allclose(er.grad_f64(g, bl, 3, "sqrtn"), [[0.5, 1], [5.5, 11], [0, 0]])


def test_sample_fanout_with_feature_packing_rule():
    """engine ids vs TF-packed ids on hand-built hops where node 0 exists and is drawn"""
    eng = np.asarray([[5, 0, 7],     # node 0 drawn second: the row is copied, 0 included
                      [0, 4, 4],     # node 0 drawn first: packed as the default fill although 4 and 4 are real draws
                      [0, 0, 0],     # no result (absent node / no edge): the default fill
                      [3, 3, 0]])
    packed, kept = er.tf_pack(eng, -1)
    assert packed.tolist() == [[5, 0, 7], [-1, -1, -1], [-1, -1, -1], [3, 3, 0]]
    assert kept.tolist() == [True, False, False, True]
    # the features of the packed-away row are those of its engine ids, not of default_node
    ids = np.asarray([0, 3, 4, 5, 7], np.uint64)
    ptr = np.asarray([0, 1, 1, 2, 4, 5], np.int64)            # one slot: node 0 -> [9], 3 -> [], 4 -> [2], 5 -> [6, 1], 7 -> [8]
    val = np.asarray([9, 2, 6, 1, 8], np.uint64)
    assert er.bags(ids, ptr, val, 1, eng[1], 0, 11) == [[9], [2], [2]]
    assert er.bags(ids, ptr, val, 1, packed[1], 0, 11) == [[11], [11], [11]]
