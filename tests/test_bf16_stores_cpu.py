"""CPU: bfloat16 stores of ScalableSageEncoder / ScalableGCNEncoder without a device -- the constructors' refusals (before
any allocation), the stores' dtypes and shapes, their initialisation against the f32 encoder's, and the numpy restatement of
one bf16 accumulation against a hand-built case."""
import numpy as np
import pytest
import torch

import bf16_reference as bf
import sr_reference as sr
import store_reference as st
from euler_b200.encoders import ScalableGCNEncoder, ScalableSageEncoder

KW = dict(feature_idx=['f1'], feature_dim=[4], max_id=12, use_id=True, embedding_dim=3)
HUGE = dict(feature_idx=['f1'], feature_dim=[4], max_id=10 ** 13)   # stores of 10^13 rows: reaching an allocation fails


def _both(L, **kw):
    return [ScalableSageEncoder([0], 3, L, 8, **kw), ScalableGCNEncoder([0], L, 8, **kw)]


@pytest.mark.parametrize("cls,args", [(ScalableSageEncoder, ([0], 3, 2, 8)), (ScalableGCNEncoder, ([0], 2, 8))])
def test_constructor_refusals_before_allocation(cls, args):
    with pytest.raises(ValueError, match="fused=True"):
        cls(*args, store_dtype=torch.bfloat16, fused=False, **HUGE)
    for dt in (torch.float16, torch.float64, 'bfloat16', None):
        with pytest.raises(ValueError, match="store_dtype"):
            cls(*args, store_dtype=dt, **HUGE)
    for seed in (-1, 2 ** 64, 1.5, None):
        with pytest.raises(ValueError, match="store_seed"):
            cls(*args, store_dtype=torch.bfloat16, store_seed=seed, **HUGE)
    with pytest.raises(ValueError, match="float32 tables only"):       # the node-encoder tables still refuse bf16
        cls(*args, table_dtype=torch.bfloat16, store_dtype=torch.bfloat16, **HUGE)
    cls(*args, store_dtype=torch.bfloat16, store_seed=2 ** 64 - 1, **KW)   # the largest seed is accepted


@pytest.mark.parametrize("L", (1, 2, 3))
def test_store_dtypes_and_shapes(L):
    for dt in (torch.float32, torch.bfloat16):
        for enc in _both(L, store_dtype=dt, **KW):
            assert len(enc.stores) == len(enc.gradient_stores) == L - 1
            for s, g in zip(enc.stores, enc.gradient_stores):
                assert s.dtype == g.dtype == dt and s.shape == g.shape == (14, 8)
                assert s.is_contiguous() and g.is_contiguous() and not g.any()
            assert enc.store_sr_step.dtype == torch.int64 and enc.store_sr_step.shape == () and int(enc.store_sr_step) == 0
            assert enc.store_dtype == dt and enc.store_seed == 0
            state = enc.state_dict()
            assert not any(k.startswith(('store_', 'gradient_store_')) for k in state)   # non-persistent, as the f32 stores


def test_bf16_stores_are_the_f32_initialisation_rounded_to_nearest():
    for L in (2, 3):
        for cls, args in ((ScalableSageEncoder, ([0], 3, L, 8)), (ScalableGCNEncoder, ([0], L, 8))):
            encs = [cls(*args, store_init_maxval=0.5, store_dtype=dt, store_seed=7, generator=torch.Generator().manual_seed(5),
                        **KW) for dt in (torch.float32, torch.bfloat16)]
            for s32, s16 in zip(encs[0].stores, encs[1].stores):
                want = bf.round_bits(s32.numpy())
                assert np.array_equal(s16.view(torch.int16).numpy().view(np.uint16), want)
                assert torch.equal(s16, s32.to(torch.bfloat16))
            assert encs[1].store_seed == 7


def test_accumulate_restatement_against_a_hand_built_case():
    """Row 3 of a 5 x 4 store holds 1.0 (bf16 0x3F80, an ulp of 2^-7).  Ids [3, 1, 3] with count 1 and 'sum' add
    S_3 = g0 + g2 = 2^-9 + 0 = a quarter ulp to each column of row 3 (f32 bits 0x3F804000): it rounds up to 0x3F81 exactly
    when the low 16 bits of the random word are at least 0xC000, else stays 0x3F80.  Row 1 (0) gets -3 exactly; the other
    rows keep their bits."""
    G = np.zeros((5, 4), np.uint16)
    G[3] = 0x3F80
    G[0] = 0x1234
    grad = np.zeros((3, 4), np.float32)
    grad[0] = 2.0 ** -9
    grad[1] = -3.0
    seed, step, tensor = 0x1234_5678_9ABC_DEF0, 41, 2
    got = st.accumulate(G, [3, 1, 3], grad, 1, "sum", seed, step, tensor)
    words = sr.philox_bits(seed, step, tensor, 3 * 4 + np.arange(4))[0]
    want3 = np.where((words & 0xFFFF) >= 0xC000, 0x3F81, 0x3F80).astype(np.uint16)
    assert np.array_equal(got[3], want3)
    assert np.array_equal(bf.widen(got[1]), np.full(4, -3.0, np.float32))
    assert np.array_equal(got[[0, 2, 4]], G[[0, 2, 4]])
    # 'mean' over count 2 divides each entry by 2 first
    half = st.accumulate(G, [3, 3, 1, 1], grad[:2], 2, "mean", seed, step, tensor)
    assert np.array_equal(bf.widen(half[1]), np.full(4, -3.0, np.float32))   # (-3 / 2) + (-3 / 2), exact
    words = sr.philox_bits(seed, step, tensor, 12 + np.arange(4))[0]
    assert np.array_equal(half[3], np.where((words & 0xFFFF) >= 0xC000, 0x3F81, 0x3F80).astype(np.uint16))


def test_distinct_sums_order():
    """the chunk rule: 300 entries of one id sum the first 256 and the last 44 apart, then add the two sums from +0"""
    ids = np.zeros(300, np.int64)
    grad = np.ones((300, 1), np.float32)
    grad[0] = 2.0 ** 24                      # 2^24 + 1 rounds back to 2^24: the first chunk's sum is 2^24
    s = st.distinct_sums(ids, grad, 1, "sum")[0]
    assert s[0] == np.float32(2.0 ** 24) + np.float32(44.0)
    s = st.distinct_sums(np.zeros(1, np.int64), -np.zeros((1, 1), np.float32), 1, "sum")[0]
    assert s[0] == 0 and not np.signbit(s[0])  # +0 + -0 = +0
