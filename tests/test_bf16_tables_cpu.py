"""CPU: the numpy restatement of the stochastic rounding that writes trained bfloat16 tables (sr_reference.sr_bits, the
device's sr_st), its random bits, and the Python-side refusals of bf16 tables that need no device."""
import numpy as np
import pytest
import torch

import bf16_reference as bf
import graphs  # noqa: F401  (sys.path)
import sr_reference as sr


def _values(rng, n=1 << 16):
    """random f32 bit patterns of every exponent, the special values, and exact ties at both kept parities"""
    u = rng.randint(0, 2 ** 32, size=n, dtype=np.uint64).astype(np.uint32)
    ties = (rng.randint(0, 2 ** 16, size=256).astype(np.uint32) << 16) | 0x8000
    return np.concatenate([u.view(np.float32), bf.special_values(), ties.view(np.float32)])


def test_zero_bits_truncate_toward_zero():
    x = _values(np.random.RandomState(0))
    got = sr.sr_bits(x, np.zeros(x.size, np.uint32))
    fin = np.isfinite(x)
    np.testing.assert_array_equal(got[fin], (x[fin].view(np.uint32) >> 16).astype(np.uint16))
    w = bf.widen(got[fin])
    assert np.all(np.abs(w) <= np.abs(x[fin]))


def test_half_bits_round_to_nearest_ties_away():
    x = _values(np.random.RandomState(1))
    got = sr.sr_bits(x, np.full(x.size, 0x8000, np.uint32))
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    fin = np.isfinite(x)
    tie = fin & ((x.view(np.uint32) & 0xFFFF) == 0x8000)
    assert tie.sum() >= 256
    np.testing.assert_array_equal(got[fin & ~tie], want[fin & ~tie])
    # an exact tie rounds away from zero: the magnitude's upper half plus one
    np.testing.assert_array_equal(got[tie], ((x[tie].view(np.uint32) >> 16) + 1).astype(np.uint16))


@pytest.mark.parametrize("r", [0, 0x8000, 0xFFFF, 0xFFFFFFFF])
def test_nan_and_inf_pass_through(r):
    x = bf.special_values()
    got = sr.sr_bits(x, np.full(x.size, r, np.uint32))
    w = bf.widen(got)
    nan = np.isnan(x)
    assert np.all(np.isnan(w[nan]))
    np.testing.assert_array_equal(np.signbit(w[nan]), np.signbit(x[nan]))
    inf = np.isinf(x)
    np.testing.assert_array_equal(w[inf], x[inf])


def test_finite_values_stay_between_their_neighbours():
    x = _values(np.random.RandomState(2))
    x = x[np.isfinite(x)]
    r = np.random.RandomState(3).randint(0, 2 ** 32, size=x.size, dtype=np.uint64).astype(np.uint32)
    got = sr.sr_bits(x, r)
    lo = (x.view(np.uint32) >> 16).astype(np.uint16)
    exact = (x.view(np.uint32) & 0xFFFF) == 0
    np.testing.assert_array_equal(got[exact], lo[exact])
    assert np.all((got[~exact] == lo[~exact]) | (got[~exact] == lo[~exact] + 1))


@pytest.mark.parametrize("value", [np.float32(0.1), np.float32(-3.3e-5), np.float32(1 + 2 ** -10), np.float32(6.0e4)])
def test_mean_over_keys_is_unbiased(value):
    """the mean of the widened roundings of one value over 2^16 elements' keys lies within 4 standard errors of it"""
    n = 1 << 16
    words = sr.philox_bits(12345, 7, 2, np.arange(n))
    w = bf.widen(sr.sr_bits(np.full(n, value, np.float32), words[0])).astype(np.float64)
    lo = bf.widen(np.uint16(np.float32(value).view(np.uint32) >> 16)).astype(np.float64)
    ulp = abs(float(bf.widen(np.uint16((np.float32(value).view(np.uint32) >> 16) + 1))) - float(lo))
    p = abs(float(value) - float(lo)) / ulp
    se = ulp * np.sqrt(p * (1 - p) / n)
    assert abs(w.mean() - float(value)) <= 4 * se + 1e-12 * abs(float(value))


def test_philox_words_are_distinct_per_key():
    a = sr.philox_bits(1, 0, 0, np.arange(1000))
    for other in (sr.philox_bits(2, 0, 0, np.arange(1000)), sr.philox_bits(1, 1, 0, np.arange(1000)),
                  sr.philox_bits(1, 0, 1, np.arange(1000)), sr.philox_bits(1, 0, 0, np.arange(1000, 2000))):
        assert np.mean(a[0] == other[0]) < 0.01
    assert len(np.unique(a[0] & 0xFFFF)) > 900


def test_refusals_without_a_device():
    from euler_b200 import optimizers, unsupervised
    t = torch.nn.Parameter(torch.zeros(4, 4, dtype=torch.bfloat16), requires_grad=False)
    for name in ('sgd', 'momentum', 'adagrad', 'adam'):
        with pytest.raises(ValueError, match="fused"):
            optimizers.get(name)([t], 0.1, fused=False)
    with pytest.raises(ValueError, match="seed"):
        optimizers.get('adam')([t], 0.1, seed=-1)
    with pytest.raises(ValueError, match="fused=True"):
        unsupervised.DeepWalk(0, 0, 10, 4, table_dtype=torch.bfloat16, fused=False)
    with pytest.raises(ValueError, match="table_dtype"):
        unsupervised.DeepWalk(0, 0, 10, 4, table_dtype=torch.float16)
    assert torch.equal(t, torch.zeros(4, 4, dtype=torch.bfloat16))
    o = optimizers.get('adam')([t], 0.1, seed=5)
    assert o.sr_step is not None and int(o.sr_step) == 0 and 'sr_step' in o.state_dict()
    f = torch.nn.Parameter(torch.zeros(3))
    assert optimizers.get('adam')([f], 0.1).sr_step is None   # an f32 optimizer keeps no counter
