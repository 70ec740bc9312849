"""CPU: the numpy restatement of the stochastic rounding that writes trained bfloat16 tables (sr_reference.sr_bits, the
device's sr_st), its random bits, and the Python-side refusals of bf16 tables that need no device."""
import numpy as np
import pytest
import torch

import bf16_reference as bf
import graphs  # noqa: F401  (sys.path)
import optim_reference as ref
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


def _philox4x32_10(ctr, key):
    """Philox4x32-10 of one counter (four uint32 words) and key (two), in Python integers: Random123's round as written"""
    m = 0xFFFFFFFF
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & m, p1 & m, ((p0 >> 32) ^ c3 ^ k1) & m, p0 & m
        k0, k1 = (k0 + 0x9E3779B9) & m, (k1 + 0xBB67AE85) & m
    return [c0, c1, c2, c3]


# Random123's published known answers for Philox4x32-10 (kat_vectors): counter, key, result
_PHILOX_KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", _PHILOX_KAT)
def test_philox_matches_the_published_known_answers(ctr, key, want):
    """philox_bits' counter is (element lo, element hi, step, tensor) and its key (seed lo, seed hi)"""
    element = ctr[0] | (ctr[1] << 32)
    seed = key[0] | (key[1] << 32)
    got = sr.philox_bits(seed, ctr[2], ctr[3], np.array([element], np.uint64))
    assert [int(w[0]) for w in got] == list(want)
    assert _philox4x32_10(ctr, key) == list(want)


def test_philox_element_high_word_is_counter_word_one():
    """elements at and past 2^32, where the counter's second word is non-zero, against counters built by hand"""
    seed, step, tensor = 0xDEADBEEF12345678, 5, 2
    elems = [2 ** 32 - 1, 2 ** 32, 2 ** 32 + 127, 3 * 2 ** 32 + 5, (2 ** 25 + 2 ** 13 - 1) * 128 + 127, 2 ** 63 + 9]
    got = sr.philox_bits(seed, step, tensor, np.array(elems, np.uint64))
    for i, e in enumerate(elems):
        want = _philox4x32_10((e & 0xFFFFFFFF, e >> 32, step, tensor), (seed & 0xFFFFFFFF, seed >> 32))
        assert [int(w[i]) for w in got] == want, hex(e)
    lo = sr.philox_bits(seed, step, tensor, np.array([e & 0xFFFFFFFF for e in elems[1:4]], np.uint64))
    assert all(np.all(a != b) for a, b in zip(lo, [w[1:4] for w in got]))   # word 1 changes every word of the block


@pytest.mark.parametrize("name", ['momentum', 'adagrad', 'adam'])
def test_step_on_picked_rows_is_the_step_on_the_whole_table(name):
    """step(rows=...) over picked rows of a table gives those rows' bits of the step over the whole table; with rows far
    past 2^32 / D every element draws from philox_bits at rows[i] D + d"""
    rng = np.random.RandomState(20 + len(name))
    N, D = 300, 5
    whole = [bf.round_bits(np.abs(rng.randn(N, D)).astype(np.float32) + np.float32(0.1)) for _ in range(3 if name == 'adam' else 2)]
    g_rows = np.unique(rng.randint(0, N, size=40))
    g_vals = rng.randn(g_rows.size, D).astype(np.float32)
    pick = np.unique(np.concatenate([g_rows[::2], rng.randint(0, N, size=30)]))
    picked = [t[pick].copy() for t in whole]
    local = np.searchsorted(pick, g_rows[np.isin(g_rows, pick)])
    vals = g_vals[np.isin(g_rows, pick)]
    adams = [ref.Adam(0.01) if name == 'adam' else None for _ in range(2)]
    sr.step(name, whole, (g_rows, g_vals), 9, 3, 1, 0.1, adam=adams[0], momentum=0.9)
    sr.step(name, picked, (local, vals), 9, 3, 1, 0.1, adam=adams[1], momentum=0.9, rows=pick)
    for w, p in zip(whole, picked):
        np.testing.assert_array_equal(w[pick], p)
    # rows whose elements lie past 2^32: the rounding uses the words of their global element indices
    big = np.array([0, 2 ** 32 // D - 1, 2 ** 32 // D, 2 ** 33 // D + 7], np.int64)
    tabs = [bf.round_bits(np.abs(rng.randn(big.size, D)).astype(np.float32) + np.float32(0.1)) for _ in whole]
    f = [bf.widen(t).reshape(big.size, D) for t in tabs]
    grad = (np.arange(big.size), rng.randn(big.size, D).astype(np.float32))
    adam = ref.Adam(0.01) if name == 'adam' else None
    sr.step(name, tabs, grad, 9, 3, 1, 0.1, adam=adam, momentum=0.9, rows=big)
    if name == 'adam':
        ref.Adam(0.01).update(f[0], f[1], f[2], grad)
    elif name == 'adagrad':
        ref.adagrad(f[0], f[1], grad, 0.1)
    else:
        ref.momentum(f[0], f[1], grad, 0.1, 0.9)
    for w, (t, v) in enumerate(zip(tabs, f)):
        for i, r in enumerate(big):
            words = [_philox4x32_10(((int(r) * D + d) & 0xFFFFFFFF, (int(r) * D + d) >> 32, 3, 1), (9, 0))[w]
                     for d in range(D)]
            np.testing.assert_array_equal(t[i], sr.sr_bits(v[i], np.array(words, np.uint32)), err_msg="row %d" % r)


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
