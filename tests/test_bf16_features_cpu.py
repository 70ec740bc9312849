"""CPU: the bfloat16 feature storage's rounding rule, restated in numpy (tests/bf16_reference.py) and checked against torch's
own f32 -> bf16 conversion; and the feat_dtype argument checks, which run before the library is touched."""
import numpy as np
import pytest
import torch

import bf16_reference as br
import graphs  # noqa: F401  (sys.path)


def _torch_bits(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def _agree(x):
    """the restatement equals torch bit for bit on every non-NaN value, and both give a NaN exactly where x is one"""
    got, want = br.round_bits(x), _torch_bits(x)
    nan = np.isnan(x)
    assert np.array_equal(np.isnan(br.widen(got)), nan) and np.array_equal(np.isnan(br.widen(want)), nan)
    bad = np.flatnonzero((got != want) & ~nan)
    assert bad.size == 0, [(hex(int(x.view(np.uint32)[i])), hex(int(got[i])), hex(int(want[i]))) for i in bad[:8]]


def test_special_values_round_like_torch():
    x = br.special_values()
    _agree(x)
    bits = br.round_bits(x)
    u = x.view(np.uint32)
    assert np.array_equal(bits[u == 0x7F800000], [0x7F80]) and np.array_equal(bits[u == 0xFF800000], [0xFF80])   # +-Inf kept
    assert np.array_equal(bits[u == 0x7F7FFFFF], [0x7F80]) and np.array_equal(bits[u == 0xFF7FFFFF], [0xFF80])   # round up to Inf
    assert bits[u == 0x7F7F7FFF][0] == 0x7F7F and bits[u == 0x7F7F8000][0] == 0x7F80                           # the last tie: up
    assert bits[u == 0x3F808000][0] == 0x3F80 and bits[u == 0x3F818000][0] == 0x3F82                           # ties to even
    assert bits[u == 0x00000001][0] == 0 and bits[u == 0x80000001][0] == 0x8000                                # signed zero kept
    assert bits[u == 0x00018000][0] == 0x0002 and bits[u == 0x00028000][0] == 0x0002                           # subnormal ties
    assert np.all(bits[np.isnan(x)] == br.CANONICAL_NAN)


def test_halfway_values_at_both_parities():
    rng = np.random.RandomState(1)
    hi = rng.randint(0, 0x7F80, size=1 << 16).astype(np.uint32)           # every finite magnitude, both parities of the kept half
    sign = rng.randint(0, 2, size=hi.size).astype(np.uint32) << 31
    x = ((hi << 16) | 0x8000 | sign).view(np.float32)
    _agree(x)
    kept = br.round_bits(x) & 0x7FFF
    assert np.array_equal(kept, np.where(hi & 1, hi + 1, hi).astype(np.uint16))


def test_random_bit_patterns():
    x = np.random.RandomState(7).randint(0, 1 << 32, size=1 << 24, dtype=np.uint64).astype(np.uint32).view(np.float32)
    _agree(x)


def test_widening_is_exact_and_round_trips():
    bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    f = br.widen(bits)
    finite = ~np.isnan(f)
    assert np.array_equal(br.round_bits(f)[finite], bits[finite])
    assert np.array_equal(torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16).float().numpy().view(np.uint32),
                          f.view(np.uint32))


@pytest.fixture
def no_library(monkeypatch):
    from euler_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "load", refuse)


@pytest.mark.parametrize("bad", ["float16", "bf16", "FLOAT32", "", None, 1, np.float32])
def test_unknown_feat_dtype_raises_before_the_library(no_library, bad):
    import euler_b200
    G = euler_b200.Graph
    ids, ptr, nbr = np.array([1, 2], np.uint64), np.array([0, 1, 1], np.int64), np.array([2], np.uint64)
    calls = [lambda: G.from_csr(ids, ptr, nbr, w=np.ones(1, np.float32), feat=np.ones((2, 4), np.float32), feat_dtype=bad),
             lambda: G.rmat(100, 1000, feat_dim=8, feat_dtype=bad),
             lambda: G.rmat_shard(100, 1000, 0, 2, feat_dim=8, feat_dtype=bad),
             lambda: G.rmat_hetero(100, 1000, 2, 2, feat_dim=8, feat_dtype=bad),
             lambda: G.load("/nonexistent", feat_dtype=bad)]
    for call in calls:
        with pytest.raises(euler_b200.EulerError, match="feat_dtype"):
            call()
    if isinstance(bad, str):
        with pytest.raises(euler_b200.EulerError, match="feat_dtype"):
            euler_b200.initialize_graph({"mode": "local", "data_path": "/nonexistent", "feature_dtype": bad})


def test_known_feat_dtypes_reach_the_library(no_library):
    import euler_b200
    for dt in ("float32", "bfloat16"):
        with pytest.raises(AssertionError, match="library was called"):
            euler_b200.Graph.rmat(100, 1000, feat_dim=8, feat_dtype=dt)


def test_sharded_feature_calls_refuse_a_bf16_graph_before_any_exchange():
    import euler_b200
    from euler_b200.sharded import ShardedGraph

    class Bf16Graph:
        feat_dtype = "bfloat16"

    class Ops:
        graph = Bf16Graph()

        def __getattr__(self, name):
            raise AssertionError("ShardedGraph called ops.%s" % name)

    class Xchg:
        world, rank = 2, 0

        def __getattr__(self, name):
            raise AssertionError("ShardedGraph called xchg.%s" % name)

    with pytest.raises(euler_b200.EulerError, match="float32 feature tables only"):
        ShardedGraph(Ops(), Xchg()).get_dense_feature([1, 2, 3], 0, 4)
