"""CPU: the feature placement arguments (feat_place / feat_cache_rows, initialize_graph's feature_place /
feature_cache_rows).  Every refusal happens before any allocation: the Python checks before the library is touched, the
library's own (rows beyond the graph's, host tables of 2^31 rows) before it looks for a device."""
import ctypes as C

import numpy as np
import pytest

import graphs  # noqa: F401  (sys.path)

IDS, PTR, NBR = np.array([1, 2], np.uint64), np.array([0, 1, 1], np.int64), np.array([2], np.uint64)


def _constructors(G, **kw):
    return [lambda: G.from_csr(IDS, PTR, NBR, w=np.ones(1, np.float32), feat=np.ones((2, 4), np.float32), **kw),
            lambda: G.rmat(100, 1000, feat_dim=8, **kw),
            lambda: G.rmat_hetero(100, 1000, 2, 2, feat_dim=8, **kw),
            lambda: G.load("/nonexistent", **kw)]


@pytest.fixture
def no_library(monkeypatch):
    from euler_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "load", refuse)


@pytest.mark.parametrize("bad", ["Host", "hbm", "", None, 1, "cpu"])
def test_unknown_place_raises_before_the_library(no_library, bad):
    import euler_b200
    for call in _constructors(euler_b200.Graph, feat_place=bad):
        with pytest.raises(euler_b200.EulerError, match="feat_place must be one of"):
            call()


@pytest.mark.parametrize("bad", [-1, -100, 1.5, "3", None, True])
def test_bad_cache_rows_raise_before_the_library(no_library, bad):
    import euler_b200
    for call in _constructors(euler_b200.Graph, feat_place="host", feat_cache_rows=bad):
        with pytest.raises(euler_b200.EulerError, match="feat_cache_rows must be an integer >= 0"):
            call()


def test_a_cache_beside_a_device_table_is_refused(no_library):
    import euler_b200
    for call in _constructors(euler_b200.Graph, feat_cache_rows=1):
        with pytest.raises(euler_b200.EulerError, match="needs feat_place='host'"):
            call()
    for call in _constructors(euler_b200.Graph, feat_place="device", feat_cache_rows=5):
        with pytest.raises(euler_b200.EulerError, match="needs feat_place='host'"):
            call()


def test_rmat_shard_takes_no_placement():
    import euler_b200
    with pytest.raises(TypeError):
        euler_b200.Graph.rmat_shard(100, 1000, 0, 2, feat_dim=8, feat_place="host")


@pytest.mark.parametrize("cfg,match", [({"feature_place": "hbm"}, "feat_place must be one of"),
                                       ({"feature_place": "host", "feature_cache_rows": "-1"}, "feature_cache_rows must be"),
                                       ({"feature_place": "host", "feature_cache_rows": "x"}, "feature_cache_rows must be"),
                                       ({"feature_cache_rows": "4"}, "needs feat_place='host'"),
                                       ({"feature_place": "host", "feature_dtype": "fp8"}, "feat_dtype")])
def test_initialize_graph_refuses_before_the_library(no_library, cfg, match):
    import euler_b200
    with pytest.raises(euler_b200.EulerError, match=match):
        euler_b200.initialize_graph(dict({"mode": "local", "data_path": "/nonexistent"}, **cfg))


def test_valid_placements_reach_the_library(no_library):
    import euler_b200
    for kw in ({}, {"feat_place": "device"}, {"feat_place": "host"}, {"feat_place": "host", "feat_cache_rows": 100},
               {"feat_place": "host", "feat_cache_rows": np.int64(3), "feat_dtype": "bfloat16"}):
        with pytest.raises(AssertionError, match="library was called"):
            euler_b200.Graph.rmat(100, 1000, feat_dim=8, **kw)


def test_default_storage_is_todays():
    """the defaults describe an f32 table in HBM without a cache: what every constructor built before the option existed"""
    from euler_b200 import _lib
    from euler_b200.graph import feat_storage
    st = feat_storage()
    assert (st.dtype, st.place, st.cache_rows) == (0, 0, 0)
    assert C.sizeof(_lib.FeatStorage) == 16
    assert _lib.FEAT_PLACES == {"device": 0, "host": 1}


def _lib_or_skip():
    from euler_b200 import _lib
    try:
        return _lib.load()
    except Exception as e:   # pragma: no cover - the library is built by the package build
        pytest.skip("library not built: %s" % e)


def test_library_refuses_rows_beyond_the_graph_before_the_device():
    """C > n is known only to the library (a loaded graph's n comes from its files); it refuses before any device work, so
    the refusal is the same with or without a GPU"""
    from euler_b200 import _lib
    import euler_b200
    lib = _lib_or_skip()
    G = euler_b200.Graph
    with pytest.raises(euler_b200.EulerError, match=r"feature cache rows 101 outside \[0, 100\]"):
        G.rmat(100, 1000, feat_dim=8, feat_place="host", feat_cache_rows=101)
    with pytest.raises(euler_b200.EulerError, match=r"feature cache rows 51 outside \[0, 50\]"):
        G.rmat_hetero(100, 1000, 2, 2, shard_index=1, shard_number=2, feat_dim=8, feat_place="host", feat_cache_rows=51)
    with pytest.raises(euler_b200.EulerError, match=r"feature cache rows 3 outside \[0, 2\]"):
        G.from_csr(IDS, PTR, NBR, w=np.ones(1, np.float32), feat=np.ones((2, 4), np.float32), feat_place="host",
                   feat_cache_rows=3)
    with pytest.raises(euler_b200.EulerError, match=r"feature cache rows 100000 outside \[0, "):
        G.load(graphs.os.path.join(graphs.ROOT, "tests", "golden", "tiny_euler"), feat_place="host", feat_cache_rows=100000)
    with pytest.raises(euler_b200.EulerError, match="fewer than 2\\^31 rows"):
        G.rmat((1 << 31) + 1, 10, feat_dim=8, feat_place="host")
    # the C descriptor's own checks: an unknown place, C < 0, a cache beside a device table
    h = C.c_void_p()
    for st in ((0, 2, 0), (0, 1, -1), (0, 0, 1), (2, 1, 0)):
        rc = lib.eu_graph_create_rmat_storage(100, 1000, 0.57, 0.19, 0.19, 42, 8, 7, 0, C.byref(_lib.FeatStorage(*st)),
                                              C.byref(h))
        assert rc == 1 and not h.value, (st, lib.eu_last_error())   # EU_ERR_INVALID, nothing returned
    assert lib.eu_graph_feat_place(None) == -1 and lib.eu_graph_feat_cache_rows(None) == -1
    assert lib.eu_graph_host_bytes(None) == -1


def test_sharded_feature_calls_refuse_a_host_placed_graph_before_any_exchange():
    import euler_b200
    from euler_b200.sharded import ShardedGraph

    class HostGraph:
        feat_dtype = "float32"
        feat_place = "host"

    class Ops:
        graph = HostGraph()

        def __getattr__(self, name):
            raise AssertionError("ShardedGraph called ops.%s" % name)

    class Xchg:
        world, rank = 2, 0

        def __getattr__(self, name):
            raise AssertionError("ShardedGraph called xchg.%s" % name)

    with pytest.raises(euler_b200.EulerError, match="feature tables held in HBM only"):
        ShardedGraph(Ops(), Xchg()).get_dense_feature([1, 2, 3], 0, 4)
