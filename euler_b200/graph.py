"""Host-side handles: Graph (HBM-resident CSR) and Context (stream + RNG engine + scratch).

Mirrors the reference's euler::Graph surface for this path (euler/core/graph/graph.h:53-93): Init
from a data directory, node/edge type lookup by name, and construction from arrays the way
tests build graphs through Node::Init (euler/core/graph/node.cc:37-96).  torch is used only to
own device tensors and streams; all work happens in libeuler_b200.so.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import EU_RNG_MINSTD, EU_RNG_PHILOX, EulerError, GraphDesc, check

_RNG = {"minstd": EU_RNG_MINSTD, "philox": EU_RNG_PHILOX, EU_RNG_MINSTD: EU_RNG_MINSTD,
        EU_RNG_PHILOX: EU_RNG_PHILOX}


def _np(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


def _ptr(a):
    return None if a is None else a.ctypes.data


def feat_dtype_code(feat_dtype):
    """eu_feat_dtype of a storage type name: 'float32' or 'bfloat16'; EulerError for anything else, before any allocation."""
    try:
        return _lib.FEAT_DTYPES[feat_dtype]
    except (KeyError, TypeError):
        raise EulerError("feat_dtype must be one of %s, got %r" % (sorted(_lib.FEAT_DTYPES), feat_dtype)) from None


def feat_storage(feat_dtype="float32", feat_place="device", feat_cache_rows=0):
    """eu_feat_storage of a storage type, a place ('device' or 'host') and a number of HBM cache rows; EulerError for an
    unknown type or place, a negative or non-integer row count, or a cache beside a device-placed table, before any
    allocation.  Rows beyond the graph's are refused by the constructor, also before any allocation."""
    dt = feat_dtype_code(feat_dtype)
    try:
        place = _lib.FEAT_PLACES[feat_place]
    except (KeyError, TypeError):
        raise EulerError("feat_place must be one of %s, got %r" % (sorted(_lib.FEAT_PLACES), feat_place)) from None
    if isinstance(feat_cache_rows, bool) or not isinstance(feat_cache_rows, (int, np.integer)) or feat_cache_rows < 0:
        raise EulerError("feat_cache_rows must be an integer >= 0, got %r" % (feat_cache_rows,))
    if feat_cache_rows > 0 and feat_place != "host":
        raise EulerError("feat_cache_rows > 0 needs feat_place='host' (a device-placed table is in HBM already)")
    return _lib.FeatStorage(dt, place, int(feat_cache_rows))


class Graph:
    def __init__(self, handle, device):
        self._h = handle
        self.device = device

    # ---- constructors
    @classmethod
    def from_csr(cls, ids, grp_ptr, nbr, n_edge_types=1, cum_w=None, grp_cum=None, w=None,
                 node_type=None, node_w=None, n_node_types=1, feat=None, feat_slot_dims=None,
                 sampler_order=None, device=0, u64_ptr=None, u64_val=None, n_u64_slots=0, bin_ptr=None, bin_val=None,
                 n_bin_slots=0, binary_feature_names=None, feat_dtype="float32", feat_place="device", feat_cache_rows=0):
        """binary_feature_names: one name per binary slot (default bin_0, bin_1, ...); a slot named 'graph_label' holds each
        node's graph label for sample_graph_label / get_graph_by_label.  feat_dtype: the dense table's storage type,
        'float32' or 'bfloat16' (each value rounded to nearest even on the device; every op reads it widened to f32).
        feat_place 'host': the table sits in mapped pinned host memory and kernels read it in place, with copies of its
        feat_cache_rows rows of highest in-degree in HBM; every op returns the bits it returns on the device-placed graph."""
        st = feat_storage(feat_dtype, feat_place, feat_cache_rows)
        ids = _np(ids, np.uint64)
        keep = [ids, _np(node_type, np.int32), _np(node_w, np.float32), _np(grp_ptr, np.int64),
                _np(nbr, np.uint64), _np(cum_w, np.float32), _np(grp_cum, np.float32),
                _np(w, np.float32), _np(feat, np.float32), _np(sampler_order, np.int64),
                _np(feat_slot_dims, np.int32)]
        d = GraphDesc()
        d.n_nodes = len(ids)
        d.n_edge_types = n_edge_types
        d.n_node_types = n_node_types
        d.ids, d.node_type, d.node_w, d.grp_ptr, d.nbr, d.cum_w, d.grp_cum, d.w = map(_ptr, keep[:8])
        d.feat_dim = 0 if feat is None else keep[8].shape[1]
        d.feat = _ptr(keep[8])
        d.sampler_order = _ptr(keep[9])
        d.n_feat_slots = 0 if feat_slot_dims is None else len(keep[10])
        d.feat_slot_dims = _ptr(keep[10])
        keep += [_np(u64_ptr, np.int64), _np(u64_val, np.uint64), _np(bin_ptr, np.int64), _np(bin_val, np.uint8)]
        if n_u64_slots and u64_ptr is not None:
            d.n_u64_slots, d.u64_ptr, d.u64_val = int(n_u64_slots), _ptr(keep[11]), _ptr(keep[12] if len(keep[12]) else np.zeros(1, np.uint64))
        if n_bin_slots and bin_ptr is not None:
            d.n_bin_slots, d.bin_ptr, d.bin_val = int(n_bin_slots), _ptr(keep[13]), _ptr(keep[14] if len(keep[14]) else np.zeros(1, np.uint8))
        h = C.c_void_p()
        check(_lib.load().eu_graph_create_storage(C.byref(d), device, C.byref(st), C.byref(h)))
        g = cls(h, device)
        for k, name in enumerate(binary_feature_names or ()):
            check(_lib.load().eu_graph_set_binary_feature_name(h, k, str(name).encode()))
        return g

    @classmethod
    def rmat(cls, n_nodes, n_edges, a=0.57, b=0.19, c=0.19, seed=42, feat_dim=0, feat_seed=7, device=0, feat_dtype="float32",
             feat_place="device", feat_cache_rows=0):
        """feat_dtype 'bfloat16': the f32 features rounded to bfloat16 on the device.  feat_place / feat_cache_rows: as
        from_csr."""
        st = feat_storage(feat_dtype, feat_place, feat_cache_rows)
        h = C.c_void_p()
        check(_lib.load().eu_graph_create_rmat_storage(n_nodes, n_edges, a, b, c, seed, feat_dim, feat_seed,
                                                       device, C.byref(st), C.byref(h)))
        return cls(h, device)

    @classmethod
    def rmat_shard(cls, n_nodes, n_edges, shard_index, shard_number, a=0.57, b=0.19, c=0.19, seed=42, feat_dim=0,
                   feat_seed=7, device=0, feat_dtype="float32"):
        """The rows of Graph.rmat(...) owned by shard `shard_index` (owner(id) = id % shard_number)."""
        dt = feat_dtype_code(feat_dtype)
        h = C.c_void_p()
        check(_lib.load().eu_graph_create_rmat_shard_dtype(n_nodes, n_edges, a, b, c, seed, feat_dim, feat_seed, device,
                                                           shard_index, shard_number, dt, C.byref(h)))
        return cls(h, device)

    @classmethod
    def rmat_hetero(cls, n_nodes, n_edges, n_edge_types, n_node_types, shard_index=0, shard_number=1, a=0.57, b=0.19,
                    c=0.19, seed=44, feat_dim=0, feat_seed=7, device=0, feat_dtype="float32", feat_place="device",
                    feat_cache_rows=0):
        """Heterogeneous R-MAT graph (edge type = hash(edge) % T, node type = id % NT), optionally one shard of it.
        feat_place / feat_cache_rows: as from_csr."""
        st = feat_storage(feat_dtype, feat_place, feat_cache_rows)
        h = C.c_void_p()
        check(_lib.load().eu_graph_create_rmat_hetero_storage(n_nodes, n_edges, n_edge_types, n_node_types, a, b, c, seed,
                                                              feat_dim, feat_seed, device, shard_index, shard_number,
                                                              C.byref(st), C.byref(h)))
        return cls(h, device)

    @classmethod
    def load(cls, data_path, shard_index=0, shard_number=1, device=0, load_edges=True, feat_dtype="float32",
             feat_place="device", feat_cache_rows=0):
        """Graph::Init (graph.h:53-56); load_edges=False = load_data_type 'node'; feat_dtype: the node feature table's
        storage type ('float32' or 'bfloat16'); feat_place / feat_cache_rows: as from_csr"""
        st = feat_storage(feat_dtype, feat_place, feat_cache_rows)
        h = C.c_void_p()
        check(_lib.load().eu_graph_load_storage(str(data_path).encode(), shard_index, shard_number, device, int(load_edges),
                                                C.byref(st), C.byref(h)))
        return cls(h, device)

    def close(self):
        if self._h:
            _lib.load().eu_graph_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- accessors
    @property
    def num_nodes(self):
        return _lib.load().eu_graph_num_nodes(self._h)

    @property
    def num_edges(self):
        return _lib.load().eu_graph_num_edges(self._h)

    @property
    def num_edge_types(self):
        return _lib.load().eu_graph_num_edge_types(self._h)

    @property
    def num_node_types(self):
        return _lib.load().eu_graph_num_node_types(self._h)

    @property
    def feat_dim(self):
        return _lib.load().eu_graph_feat_dim(self._h)

    @property
    def feat_dtype(self):
        """'float32' or 'bfloat16': the storage type of the dense node feature table (ops always return f32)"""
        code = _lib.load().eu_graph_feat_dtype(self._h)
        return {v: k for k, v in _lib.FEAT_DTYPES.items()}[code]

    @property
    def feat_place(self):
        """'device' or 'host': where the dense node feature table lives"""
        code = _lib.load().eu_graph_feat_place(self._h)
        return {v: k for k, v in _lib.FEAT_PLACES.items()}[code]

    @property
    def feat_cache_rows(self):
        """rows of a host-placed table copied into HBM (0 for a device-placed one)"""
        return _lib.load().eu_graph_feat_cache_rows(self._h)

    @property
    def hbm_bytes(self):
        return _lib.load().eu_graph_hbm_bytes(self._h)

    @property
    def host_bytes(self):
        """pinned host bytes: the host-placed feature table (0 for a device-placed one)"""
        return _lib.load().eu_graph_host_bytes(self._h)

    def feat_cache_slots(self):
        """int32[n]: each row's HBM cache row, or -1 (all -1 for a device-placed table)"""
        out = np.zeros(self.num_nodes, np.int32)
        check(_lib.load().eu_graph_export_feat_slots(self._h, _ptr(out)))
        return out

    def edge_type_id(self, name):
        return _lib.load().eu_graph_edge_type_id(self._h, str(name).encode())

    def node_type_id(self, name):
        return _lib.load().eu_graph_node_type_id(self._h, str(name).encode())

    def dense_feature_id(self, name):
        return _lib.load().eu_graph_dense_feature_id(self._h, str(name).encode())

    def dense_feature_dim(self, fid):
        return _lib.load().eu_graph_dense_feature_dim(self._h, fid)

    def sparse_feature_id(self, name):
        return _lib.load().eu_graph_sparse_feature_id(self._h, str(name).encode())

    def binary_feature_id(self, name):
        return _lib.load().eu_graph_binary_feature_id(self._h, str(name).encode())

    def edge_feature_id(self, kind, name):
        """kind: 'dense' | 'sparse' | 'binary'"""
        fn = getattr(_lib.load(), "eu_graph_edge_%s_feature_id" % kind)
        return fn(self._h, str(name).encode())

    def set_edges(self, src, dst, type, weight=None, dense=None, dense_dims=None, dense_names=None):
        """Attach edge records (eu_graph_set_edges) for sample_edge and the edge feature ops, as an Euler directory's Edge
        files do: src, dst [E] node ids, type [E] edge types, weight [E] (default 1.0).  dense: f32[E, F], the dense slots
        concatenated per edge, with their widths dense_dims (default one slot of F) and names dense_names (default feat0,
        feat1, ...; the knowledge-graph models read the relation id from a slot named 'id')."""
        src, dst, typ = _np(src, np.uint64), _np(dst, np.uint64), _np(type, np.int32)
        n = len(src)
        if len(dst) != n or len(typ) != n:
            raise EulerError("set_edges: src, dst and type must have one length")
        keep = [src, dst, typ, _np(weight, np.float32)]
        d = _lib.EdgeDesc()
        d.n_edges = n
        d.src, d.dst, d.type, d.w = map(_ptr, keep)
        names = list(dense_names or ())
        if dense is not None:
            feat = np.ascontiguousarray(np.asarray(dense, dtype=np.float32).reshape(n, -1))
            dims = _np(dense_dims if dense_dims is not None else [feat.shape[1]], np.int32)
            if int(dims.sum()) != feat.shape[1] or (names and len(names) != len(dims)):
                raise EulerError("set_edges: dense_dims must add up to dense's width, one name per slot")
            keep += [feat, dims]
            d.feat_dim, d.feat, d.n_feat_slots, d.feat_slot_dims = feat.shape[1], _ptr(feat), len(dims), _ptr(dims)
        elif names:
            raise EulerError("set_edges: dense_names without dense")
        lib = _lib.load()
        check(lib.eu_graph_set_edges(self._h, C.byref(d)))
        for k, name in enumerate(names):
            check(lib.eu_graph_set_edge_dense_feature_name(self._h, k, str(name).encode()))
        return self

    @property
    def num_edge_records(self):
        """edges attached for sample_edge / edge features (0 when the graph was built without them)"""
        return _lib.load().eu_graph_num_edge_records(self._h)

    def export(self, with_feat=True):
        """Copy the CSR back to host numpy arrays (used by tests / the CPU baseline arm).  feat is f32 whatever the table's
        storage type: a bfloat16 table comes back widened, exactly."""
        n, E, T = self.num_nodes, self.num_edges, self.num_edge_types
        out = dict(ids=np.zeros(n, np.uint64), node_type=np.zeros(n, np.int32),
                   node_w=np.zeros(n, np.float32), grp_ptr=np.zeros(n * T + 1, np.int64),
                   nbr=np.zeros(E, np.uint64), cum_w=np.zeros(E, np.float32),
                   grp_cum=np.zeros(n * T, np.float32) if T > 1 else None,
                   feat=np.zeros((n, self.feat_dim), np.float32) if with_feat and self.feat_dim else None)
        check(_lib.load().eu_graph_export(self._h, *[_ptr(out[k]) for k in
                                                     ("ids", "node_type", "node_w", "grp_ptr", "nbr",
                                                      "cum_w", "grp_cum", "feat")]))
        out["T"] = T
        return out


class Context:
    """One execution lane (see include/euler_b200.h): stream + RNG engine + scratch."""

    def __init__(self, graph, rng="minstd", seed=1, stream=None):
        self.graph = graph
        self._h = C.c_void_p()
        self.rng = _RNG[rng]
        check(_lib.load().eu_ctx_create(graph._h, self.rng, seed, stream, C.byref(self._h)))

    def seed(self, s):
        check(_lib.load().eu_ctx_seed(self._h, s))

    def set_engines(self, n, seeds=None):
        """n engines; batch b of a batched call runs on engine b (seeds[b], default seed + b)."""
        arr = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64)
        check(_lib.load().eu_ctx_set_engines(self._h, n, None if arr is None else arr.ctypes.data))

    def set_stream(self, stream_ptr):
        check(_lib.load().eu_ctx_set_stream(self._h, stream_ptr))

    def reserve(self, rows):
        check(_lib.load().eu_ctx_reserve(self._h, rows))

    def sync(self):
        check(_lib.load().eu_ctx_sync(self._h))

    def draws(self):
        d = C.c_uint64(0)
        check(_lib.load().eu_ctx_draws(self._h, C.byref(d)))
        return d.value

    def close(self):
        if self._h:
            _lib.load().eu_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
