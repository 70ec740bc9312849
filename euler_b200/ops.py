"""tf_euler's Python op API for the minibatch-construction path, over torch CUDA tensors.

Same names, argument meaning and error behaviour as the reference wrappers
(tf_euler/python/euler_ops/{base,neighbor_ops,walk_ops,sample_ops,feature_ops,mp_ops,type_ops}.py);
each function cites the wrapper it mirrors.  Tensors are torch tensors on the graph's device; every
op enqueues kernels from libeuler_b200.so on the current torch stream.  Nothing here computes on the
CPU and nothing falls back to PyTorch ops: if the library or the GPU is missing, calls raise.
"""
import ctypes as C
import functools
import math
import threading

import numpy as np
import torch

from . import _lib
from ._lib import EulerError, check
from .graph import Context, Graph, feat_dtype_code, feat_storage

_state = threading.local()
_default = {"graph": None, "rng": "minstd", "seed": 1}


# ------------------------------------------------------------------------------------ init
def initialize_graph(config):
    """base.initialize_graph (tf_euler/python/euler_ops/base.py:37-60): str or dict of k=v;
    TypeError otherwise.  Returns what InitQueryProxy returns."""
    if isinstance(config, dict):
        config = ';'.join('{}={}'.format(key, value) for key, value in config.items())
    if not isinstance(config, str):
        raise TypeError('Expect str or dict for graph config, got {}.'.format(type(config).__name__))
    # feature_dtype=float32|bfloat16: the node feature table's storage type (Graph.load's feat_dtype); feature_place=device|host
    # and feature_cache_rows=C: where it lives and how many of its rows are cached in HBM (Graph.load's feat_place and
    # feat_cache_rows).  All are checked before the load.
    opts = {}
    for item in config.split(';'):
        key, eq, value = item.partition('=')
        if key in ('feature_dtype', 'feature_place', 'feature_cache_rows') and eq:
            opts[key] = value
    if 'feature_dtype' in opts:
        feat_dtype_code(opts['feature_dtype'])
    if 'feature_place' in opts or 'feature_cache_rows' in opts:
        rows = opts.get('feature_cache_rows', '0')
        if not rows.isdigit():
            raise EulerError("feature_cache_rows must be an integer >= 0, got %r" % rows)
        feat_storage(opts.get('feature_dtype', 'float32'), opts.get('feature_place', 'device'), int(rows))
    lib = _lib.load()
    ok = bool(lib.InitQueryProxy(config.encode()))
    h = lib.eu_default_graph()
    if h:
        kv = dict(item.split('=') for item in config.split(';') if item)
        g = Graph(C.c_void_p(h), int(kv.get('device', 0)))
        g.close = lambda: None  # owned by the library's default slot
        set_graph(g, rng=kv.get('rng', 'minstd'), seed=int(kv.get('seed', 1)))
    return ok


def initialize_embedded_graph(data_dir, sampler_type='all', data_type='all'):
    """base.initialize_embedded_graph (base.py:63-67)."""
    return initialize_graph({'mode': 'local', 'data_path': data_dir, 'data_type': data_type,
                             'sampler_type': sampler_type})


def set_graph(graph, rng="minstd", seed=1):
    """Install an already-built Graph (synthetic / from arrays) as the process default."""
    _default.update(graph=graph, rng=rng, seed=seed)
    _state.__dict__.pop("ctx", None)


def get_graph():
    if _default["graph"] is None:
        raise EulerError("graph is not initialized: call initialize_graph / set_graph first")
    return _default["graph"]


def context():
    """Per-thread Context of the default graph (one engine per client thread, like
    euler/common/random.cc:22's thread_local engine)."""
    ctx = getattr(_state, "ctx", None)
    if ctx is None or ctx.graph is not _default["graph"]:
        ctx = Context(get_graph(), _default["rng"], _default["seed"])
        _state.ctx = ctx
        _state.stream = None    # a fresh Context is not bound to any torch stream yet
    return ctx


def seed(s):
    """Re-seed this thread's engine (the reference has no seed API; parity tests need one)."""
    context().seed(s)


def _dev():
    return torch.device("cuda", get_graph().device)


def _ctx_on_stream():
    """This thread's Context, bound to torch's current stream.  All ops of a Context share its scratch (dedup tables, engine
    state, staging), so when the current stream CHANGES the new stream is first ordered after everything the Context issued on
    the old one (an event, no host sync)."""
    ctx = context()
    cur = torch.cuda.current_stream(_dev())
    prev = getattr(_state, "stream", None)
    if prev is not None and prev.cuda_stream != cur.cuda_stream:
        ev = torch.cuda.Event()
        ev.record(prev)
        cur.wait_event(ev)
    if prev is None or prev.cuda_stream != cur.cuda_stream:
        ctx.set_stream(cur.cuda_stream)
        _state.stream = cur
    return ctx


def _arg(x):
    """one argument of a library call: a tensor or numpy array as its data pointer, a list of them (None for a hole) as a
    void* array, anything else as it is"""
    if isinstance(x, torch.Tensor):
        return x.data_ptr()
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if isinstance(x, (list, tuple)):
        return (C.c_void_p * max(len(x), 1))(*[_arg(v) for v in x])
    return x


def _call(name, *args, ctx=None):
    """the library's entry point `name` on the Context handle (this thread's, on torch's current stream, unless ctx is
    given) and args; raises EulerError when it fails"""
    ctx = ctx or _ctx_on_stream()
    check(getattr(_lib.load(), name)(ctx._h, *[_arg(a) for a in args]))


def _ragged_lengths(name, rows, *args):
    """the first phase of include/euler_b200.h's ragged protocol, for an entry point whose arguments after args are
    (cap, indptr, *outs): called with cap = 0 it fills indptr i64[rows + 1] only.  Returns (indptr, total = indptr[-1]),
    read back with one host sync."""
    n_outs = len(_lib.SIGNATURES[name][1]) - 3 - len(args)     # the context handle, cap and indptr are the other three
    indptr = torch.empty(rows + 1, dtype=torch.int64, device=_dev())
    _call(name, *args, 0, indptr, *[None] * n_outs)
    return indptr, int(indptr[-1].item())


def _ragged(name, rows, alloc, *args, lengths=None):
    """the whole ragged protocol: the first phase (unless lengths = (indptr, total) holds its result), then the outputs
    alloc(total) returns, filled by a second call when total > 0.  Returns (indptr, total, outputs)."""
    indptr, total = lengths or _ragged_lengths(name, rows, *args)
    outs = alloc(total)
    if total:
        _call(name, *args, total, indptr, *outs)
    return indptr, total, outs


def _sparse_tensor(indptr, values, n, total, max_len=None):
    """the SparseTensor content (indices i64[total, 2], values, dense_shape (n, max_len)) of the ragged rows
    values[indptr[i]:indptr[i+1]]; max_len=None reads the longest row back (one host sync)"""
    dev = indptr.device
    lens = indptr[1:] - indptr[:-1]
    rows = torch.repeat_interleave(torch.arange(n, device=dev), lens, output_size=total)
    cols = torch.arange(total, device=dev) - indptr[:-1][rows]
    if max_len is None:
        max_len = int(lens.max().item()) if n else 0
    return torch.stack([rows, cols], dim=1), values, (n, max_len)


def _t(x, dtype):
    if isinstance(x, torch.Tensor):
        return x.to(device=_dev(), dtype=dtype).contiguous()
    return torch.as_tensor(np.asarray(x), dtype=dtype, device=_dev()).contiguous()


def _i32_host(x):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x).reshape(-1), dtype=np.int32)


def _out_dtype(op, dtype):
    """the eu_feat_dtype code of an output dtype (torch.float32 or torch.bfloat16); any other dtype raises EulerError"""
    code = _lib.TORCH_DTYPES.get(dtype)
    if code is None:
        raise EulerError("%s: the output dtype must be torch.float32 or torch.bfloat16, got %r" % (op, dtype))
    return code


def _slot(name, lookup):
    """a feature slot: an int is the slot id, anything else a name lookup resolves"""
    return int(name) if isinstance(name, (int, np.integer)) else lookup(str(name))


def _neighbor_triple(shape):
    """empty (ids i64, weights f32, types i32) neighbor outputs of one shape"""
    dev = _dev()
    return tuple(torch.empty(shape, dtype=dt, device=dev) for dt in (torch.int64, torch.float32, torch.int32))


def _neighbor_rows(entry, nodes, edge_types, k, *default_node):
    """the k (ids, weights, types) per node that sample_neighbor, get_top_k_neighbor and sample_neighbor_api return: entry
    takes (nodes, n, types, n_types, k[, default_node], ids, weights, types)"""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    ids, w, t = _neighbor_triple((nodes.numel(), k))
    _call(entry, nodes, nodes.numel(), et, len(et), k, *default_node, ids, w, t)
    return ids, w, t


# ------------------------------------------------------------------------------------ type ops
def get_edge_type_id(type_id_or_names):
    """type_ops.get_edge_type_id (type_ops.py:57-68): names resolved through graph meta."""
    return _type_ids(type_id_or_names, get_graph().edge_type_id)


def get_node_type_id(type_id_or_names):
    """type_ops.get_node_type_id (type_ops.py:42-54)."""
    return _type_ids(type_id_or_names, get_graph().node_type_id)


def _type_ids(v, lookup):
    if isinstance(v, torch.Tensor):
        return _i32_host(v)
    arr = np.asarray(v).reshape(-1)
    if arr.dtype.kind in "US":
        return np.asarray([lookup(str(s)) for s in arr], np.int32)
    return arr.astype(np.int32)


def _hop_types(op, edge_types, hops=None):
    """one edge-type list per hop (exactly `hops` of them when given), all of one length T: i32[L, T], [0, 0] for none"""
    ets = [get_edge_type_id(e) for e in edge_types]
    if (hops is not None and len(ets) != hops) or any(len(e) != len(ets[0]) for e in ets):
        raise EulerError("%s: edge_types must hold one equal-length type list per hop" % op)
    return np.ascontiguousarray(np.stack(ets) if ets else np.zeros((0, 0)), dtype=np.int32)


def _fanout_args(op, B, edge_types, counts):
    """the hop arguments of the fanout entry points, (types i32[L, T], T, counts i32[L], L), and hop i's shape
    (B, c1, ..., ci) for each hop"""
    et = _hop_types(op, edge_types, len(counts))
    shapes = [(B,) + tuple(int(c) for c in counts[:i + 1]) for i in range(len(counts))]
    return (et, et.shape[1], np.ascontiguousarray(counts, dtype=np.int32), len(counts)), shapes


def _hop_outputs(shapes):
    """per hop shape a neighbor triple, returned as three lists (ids, weights, types)"""
    triples = [_neighbor_triple(sh) for sh in shapes]
    return tuple([tr[k] for tr in triples] for k in range(3))


# ------------------------------------------------------------------------------------ sampling
def sample_neighbor(nodes, edge_types, count, default_node=-1, condition=''):
    """neighbor_ops.sample_neighbor (neighbor_ops.py:39-41).  Returns (neighbors i64[B,count],
    weights f32[B,count], types i32[B,count])."""
    if condition:
        raise EulerError("sample_neighbor: `condition` (index queries) is outside this path")
    return _neighbor_rows("eu_sample_neighbor", nodes, edge_types, count, default_node)


def sample_fanout(nodes, edge_types, counts, default_node=-1):
    """neighbor_ops.sample_fanout (neighbor_ops.py:122-158).  edge_types: list (per hop) of 1-D
    type lists of equal length.  Returns (neighbors_list[L+1], weights_list[L], types_list[L]),
    all flattened like the reference."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    B = nodes.numel()
    hop_args, shapes = _fanout_args("sample_fanout", B, edge_types, counts)
    ids, ws, ts = _hop_outputs([math.prod(sh) for sh in shapes])
    _call("eu_sample_fanout", nodes, B, *hop_args, default_node, ids, ws, ts)
    return [nodes] + ids, ws, ts


def sample_fanout_with_feature(nodes, edge_types, count, default_node, dense_feature_names, dense_dimensions,
                               sparse_feature_names, sparse_default_values, dense_dtype=torch.float32):
    """neighbor_ops.sample_fanout_with_feature (neighbor_ops.py:49-69; kernel sample_fanout_with_feature_op.cc).  The hops are
    sample_fanout's (the same draws on the same context state); the features of hop i are those of its engine ids, as the
    reference's v_select(nb_i) takes them (a row whose first draw is node 0 is packed as default_node but keeps the features of
    its draws).  Returns, as the reference's wrapper does:
        neighbors        [nodes] + L flattened hops
        weights, types   L tensors shaped [B, c1, ..., ci]
        dense_features   (L+1) * len(dense_feature_names) tensors of dense_dtype [rows_i, dim], hop-major
        sparse_features  (L+1) * len(sparse_feature_names) (indices, values, dense_shape) triples, hop-major, as get_sparse_feature
    dense_dtype=torch.bfloat16 gives the f32 dense features rounded to nearest even on the device, bit for bit; everything else
    (the draws included) is the f32 call's.  One host synchronisation per call when sparse features are asked for (all ragged
    totals together), none otherwise."""
    code = _out_dtype("sample_fanout_with_feature", dense_dtype)
    g = get_graph()
    nodes = _t(nodes, torch.int64).reshape(-1)
    L = len(count)
    B, dev = nodes.numel(), nodes.device
    hop_args, shapes = _fanout_args("sample_fanout_with_feature", B, edge_types, count)
    if len(dense_feature_names) != len(dense_dimensions) or len(sparse_feature_names) != len(sparse_default_values):
        raise EulerError("sample_fanout_with_feature: one dimension per dense feature and one default per sparse feature")
    rows = [B] + [math.prod(sh) for sh in shapes]
    ids, ws, ts = _hop_outputs(shapes)
    ids = [x.view(-1) for x in ids]
    eng = [torch.empty_like(x) for x in ids]
    dfid = np.asarray([_slot(n, g.dense_feature_id) for n in dense_feature_names], np.int32)
    ddim = np.asarray(dense_dimensions, np.int32)
    sfid = np.asarray([g.sparse_feature_id(str(n)) for n in sparse_feature_names], np.int32)
    nd, ns = len(dfid), len(sfid)
    dense = [torch.empty((rows[l], int(ddim[j])), dtype=dense_dtype, device=dev) for l in range(L + 1) for j in range(nd)]
    ptrs = [torch.empty(rows[l] + 1, dtype=torch.int64, device=dev) for l in range(L + 1) for j in range(ns)]
    total, maxlen = np.zeros(max(len(ptrs), 1), np.int64), np.zeros(max(len(ptrs), 1), np.int64)
    _call("eu_sample_fanout_with_feature_out_dtype", nodes, B, *hop_args, default_node, ids, ws, ts, eng, nd, dfid, ddim, code, dense,
          ns, sfid, ptrs, total, maxlen)
    sparse = []
    for l in range(L + 1):
        hop_ids = nodes if l == 0 else eng[l - 1]
        for j in range(ns):
            k = l * ns + j
            _, tot, (vals,) = _ragged("eu_get_sparse_feature", rows[l], _values_i64, hop_ids, rows[l], int(sfid[j]),
                                      int(sparse_default_values[j]), lengths=(ptrs[k], int(total[k])))
            sparse.append(_sparse_tensor(ptrs[k], vals, rows[l], tot, int(maxlen[k])))
    return [nodes] + ids, ws, ts, dense, sparse


def sample_fanout_batched(nodes, edge_types, counts, default_node=-1, ctx=None):
    """nb independent sample_fanout calls in one set of kernel launches.  nodes: [nb, B]; batch b runs on engine b
    of `ctx` (Context.set_engines), i.e. it returns exactly what sample_fanout(nodes[b]) returns on a context
    seeded like engine b.  Returns (neighbors_list[L+1], weights_list[L], types_list[L]) with a leading nb dim."""
    nodes = _t(nodes, torch.int64)
    nb, B = nodes.shape
    hop_args, shapes = _fanout_args("sample_fanout_batched", B, edge_types, counts)
    ids, ws, ts = _hop_outputs([(nb, math.prod(sh)) for sh in shapes])
    _call("eu_sample_fanout_batched", nodes, nb, B, *hop_args, default_node, ids, ws, ts, ctx=ctx)
    return [nodes] + ids, ws, ts


def sample_node(count, node_type, condition=''):
    """sample_ops.sample_node (sample_ops.py:38-54); node_type '-1' (or -1) = all types."""
    if condition:
        raise EulerError("sample_node: `condition` (index queries) is outside this path")
    if isinstance(node_type, str) and node_type == '-1':
        types = np.asarray([-1], np.int32)
    else:
        types = get_node_type_id(node_type)
    count = int(count)
    out = torch.empty(count, dtype=torch.int64, device=_dev())
    _call("eu_sample_node", count, types, len(types), out)
    return out


def get_node_type(nodes):
    """the node type of every node (base._LIB_OP.get_node_type, euler::GetNodeType api.cc:50-61): i32[B], INT32_MIN for an
    id that is not a node"""
    nodes = _t(nodes, torch.int64).reshape(-1)
    out = torch.empty(nodes.numel(), dtype=torch.int32, device=nodes.device)
    _call("eu_get_node_type", nodes, nodes.numel(), out)
    return out


def sample_n_with_types(count, types):
    """base._LIB_OP.sample_n_with_types (kernel tf_euler/kernels/sample_n_with_types_op.cc): row i of the i64[n, count]
    result is `count` nodes drawn from node type types[i], the rows drawn in order from this thread's engine.  A type that
    is INT32_MIN (an absent source) or out of range raises EulerError, and so does a type of total weight 0 (upstream
    aborts); a refused call draws nothing."""
    types = _t(types, torch.int32).reshape(-1)
    count = int(count)
    out = torch.empty((types.numel(), count), dtype=torch.int64, device=types.device)
    _call("eu_sample_n_with_types", types, types.numel(), count, out)
    return out


def sample_node_with_src(src_nodes, count):
    """sample_ops.sample_node_with_src (sample_ops.py:75-87): for every source node, `count` nodes of its type,
    i64[len(src_nodes), count]"""
    return sample_n_with_types(count, get_node_type(src_nodes))


def random_walk(nodes, edge_types, p=1.0, q=1.0, default_node=-1):
    """walk_ops.random_walk (walk_ops.py:29-43).  edge_types: list of L 1-D type lists.
    Returns i64[B, L+1]."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = _hop_types("random_walk", edge_types)
    L, B = et.shape[0], nodes.numel()
    out = torch.empty((B, L + 1), dtype=torch.int64, device=nodes.device)
    _call("eu_random_walk", nodes, B, et, et.shape[1], L, float(p), float(q), default_node, out)
    return out


def get_dense_feature(nodes, feature_names, dimensions, thread_num=1, out_dtype=torch.float32):
    """feature_ops.get_dense_feature (feature_ops.py:111-125): list of [M, dim_i] tensors of out_dtype; names are
    looked up as "dense_"+name in the graph meta (get_dense_feature_op.cc:83); ints are slot ids.  out_dtype=torch.bfloat16
    gives the f32 result rounded to nearest even on the device, bit for bit (a bf16 table's stored bits, unchanged)."""
    del thread_num  # the reference splits the batch over TF threads; one launch here
    code = _out_dtype("get_dense_feature", out_dtype)
    nodes = _t(nodes, torch.int64).reshape(-1)
    g = get_graph()
    outs = []
    for name, dim in zip(feature_names, dimensions):
        out = torch.empty((nodes.numel(), int(dim)), dtype=out_dtype, device=nodes.device)
        _call("eu_get_dense_feature_out_dtype", nodes, nodes.numel(), _slot(name, g.dense_feature_id), int(dim), code, out)
        outs.append(out)
    return outs


def neighbor_top_k_feature(nodes, neighbors, feature_name, dimension, k, out_dtype=torch.float32):
    """LGCEncoder's input block (encoders.py:895-922) in one device op: nodes i64 of any shape (flattened to [B]), neighbors
    i64[B, count] (sample_neighbor's rows), the dense slot feature_name (a name, or an int slot id) read dimension columns
    wide.  Returns f32[B, k + 1, dimension]: row 0 is get_dense_feature(nodes), rows 1 .. k the k largest values of each
    column over the node's neighbours, descending; equal values keep the lower neighbour index first (tf.nn.top_k's rule),
    NaN ranks above every number.  It equals cat(get_dense_feature(nodes), the first k rows of a stable descending sort of
    get_dense_feature(neighbors) per column) to the bit.  No gradient (the rows are graph data).  1 <= k <= count and
    k <= NEIGHBOR_TOP_K_MAX (16), or EulerError.  out_dtype=torch.bfloat16 stores the same selection rounded to nearest even,
    bit for bit the f32 result's rounding."""
    code = _out_dtype("neighbor_top_k_feature", out_dtype)
    nodes = _t(nodes, torch.int64).reshape(-1)
    neighbors = _t(neighbors, torch.int64)
    B = nodes.numel()
    if neighbors.dim() != 2 or neighbors.shape[0] != B:
        raise EulerError("neighbor_top_k_feature: neighbors must be [B, count] for B = %d nodes, got %s" % (B, tuple(neighbors.shape)))
    k, dim = int(k), int(dimension)
    out = torch.empty((B, max(k, 0) + 1, max(dim, 0)), dtype=out_dtype, device=nodes.device)   # bad sizes: the library refuses
    _call("eu_neighbor_top_k_feature_out_dtype", nodes, B, neighbors, neighbors.shape[1],
          _slot(feature_name, get_graph().dense_feature_id), dim, k, code, out)
    return out


def _values_i64(total):
    return (torch.empty(total, dtype=torch.int64, device=_dev()),)


def _sparse_features(entry, keys, feature_names, default_values, fid_of):
    """get_sparse_feature over keys (node ids, or edges for eu_get_edge_sparse_feature): per feature the SparseTensor content"""
    names = [str(x) for x in feature_names]
    defaults = [0] * len(names) if default_values is None else [int(x) for x in default_values]
    n, outs = keys.shape[0], []
    for name, dv in zip(names, defaults):
        indptr, total, (vals,) = _ragged(entry, n, _values_i64, keys, n, fid_of(name), dv)
        outs.append(_sparse_tensor(indptr, vals, n, total))
    return outs


def _binary_features(entry, keys, feature_names, fid_of):
    """get_binary_feature over keys (node ids, or edges for eu_get_edge_binary_feature): per feature n byte strings"""
    n, outs = keys.shape[0], []
    for name in feature_names:
        indptr, _, (buf,) = _ragged(entry, n, lambda t: (torch.empty(t, dtype=torch.uint8, device=_dev()),), keys, n,
                                    fid_of(str(name)))
        raw, ptr = bytes(buf.cpu().numpy().tobytes()), indptr.cpu().tolist()
        outs.append([raw[ptr[i]:ptr[i + 1]] for i in range(n)])
    return outs


def get_sparse_feature(nodes, feature_names, default_values=None, thread_num=1):
    """feature_ops.get_sparse_feature (feature_ops.py:57-73; kernel get_sparse_feature_op.cc:52-130).  Per feature the
    reference returns a SparseTensor; here the same content as (indices i64[nnz, 2], values i64[nnz], dense_shape (N, max_len)):
    row i lists the uint64 values of the node, a node without values gets the single entry (i, 0) = default value."""
    fid_of = get_graph().sparse_feature_id
    return _sparse_features("eu_get_sparse_feature", _t(nodes, torch.int64).reshape(-1), feature_names, default_values, fid_of)


def get_binary_feature(nodes, feature_names, thread_num=1):
    """feature_ops.get_binary_feature (feature_ops.py:158-171): per feature a list of N byte strings (b'' for absent nodes)."""
    fid_of = get_graph().binary_feature_id
    return _binary_features("eu_get_binary_feature", _t(nodes, torch.int64).reshape(-1), feature_names, fid_of)


def sample_edge(count, edge_type):
    """sample_ops.sample_edge (tf_euler/python/euler_ops/sample_ops.py; kernel sample_edge_op.cc): i64[count, 3] rows of
    (src, dst, type), drawn by edge weight among the edges of ONE type (several types return nothing in the reference)."""
    types = get_edge_type_id(edge_type)
    count = int(count)
    out = torch.empty((count, 3), dtype=torch.int64, device=_dev())
    _call("eu_sample_edge", count, types, len(types), out)
    return out


def _edges(edges):
    e = _t(edges, torch.int64)
    if e.dim() != 2 or e.shape[1] != 3:
        raise EulerError("edges must be a matrix with shape [n, 3]")
    return e.contiguous()


def get_edge_dense_feature(edges, feature_names, dimensions, thread_num=1):
    """feature_ops.get_edge_dense_feature: list of f32[E, dim] (zeros for unknown edges / features)"""
    e = _edges(edges)
    g, outs = get_graph(), []
    for name, dim in zip(feature_names, dimensions):
        out = torch.empty((e.shape[0], int(dim)), dtype=torch.float32, device=e.device)
        _call("eu_get_edge_dense_feature", e, e.shape[0], g.edge_feature_id("dense", name), int(dim), out)
        outs.append(out)
    return outs


def get_edge_sparse_feature(edges, feature_names, default_values=None, thread_num=1):
    """feature_ops.get_edge_sparse_feature: per feature (indices i64[nnz, 2], values i64[nnz], dense_shape)"""
    e = _edges(edges)
    fid_of = functools.partial(get_graph().edge_feature_id, "sparse")
    return _sparse_features("eu_get_edge_sparse_feature", e, feature_names, default_values, fid_of)


def get_edge_binary_feature(edges, feature_names, thread_num=1):
    """feature_ops.get_edge_binary_feature: per feature a list of E byte strings"""
    e = _edges(edges)
    fid_of = functools.partial(get_graph().edge_feature_id, "binary")
    return _binary_features("eu_get_edge_binary_feature", e, feature_names, fid_of)


def get_full_neighbor(nodes, edge_types):
    """neighbor_ops.get_full_neighbor (tf_euler/python/euler_ops/neighbor_ops.py; kernel get_full_neighbor_op.cc over
    euler::GetFullNeighbor api.cc:208-221).  The reference returns three SparseTensors [N, max_degree] (ids, weights,
    types) whose values are listed node by node; here the same values come back ragged: (indptr i64[N+1], ids i64[nnz],
    weights f32[nnz], types i32[nnz]) -- SparseTensor indices are (i, k - indptr[i]) for k in [indptr[i], indptr[i+1])."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = np.ascontiguousarray(edge_types, dtype=np.int32).reshape(-1)
    indptr, _, outs = _ragged("eu_get_full_neighbor", nodes.numel(), _neighbor_triple, nodes, nodes.numel(), et, len(et))
    return (indptr,) + outs


def get_sorted_full_neighbor(nodes, edge_types, condition=''):
    """neighbor_ops.get_sorted_full_neighbor (neighbor_ops.py:100-119): get_full_neighbor with every node's entries ordered by
    neighbor id; same ragged return."""
    if condition:
        raise EulerError("get_sorted_full_neighbor: `condition` (index queries) is outside this path")
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    indptr, _, outs = _ragged("eu_get_sorted_full_neighbor", nodes.numel(), _neighbor_triple, nodes, nodes.numel(), et, len(et))
    return (indptr,) + outs


def get_top_k_neighbor(nodes, edge_types, k, default_node=-1, condition=''):
    """neighbor_ops.get_top_k_neighbor (neighbor_ops.py:44-46): (ids i64[N,k], weights f32[N,k], types i32[N,k]), the k
    heaviest edges of each node, heaviest first, filled with default_node / 0 / -1."""
    if condition:
        raise EulerError("get_top_k_neighbor: `condition` (index queries) is outside this path")
    return _neighbor_rows("eu_get_top_k_neighbor", nodes, edge_types, int(k), default_node)


_HOP_APPEND_FRONTIER, _HOP_SELF_LOOPS, _HOP_SORT = 1, 2, 4     # include/euler_b200.h


def _full_hop(nodes, edge_types, flags, rows=True, weights=False, types=False):
    """one eu_full_neighbor_hop: two host syncs, the listing total (output shapes) and the unique count (the frontier's length)"""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    n, dev = nodes.numel(), nodes.device
    indptr, total = _ragged_lengths("eu_full_neighbor_hop", n, nodes, n, et, len(et), flags)
    append = bool(flags & _HOP_APPEND_FRONTIER)
    width = total + (n if flags & _HOP_SELF_LOOPS else 0)
    uniq = torch.empty(total + (n if append else 0), dtype=torch.int64, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    edge_index = torch.empty((2 if rows else 1, width), dtype=torch.int64, device=dev)
    w = torch.empty(total, dtype=torch.float32, device=dev) if weights else None
    t = torch.empty(total, dtype=torch.int32, device=dev) if types else None
    res = torch.empty(n, dtype=torch.int64, device=dev) if append else None
    _call("eu_full_neighbor_hop", nodes, n, et, len(et), flags, total, indptr, uniq, cnt, edge_index[0] if rows else None,
          edge_index[-1], w, t, res)
    return indptr, uniq[:int(cnt.item())], res, edge_index, w, t


def full_neighbor_hop(nodes, edge_types, self_loops=True, with_types=False):
    """One hop of GCNDataFlow / RelationDataFlow (gcn_dataflow.py:34-48 + neighbor_dataflow.py:84-110,
    relation_dataflow.py:31-71) in one fused device op: lists every neighbor of `nodes` (get_full_neighbor's order) and
    numbers the listed ids and then the nodes themselves by first occurrence (tf.unique(concat(neighbors, nodes))).
    Returns (n_id, res_n_id, edge_index, types):
        n_id        i64[m]        the next frontier: unique(concat(neighbors, nodes))
        res_n_id    i64[n]        the position of every node in n_id
        edge_index  i64[2, E(+n)] [row of each listed entry, its position in n_id], followed with self_loops by the n
                                  self loops [k, res_n_id[k]]
        types       i32[E]        each entry's edge type (with_types), else None"""
    flags = _HOP_APPEND_FRONTIER | (_HOP_SELF_LOOPS if self_loops else 0)
    _, n_id, res, edge_index, _, t = _full_hop(nodes, edge_types, flags, types=with_types)
    return n_id, res, edge_index, t


def full_neighbor_adjacency(nodes, edge_types):
    """One hop of get_multi_hop_neighbor (neighbor_ops.py:209-242) in one fused device op: (next_nodes, indptr, cols,
    weights) with next_nodes = tf.unique(every listed neighbor) and row i's entries [indptr[i], indptr[i+1]) =
    (cols, weights) ordered by column (tf.sparse_reorder; equal columns -- multi-edges, repeated types -- in listing order)."""
    indptr, nxt, _, cols, w, _ = _full_hop(nodes, edge_types, _HOP_SORT, rows=False, weights=True)
    return nxt, indptr, cols[0], w


def get_multi_hop_neighbor(nodes, edge_types, sampler=None):
    """neighbor_ops.get_multi_hop_neighbor (neighbor_ops.py:209-242): (nodes_list[L+1], adj_list[L]).  nodes_list[0] is
    `nodes` flattened, nodes_list[h+1] the distinct neighbors of hop h in first-occurrence order.  The reference's adjacency
    is a SparseTensor [len(nodes_list[h]), len(nodes_list[h+1])] of edge weights in (row, col) order; here it is ragged,
    (indptr i64[n+1], cols i64[nnz], weights f32[nnz]), entry k of row i being (i, cols[k]):
    torch.sparse_csr_tensor(indptr, cols, weights, size) builds the same matrix.  `sampler` is the object whose
    full_neighbor_adjacency runs each hop (this module by default)."""
    hop = full_neighbor_adjacency if sampler is None else sampler.full_neighbor_adjacency
    nodes = (_t(nodes, torch.int64) if sampler is None else torch.as_tensor(nodes, dtype=torch.int64)).reshape(-1)
    nodes_list, adj_list = [nodes], []
    for et in edge_types:
        nxt, indptr, cols, w = hop(nodes, et)
        nodes_list.append(nxt)
        adj_list.append((indptr, cols, w))
        nodes = nxt
    return nodes_list, adj_list


def graph_node_ids():
    """The node ids of the graph in engine-row order, i64[n]: row r of graph_adjacency is the node graph_node_ids()[r]."""
    out = torch.empty(get_graph().num_nodes, dtype=torch.int64, device=_dev())
    _call("eu_graph_node_ids", out)
    return out


def graph_node_rows(nodes):
    """The engine row of every node id, i64 of nodes' size; -1 for an id that is not a node."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    out = torch.empty_like(nodes)
    _call("eu_graph_node_rows", nodes, nodes.numel(), out)
    return out


def graph_adjacency(edge_types, rows=None, weights=False):
    """The adjacency of the resident graph with engine rows as columns, in one device op (include/euler_b200.h,
    eu_graph_adjacency).  rows: None (every row), a range(r0, r1) of engine rows, or a tensor of engine rows (-1 lists
    nothing).  Row i lists its node's neighbours as get_full_neighbor(node, edge_types) does, each as its engine row.
    Returns (indptr i64[R+1], cols i64[nnz], weights f32[nnz] or None, extra_ids i64[X]): a listed id that is not a node
    has column n + k with extra_ids[k] that id, k in first-occurrence order over this call's listing, so a chunked build
    numbers each chunk's absent ids on its own.  Two host syncs, three when some listed id is not a node."""
    et = get_edge_type_id(edge_types)
    n = get_graph().num_nodes
    if rows is None:
        rows = range(n)
    if isinstance(rows, range):
        if rows.step != 1 or not 0 <= rows.start <= rows.stop <= n:
            raise EulerError("graph_adjacency: rows must be a range of step 1 within [0, %d]" % n)
        row_list, r0, r1 = None, rows.start, rows.stop
    else:
        row_list = _t(rows, torch.int64).reshape(-1)
        r0, r1 = 0, row_list.numel()
    dev = _dev()
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    indptr = torch.empty(r1 - r0 + 1, dtype=torch.int64, device=dev)
    _call("eu_graph_adjacency", et, len(et), row_list, r0, r1, 0, 0, indptr, None, None, None, counts)
    nnz, absent = torch.stack([indptr[-1], counts[0]]).tolist()
    cols = torch.empty(nnz, dtype=torch.int64, device=dev)
    w = torch.empty(nnz, dtype=torch.float32, device=dev) if weights else None
    extra = torch.empty(absent, dtype=torch.int64, device=dev)
    if nnz:
        _call("eu_graph_adjacency", et, len(et), row_list, r0, r1, nnz, absent, indptr, cols, w, extra, counts)
    if absent:
        extra = extra[:int(counts[1].item())]
    return indptr, cols, w, extra


def sample_neighbor_layerwise(nodes, edge_types, count, default_node=-1, weight_func=''):
    """neighbor_ops.sample_neighbor_layerwise (neighbor_ops.py:72-77): nodes [batch, n] -> (neighbors i64[batch, count],
    adj f32[batch, n, count]); adj is the dense view of the reference's SparseTensor (1.0 where neighbors[b, k] is a neighbor of
    nodes[b, j]).  weight_func: '' or 'sqrt'."""
    nd = _t(nodes, torch.int64)
    if nd.dim() != 2:
        raise EulerError("sample_neighbor_layerwise: nodes must be [batch, n]")
    if weight_func not in ('', 'sqrt'):
        raise EulerError("sample_neighbor_layerwise: weight_func must be '' or 'sqrt' (local_sample_layer_op.cc:93-101)")
    nd = nd.contiguous()
    batch, n = nd.shape
    et = get_edge_type_id(edge_types)
    out = torch.empty((batch, int(count)), dtype=torch.int64, device=nd.device)
    adj = torch.empty((batch, n, int(count)), dtype=torch.float32, device=nd.device)
    _call("eu_sample_neighbor_layerwise", nd, batch, n, et, len(et), int(count), default_node, 1 if weight_func == 'sqrt' else 0,
          out, adj)
    return out, adj


def sparse_get_adj(nodes, nb_nodes, edge_types, n=-1, m=-1):
    """neighbor_ops.sparse_get_adj (neighbor_ops.py:33-36): nodes [batch * n], nb_nodes [batch * m] (n / m = -1: one batch row)
    -> f32[batch, n, m], the dense view of the reference's SparseTensor."""
    nd = _t(nodes, torch.int64).reshape(-1).contiguous()
    nb = _t(nb_nodes, torch.int64).reshape(-1).contiguous()
    N = nd.numel() if n == -1 else int(n)
    M = nb.numel() if m == -1 else int(m)
    batch = nd.numel() // max(N, 1)
    et = get_edge_type_id(edge_types)
    adj = torch.empty((batch, N, M), dtype=torch.float32, device=nd.device)
    _call("eu_sparse_get_adj", nd, nb, batch, N, M, et, len(et), adj)
    return adj


def _adj_coo(nd, nb, batch, N, M, et):
    """one eu_sparse_get_adj_coo: a host sync for the entry count (the output shape)"""
    dev = nd.device

    def alloc(nnz):
        return torch.empty((nnz, 3), dtype=torch.int64, device=dev), torch.empty(nnz, dtype=torch.int64, device=dev)
    _, _, (indices, values) = _ragged("eu_sparse_get_adj_coo", batch * N, alloc, nd, nb, batch, N, M, et, len(et))
    return indices, values, (batch, N, M)


def sparse_get_adj_coo(nodes, nb_nodes, edge_types, n=-1, m=-1):
    """neighbor_ops.sparse_get_adj (neighbor_ops.py:33-36) with the reference's SparseTensor as it is built
    (tf_euler/kernels/sparse_get_adj_op.cc:84-117): (indices i64[nnz, 3], values i64[nnz], dense_shape (batch, n, m)).
    Entry (b, j, k) = 1 iff nb_nodes[b, k] is a neighbor of nodes[b, j], in row-major order; a batch row without an entry
    (b, n-1, m-1) gets it with value 0.  Same arguments as sparse_get_adj."""
    nd = _t(nodes, torch.int64).reshape(-1).contiguous()
    nb = _t(nb_nodes, torch.int64).reshape(-1).contiguous()
    N = nd.numel() if n == -1 else int(n)
    M = nb.numel() if m == -1 else int(m)
    batch = nd.numel() // max(N, 1)
    return _adj_coo(nd, nb, batch, N, M, get_edge_type_id(edge_types))


def sample_neighbor_layerwise_coo(nodes, edge_types, count, default_node=-1, weight_func=''):
    """neighbor_ops.sample_neighbor_layerwise (neighbor_ops.py:72-77) with the adjacency as the reference's SparseTensor:
    (neighbors i64[batch, count], (indices i64[nnz, 3], values i64[nnz], dense_shape (batch, n, count))).  The draws (and the
    engine state they consume) are sample_neighbor_layerwise's; the adjacency is sparse_get_adj_coo of (nodes, neighbors),
    the rule sample_neighbor_layerwise_with_adj_op.cc:104-140 applies to the drawn neighbors.  A batch of zero nodes per row
    has no candidates: its neighbors are default_node and nothing is drawn."""
    nd = _t(nodes, torch.int64)
    if nd.dim() != 2:
        raise EulerError("sample_neighbor_layerwise_coo: nodes must be [batch, n]")
    if weight_func not in ('', 'sqrt'):
        raise EulerError("sample_neighbor_layerwise_coo: weight_func must be '' or 'sqrt' (local_sample_layer_op.cc:93-101)")
    nd = nd.contiguous()
    batch, n = nd.shape
    count = int(count)
    et = get_edge_type_id(edge_types)
    out = torch.empty((batch, count), dtype=torch.int64, device=nd.device)
    if n == 0:
        out.fill_(default_node)
    else:
        _call("eu_sample_neighbor_layerwise", nd, batch, n, et, len(et), count, default_node, 1 if weight_func == 'sqrt' else 0,
              out, None)
    return out, _adj_coo(nd.reshape(-1), out.reshape(-1), batch, n, count, et)


def gen_pair(paths, left_win_size, right_win_size):
    """walk_ops.gen_pair (tf_euler/kernels/gen_pair_op.cc): skip-gram pairs i64[B, n_pairs, 2] of walks i64[B, path_len]."""
    paths = _t(paths, torch.int64)
    if paths.dim() != 2:
        raise EulerError("gen_pair: paths must be [batch, path_len]")
    paths = paths.contiguous()
    B, plen = paths.shape
    pc = _lib.load().eu_gen_pair_count(plen, int(left_win_size), int(right_win_size))
    out = torch.empty((B, pc, 2), dtype=torch.int64, device=paths.device)
    _call("eu_gen_pair", paths, B, plen, int(left_win_size), int(right_win_size), out)
    return out


def sample_neighbor_api(nodes, edge_types, count):
    """euler::SampleNeighbor of the C++ api (api.cc:223-236): NO unique / gather -- a repeated id draws again.  Returns
    engine-form (ids i64[N,count], w, t); rows without a result are (0, 0.0, -1)."""
    return _neighbor_rows("eu_sample_neighbor_raw", nodes, edge_types, int(count))


def unique(ids):
    """tf.unique on the device (eu_unique): (values in first-occurrence order, inverse i32 with ids == values[inverse])."""
    ids = _t(ids, torch.int64).reshape(-1)
    n = ids.numel()
    vals = torch.empty(n, dtype=torch.int64, device=ids.device)
    inv = torch.empty(n, dtype=torch.int32, device=ids.device)
    cnt = torch.zeros(1, dtype=torch.int64, device=ids.device)
    _call("eu_unique", ids, n, vals, inv, cnt)
    return vals[:int(cnt.item())], inv


def sage_mean_aggregate(neighbor_ids, count, dim, out_dtype=torch.float32):
    """Fused get_dense_feature + scatter_mean for fixed-fanout blocks (SAGEConv's neighbor mean,
    tf_euler/python/convolution/sage_conv.py:33-38 over sage_dataflow.py:43-46 blocks).  Each neighbor contributes columns
    [0, min(dim, feat_dim)) of its whole stored feature row (every slot, concatenated), zeros beyond, and an id not in the
    graph contributes zeros.  That equals get_dense_feature(neighbor_ids, [0], [dim]) followed by scatter_mean only when the
    graph has one dense slot or dim <= slot 0's width.  out_dtype=torch.bfloat16 gives the f32 means rounded to nearest even
    on the device, bit for bit (summed and divided in f32, rounded once)."""
    code = _out_dtype("sage_mean_aggregate", out_dtype)
    ids = _t(neighbor_ids, torch.int64).reshape(-1)
    rows = ids.numel() // int(count)
    out = torch.empty((rows, int(dim)), dtype=out_dtype, device=ids.device)
    _call("eu_sage_mean_aggregate_out_dtype", ids, rows, int(count), int(dim), code, out)
    return out


# ------------------------------------------------------------------------------------ mp ops
def _raw_gather(params, indices):
    params = params.contiguous()
    out = torch.empty((indices.numel(), params.shape[1]), dtype=torch.float32, device=params.device)
    _call("eu_gather", params, params.shape[0], params.shape[1], indices, indices.numel(), out)
    return out


def _raw_scatter(name, updates, indices, size):
    updates = updates.contiguous()
    out = torch.empty((int(size), updates.shape[1]), dtype=torch.float32, device=updates.device)
    _call(name, updates, updates.shape[1], indices, indices.numel(), int(size), out)
    return out


class _Gather(torch.autograd.Function):
    """MPGather with gradient scatter_add(grad, indices, N) (mp_ops.py:39-43)."""

    @staticmethod
    def forward(ctx, params, indices):
        ctx.save_for_backward(indices)
        ctx.n = params.shape[0]
        return _raw_gather(params, indices)

    @staticmethod
    def backward(ctx, grad):
        (indices,) = ctx.saved_tensors
        return _raw_scatter("eu_scatter_add", grad, indices, ctx.n), None


class _ScatterAdd(torch.autograd.Function):
    """MPScatterAdd with gradient gather(grad, indices) (mp_ops.py:46-49)."""

    @staticmethod
    def forward(ctx, updates, indices, size):
        ctx.save_for_backward(indices)
        return _raw_scatter("eu_scatter_add", updates, indices, size)

    @staticmethod
    def backward(ctx, grad):
        (indices,) = ctx.saved_tensors
        return _raw_gather(grad, indices), None, None


class _ScatterMax(torch.autograd.Function):
    """MPScatterMax; gradient splits evenly among ties (mp_ops.py:52-62)."""

    @staticmethod
    def forward(ctx, updates, indices, size):
        out = _raw_scatter("eu_scatter_max", updates, indices, size)
        ctx.save_for_backward(updates, indices, out)
        ctx.size = size
        return out

    @staticmethod
    def backward(ctx, grad):
        updates, indices, out = ctx.saved_tensors
        indicators = (updates == _raw_gather(out, indices)).to(updates.dtype)
        num_selected = _raw_scatter("eu_scatter_add", indicators, indices, ctx.size)
        indicators = indicators / _raw_gather(num_selected, indices)
        return indicators * _raw_gather(grad, indices), None, None


def _f32(x):
    x = _t(x, torch.float32)
    return x if x.dim() == 2 else x.reshape(x.shape[0], -1)


def _check_f32(op, named, ndim=None):
    """raise unless every (name, value) of named is a float32 tensor (with ndim dimensions when given)"""
    for nm, t in named:
        if not torch.is_tensor(t) or t.dtype != torch.float32 or (ndim is not None and t.dim() != ndim):
            raise EulerError("%s: %s must be a %sfloat32 tensor" % (op, nm, "" if ndim is None else "%d-D " % ndim))


def _dst_src(op, edge_index):
    """(targets, sources) i32[E] of edge_index [2, E]"""
    ei = _t(edge_index, torch.int32)
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise EulerError("%s: edge_index must be [2, E]" % op)
    return ei[0].contiguous(), ei[1].contiguous()


def gather(params, indices):
    """mp_ops.gather = MPGather (mp_ops.py:27): out[i,:] = params[indices[i],:]."""
    return _Gather.apply(_f32(params), _t(indices, torch.int32).reshape(-1))


def scatter_add(updates, indices, size=None):
    """mp_ops.scatter_add = MPScatterAdd (mp_ops.py:28).  Bit for bit the reference's sums on a non-decreasing index; on any
    other index the sums are order-free float atomics, which flush subnormal updates and partial sums to zero."""
    return _ScatterAdd.apply(_f32(updates), _t(indices, torch.int32).reshape(-1), int(size))


def scatter_max(updates, indices, size=None):
    """mp_ops.scatter_max = MPScatterMax (mp_ops.py:29); output initialised to -1e9 and raised by strict `upd > out`: NaN never
    wins and values at or below -1e9 leave -1e9.  Bit for bit the reference's result on a non-decreasing index; on any other
    index too, except among equal zeros, where +0.0 wins over -0.0 in any order (the reference keeps the first of them).
    -0.0 beats every negative value on both paths."""
    return _ScatterMax.apply(_f32(updates), _t(indices, torch.int32).reshape(-1), int(size))


def scatter_mean(updates, indices, size=None):
    """mp_ops.scatter_mean (mp_ops.py:65-69): scatter_add / (scatter_add(ones) + 1e-7).
    Without autograd the fused kernel is used (same arithmetic)."""
    updates = _f32(updates)
    indices = _t(indices, torch.int32).reshape(-1)
    if not (torch.is_grad_enabled() and updates.requires_grad):
        return _raw_scatter("eu_scatter_mean", updates, indices, int(size))
    out = scatter_add(updates, indices, size)
    ep = 1e-7
    ones = torch.ones((updates.shape[0], 1), dtype=torch.float32, device=updates.device)
    count = scatter_add(ones, indices, size) + ep
    return out / count


def scatter_(op, updates, indices, size):
    """mp_ops.scatter_ (mp_ops.py:72-73)."""
    return globals()['scatter_' + op](updates, indices, size)


def scatter_softmax(updates, indices, size=None):
    """mp_ops.scatter_softmax (mp_ops.py:76-79)."""
    updates = _f32(updates)
    updates = updates - gather(scatter_max(updates, indices, size), indices)
    updates = torch.exp(updates)
    return updates / gather(scatter_add(updates, indices, size), indices)


def _raw_gat(h_src, s_dst, s_src, dst, src, n_dst, with_alpha):
    """one eu_gat_aggregate: (out f32[n_dst, H*C], alpha f32[E, H] or None)"""
    n_src, H = s_src.shape
    E = dst.numel()
    out = torch.empty((n_dst, h_src.shape[1]), dtype=torch.float32, device=h_src.device)
    alpha = torch.empty((E, H), dtype=torch.float32, device=h_src.device) if with_alpha else None
    _call("eu_gat_aggregate", h_src, s_dst, s_src, dst, src, E, n_dst, n_src, H, h_src.shape[1] // H, out, alpha)
    return out, alpha


class _GatAggregate(torch.autograd.Function):
    """eu_gat_aggregate / eu_gat_aggregate_backward.  Saves alpha [E, H], never the [E, H*C] messages."""

    @staticmethod
    def forward(ctx, h_src, s_dst, s_src, dst, src, n_dst):
        want_alpha = any(ctx.needs_input_grad[:3])
        out, alpha = _raw_gat(h_src, s_dst, s_src, dst, src, n_dst, want_alpha)
        if want_alpha:
            ctx.save_for_backward(h_src, s_dst, s_src, dst, src, alpha)
        ctx.dims = (n_dst, s_src.shape[0], s_src.shape[1], h_src.shape[1] // s_src.shape[1])
        return out

    @staticmethod
    def backward(ctx, grad):
        h_src, s_dst, s_src, dst, src, alpha = ctx.saved_tensors
        n_dst, n_src, H, C = ctx.dims
        grad = grad.contiguous()
        dev = grad.device
        g_h = torch.empty((n_src, H * C), dtype=torch.float32, device=dev)
        g_sd = torch.empty((n_dst, H), dtype=torch.float32, device=dev)
        g_ss = torch.empty((n_src, H), dtype=torch.float32, device=dev)
        _call("eu_gat_aggregate_backward", grad, h_src, alpha, s_dst, s_src, dst, src, dst.numel(), n_dst, n_src, H, C,
              g_h, g_sd, g_ss)
        return g_h, g_sd, g_ss, None, None, None


def gat_attention_aggregate(h_src, s_dst, s_src, edge_index, size):
    """GATConv's attention aggregation (gat_conv.py:53-78 with aggr='add', after its `fc`) in one fused device op:
        h_src f32[n_src, H*C]   source rows, heads concatenated per row
        s_dst f32[n_dst, H]     per-target scores att_i(x_target), s_src f32[n_src, H] per-source scores att_j(x_source)
        edge_index [2, E]       (target, source) per edge; size = (n_dst, n_src)
    out[i, h*C:(h+1)*C] = sum over edges (i, j) of alpha[e,h] * h_src[j, h-slice], alpha = scatter_softmax of
    leaky_relu(s_dst[i,h] + s_src[j,h], 0.2) over the edges of each target.  For non-decreasing edge_index[0] the result
    equals, bit for bit, the same composition of gather / scatter_softmax / scatter_add; the backward pass is deterministic.
    Synchronises once per call (whether edge_index[0] is sorted); an unsorted one costs a radix sort."""
    n_dst, n_src = int(size[0]), int(size[1])
    if any(not torch.is_tensor(t) or t.dim() != 2 for t in (h_src, s_dst, s_src)):
        raise EulerError("gat_attention_aggregate: h_src, s_dst and s_src must be 2-D tensors")
    h_src, s_dst, s_src = _f32(h_src), _f32(s_dst), _f32(s_src)
    H = s_dst.shape[1]
    if H < 1 or s_src.shape != (n_src, H) or s_dst.shape[0] != n_dst or h_src.shape[0] != n_src or h_src.shape[1] % H:
        raise EulerError("gat_attention_aggregate: need h_src [n_src, H*C], s_dst [n_dst, H], s_src [n_src, H]; got %s, %s, %s"
                         % (tuple(h_src.shape), tuple(s_dst.shape), tuple(s_src.shape)))
    dst, src = _dst_src("gat_attention_aggregate", edge_index)
    return _GatAggregate.apply(h_src, s_dst, s_src, dst, src, n_dst)


class _AdjacencyMean(torch.autograd.Function):
    """eu_adjacency_mean / eu_adjacency_mean_backward.  Saves its inputs only (the indices and x_neigh's row count)."""

    @staticmethod
    def forward(ctx, x_neigh, indptr, cols):
        m, D = x_neigh.shape
        n = indptr.numel() - 1
        out = torch.empty((n, D), dtype=torch.float32, device=x_neigh.device)
        _call("eu_adjacency_mean", x_neigh, m, indptr, cols, n, cols.numel(), D, out)
        ctx.save_for_backward(indptr, cols)
        ctx.m = m
        return out

    @staticmethod
    def backward(ctx, grad):
        indptr, cols = ctx.saved_tensors
        grad = grad.contiguous()
        n, D = grad.shape
        g = torch.empty((ctx.m, D), dtype=torch.float32, device=grad.device)
        _call("eu_adjacency_mean_backward", grad, indptr, cols, n, cols.numel(), ctx.m, D, g)
        return g, None, None


def adjacency_mean(x_neigh, adj):
    """The neighbour mean of the dense-combining sparse aggregators (sparse_aggregators.py:37-84) in one fused device op:
        x_neigh f32[m, D]    the neighbour rows
        adj                  (indptr i64[n+1], cols i64[nnz] [, weights]) as get_multi_hop_neighbor returns per hop; the
                             weights are ignored (upstream's _sparse_ones_like)
    out[i] = (sum of x_neigh[cols[k]] over row i's entries) / max(deg_i, 1e-7), f32[n, D]; a row without entries gives zeros.
    The sum runs in a fixed order (include/euler_b200.h): a row of at most 256 entries gives the bits of the plain
    left-to-right float32 sum.  The backward pass is deterministic.  Neither pass synchronises with the host."""
    indptr, cols = adj[0], adj[1]
    if not torch.is_tensor(x_neigh) or x_neigh.dim() != 2:
        raise EulerError("adjacency_mean: x_neigh must be a 2-D tensor")
    x_neigh = _f32(x_neigh)
    indptr, cols = _t(indptr, torch.int64).reshape(-1), _t(cols, torch.int64).reshape(-1)
    if indptr.numel() < 1:
        raise EulerError("adjacency_mean: indptr must hold n + 1 offsets")
    return _AdjacencyMean.apply(x_neigh, indptr, cols)


def _raw_agnn(x_src, nrm_dst, nrm_src, beta, dst, src, n_dst, with_alpha):
    """one eu_agnn_aggregate: (out f32[n_dst, dim], alpha f32[E] or None, cos f32[E] or None)"""
    n_src, dim = x_src.shape
    E = dst.numel()
    dev = x_src.device
    out = torch.empty((n_dst, dim), dtype=torch.float32, device=dev)
    alpha = torch.empty(E, dtype=torch.float32, device=dev) if with_alpha else None
    cos = torch.empty(E, dtype=torch.float32, device=dev) if with_alpha else None
    _call("eu_agnn_aggregate", x_src, nrm_dst, nrm_src, beta, dst, src, E, n_dst, n_src, dim, out, alpha, cos)
    return out, alpha, cos


class _AgnnAggregate(torch.autograd.Function):
    """eu_agnn_aggregate / eu_agnn_aggregate_backward.  Saves alpha and cos (8 B per edge), never [E, dim] messages."""

    @staticmethod
    def forward(ctx, x_src, nrm_dst, nrm_src, beta, dst, src, n_dst):
        want = any(ctx.needs_input_grad[:4])
        out, alpha, cos = _raw_agnn(x_src, nrm_dst, nrm_src, beta, dst, src, n_dst, want)
        if want:
            ctx.save_for_backward(x_src, nrm_dst, nrm_src, beta, dst, src, alpha, cos)
        ctx.n_dst = n_dst
        return out

    @staticmethod
    def backward(ctx, grad):
        x_src, nrm_dst, nrm_src, beta, dst, src, alpha, cos = ctx.saved_tensors
        n_src, dim = x_src.shape
        grad = grad.contiguous()
        g_x, g_ns = torch.empty_like(x_src), torch.empty_like(nrm_src)
        g_nd = torch.empty((ctx.n_dst, dim), dtype=torch.float32, device=grad.device)
        g_beta = torch.empty_like(beta)
        _call("eu_agnn_aggregate_backward", grad, x_src, nrm_dst, nrm_src, beta, alpha, cos, dst, src, dst.numel(), ctx.n_dst,
              n_src, dim, g_x, g_nd, g_ns, g_beta)
        return g_x, g_nd, g_ns, g_beta, None, None, None


def agnn_attention_aggregate(x_src, nrm_dst, nrm_src, beta, edge_index, size):
    """AGNNConv's attention aggregation (agnn_conv.py:32-54 with aggr='add') in one fused device op:
        x_src f32[n_src, D]     the source rows summed
        nrm_dst f32[n_dst, D]   the target rows' l2_normalize, nrm_src f32[n_src, D] the source rows' (not required to be
                                normalized: the op takes them as given)
        beta                    the trainable scalar, a one-element f32 tensor ([] or [1]), read on the device only
        edge_index [2, E]       (target, source) per edge; size = (n_dst, n_src)
    out[i] = sum over edges (i, j) of alpha[e] * x_src[j], alpha = scatter_softmax of beta * <nrm_dst[i], nrm_src[j]> over the
    edges of each target.  The cosine is summed in this op's fixed order (include/euler_b200.h); given it, for non-decreasing
    edge_index[0] the result equals, bit for bit, scatter_softmax / scatter_add composed from the ops above.  The backward
    pass is deterministic.  Synchronises once per call (whether edge_index[0] is sorted); an unsorted one costs a radix sort."""
    n_dst, n_src = int(size[0]), int(size[1])
    _check_f32("agnn_attention_aggregate", (("x_src", x_src), ("nrm_dst", nrm_dst), ("nrm_src", nrm_src), ("beta", beta)))
    if beta.numel() != 1:
        raise EulerError("agnn_attention_aggregate: beta must be a scalar (one element); got shape %s" % (tuple(beta.shape),))
    if any(t.dim() != 2 for t in (x_src, nrm_dst, nrm_src)):
        raise EulerError("agnn_attention_aggregate: x_src, nrm_dst and nrm_src must be 2-D tensors")
    dim = x_src.shape[1]
    if dim < 1 or x_src.shape[0] != n_src or nrm_src.shape != (n_src, dim) or nrm_dst.shape != (n_dst, dim):
        raise EulerError("agnn_attention_aggregate: need x_src and nrm_src [n_src, D] = [%d, D], nrm_dst [n_dst, D] = [%d, D]; "
                         "got %s, %s, %s" % (n_src, n_dst, tuple(x_src.shape), tuple(nrm_src.shape), tuple(nrm_dst.shape)))
    x_src, nrm_dst, nrm_src = _t(x_src, torch.float32), _t(nrm_dst, torch.float32), _t(nrm_src, torch.float32)
    b = _t(beta, torch.float32).reshape(1)
    dst, src = _dst_src("agnn_attention_aggregate", edge_index)
    return _AgnnAggregate.apply(x_src, nrm_dst, nrm_src, b, dst, src, n_dst)


def _raw_relation(x_src, matrix, rel, dst, src, n_dst):
    """one eu_relation_aggregate: out f32[n_dst, D]"""
    n_src, F = x_src.shape
    R, D = matrix.shape[0], matrix.shape[1]
    out = torch.empty((n_dst, D), dtype=torch.float32, device=x_src.device)
    _call("eu_relation_aggregate", x_src, matrix, rel, dst, src, dst.numel(), n_dst, n_src, R, D, F, out)
    return out


class _RelationAggregate(torch.autograd.Function):
    """eu_relation_aggregate / eu_relation_aggregate_backward.  Saves only its inputs: the backward pass finds the pairs and
    their sums again, never an [E, D] or [E, D, F] tensor."""

    @staticmethod
    def forward(ctx, x_src, matrix, rel, dst, src, n_dst):
        out = _raw_relation(x_src, matrix, rel, dst, src, n_dst)
        if any(ctx.needs_input_grad[:2]):
            ctx.save_for_backward(x_src, matrix, rel, dst, src)
        ctx.n_dst = n_dst
        return out

    @staticmethod
    def backward(ctx, grad):
        x_src, matrix, rel, dst, src = ctx.saved_tensors
        n_src, F = x_src.shape
        R, D = matrix.shape[0], matrix.shape[1]
        grad = grad.contiguous()
        g_x, g_m = torch.empty_like(x_src), torch.empty_like(matrix)
        _call("eu_relation_aggregate_backward", grad, x_src, matrix, rel, dst, src, dst.numel(), ctx.n_dst, n_src, R, D, F,
              g_x, g_m)
        return g_x, g_m, None, None, None, None


def relation_mean_aggregate(x_src, matrix, edge_attr, edge_index, size):
    """RelationConv's typed mean aggregation (relation_conv.py:53-70 with aggr='mean', up to apply_node) in one fused device op:
        x_src f32[n_src, F]      the source rows
        matrix f32[R, D, F]      one transform per relation
        edge_attr [E]            each edge's relation, in [0, R) (RelationDataFlow's e_id)
        edge_index [2, E]        (target, source) per edge; size = (n_dst, n_src)
    out[i] = mean over the edges e of target i of matrix[edge_attr[e]] @ x_src[edge_index[1][e]], with scatter_mean's
    divisor (count + 1e-7).  The edges are summed per (target, relation) pair before the transform, in this op's fixed order
    (include/euler_b200.h), so the result differs from the per-edge composition only in rounding; it is deterministic, and
    unsorted (target, relation) keys give the bits of the stably sorted edge list.  Gradients reach x_src and matrix.
    Synchronises once per call (twice when the keys are unsorted, which costs a radix sort)."""
    n_dst, n_src = int(size[0]), int(size[1])
    _check_f32("relation_mean_aggregate", (("x_src", x_src), ("matrix", matrix)))
    if x_src.dim() != 2 or matrix.dim() != 3:
        raise EulerError("relation_mean_aggregate: need x_src [n_src, F] (2-D) and matrix [R, D, F] (3-D); got %s, %s"
                         % (tuple(x_src.shape), tuple(matrix.shape)))
    R, D, F = matrix.shape
    if R < 1 or D < 1 or F < 1 or x_src.shape != (n_src, F):
        raise EulerError("relation_mean_aggregate: need x_src [n_src, F] = [%d, %d] and a non-empty matrix [R, D, F]; got %s, %s"
                         % (n_src, F, tuple(x_src.shape), tuple(matrix.shape)))
    if not torch.is_tensor(edge_attr) or edge_attr.dtype.is_floating_point or edge_attr.dtype.is_complex:
        raise EulerError("relation_mean_aggregate: edge_attr must be an integer tensor")
    dst, src = _dst_src("relation_mean_aggregate", edge_index)
    if edge_attr.numel() != dst.numel():
        raise EulerError("relation_mean_aggregate: edge_attr has %d entries for %d edges" % (edge_attr.numel(), dst.numel()))
    rel = _t(edge_attr, torch.int32).reshape(-1)
    return _RelationAggregate.apply(_t(x_src, torch.float32), _t(matrix, torch.float32), rel, dst, src, n_dst)


def _raw_dna(q, k, v, n0, n1, dst, src, n_dst, heads, with_alpha):
    """one eu_dna_aggregate: (out f32[n_dst, dim], alpha f32[E, H, H] or None)"""
    n_src, dim = k.shape
    E = dst.numel()
    out = torch.empty((n_dst, dim), dtype=torch.float32, device=q.device)
    alpha = torch.empty((E, heads, heads), dtype=torch.float32, device=q.device) if with_alpha else None
    _call("eu_dna_aggregate", q, k, v, n0, n1, dst, src, E, n_dst, n_src, heads, dim // heads, out, alpha)
    return out, alpha


class _DnaAggregate(torch.autograd.Function):
    """eu_dna_aggregate / eu_dna_aggregate_backward.  Saves its inputs and alpha (4 H^2 B per edge), never [E, dim] messages."""

    @staticmethod
    def forward(ctx, q, k, v, n0, n1, dst, src, n_dst, heads):
        want = any(ctx.needs_input_grad[:3])
        out, alpha = _raw_dna(q, k, v, n0, n1, dst, src, n_dst, heads, want)
        if want:
            ctx.save_for_backward(q, k, v, n0, n1, dst, src, alpha)
        ctx.dims = (n_dst, heads)
        return out

    @staticmethod
    def backward(ctx, grad):
        q, k, v, n0, n1, dst, src, alpha = ctx.saved_tensors
        n_dst, H = ctx.dims
        n_src, dim = k.shape
        grad = grad.contiguous()
        g_q, g_k, g_v = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _call("eu_dna_aggregate_backward", grad, q, k, v, n0, n1, alpha, dst, src, dst.numel(), n_dst, n_src, H, dim // H,
              g_q, g_k, g_v)
        return g_q, g_k, g_v, None, None, None, None, None, None


def dna_attention_aggregate(q, k, v, n0, n1, edge_index, size, heads):
    """DNAConv's attention aggregation (dna_conv.py:115-170 with aggr='mean', after lin_q / lin_k / lin_v) in one fused
    device op:
        q f32[n_dst, dim]        lin_q of the target rows; k, v f32[n_src, dim] lin_k / lin_v of the source rows
        n0 f32[n_dst] or [n_dst, 1], n1 f32[n_src] or [n_src, 1]   the deg^-1/2 norms of both sides (convolution.gcn_norm)
        edge_index [2, E]        (target, source) per edge; size = (n_dst, n_src); heads H divides dim, at most 8
    Per edge every query head is scored against every key head (<q_i[h], k_j[h']> / sqrt(C)), restricted_softmax runs over
    the key heads, and the message n0_i * n1_j * sum_h' a * v_j[h'] is averaged over each target's edges with
    scatter_mean's divisor.  The sums run in this op's fixed order (include/euler_b200.h): deterministic, and unsorted
    edge_index[0] gives the bits of the stably sorted edge list.  Gradients reach q, k and v; the norms get none.
    Synchronises once per call (whether edge_index[0] is sorted); an unsorted one costs a radix sort."""
    n_dst, n_src = int(size[0]), int(size[1])
    _check_f32("dna_attention_aggregate", (("q", q), ("k", k), ("v", v), ("n0", n0), ("n1", n1)))
    if any(t.dim() != 2 for t in (q, k, v)):
        raise EulerError("dna_attention_aggregate: q, k and v must be 2-D tensors")
    heads = int(heads)
    dim = q.shape[1]
    if heads < 1 or dim < 1 or dim % heads:
        raise EulerError("dna_attention_aggregate: dim = %d must be a positive multiple of heads = %d" % (dim, heads))
    if q.shape[0] != n_dst or k.shape != (n_src, dim) or v.shape != (n_src, dim):
        raise EulerError("dna_attention_aggregate: need q [n_dst, dim] = [%d, %d], k and v [n_src, dim] = [%d, %d]; got %s, %s, %s"
                         % (n_dst, dim, n_src, dim, tuple(q.shape), tuple(k.shape), tuple(v.shape)))
    for nm, t, n in (("n0", n0, n_dst), ("n1", n1, n_src)):
        if t.numel() != n or t.dim() not in (1, 2) or (t.dim() == 2 and t.shape[1] != 1):
            raise EulerError("dna_attention_aggregate: %s must be [%d] or [%d, 1]; got %s" % (nm, n, n, tuple(t.shape)))
    dst, src = _dst_src("dna_attention_aggregate", edge_index)
    q, k, v = (_t(t, torch.float32) for t in (q, k, v))
    n0, n1 = (_t(t, torch.float32).detach().reshape(-1) for t in (n0, n1))
    return _DnaAggregate.apply(q, k, v, n0, n1, dst, src, n_dst, heads)


# ------------------------------------------------------------------------------------ sparse table gradients
def _coo_buffers(entries, shape, dev):
    """the (rows i64[cap], values f32[cap, dim]) a sparse backward pass fills for a table of shape (n_rows, dim) that the
    batch reaches through `entries` lookups: cap = min(entries, n_rows), sized from the entries, never from a large table's
    rows.  (None, None) for an absent table (shape None)."""
    if shape is None:
        return None, None
    cap = min(entries, shape[0])
    return torch.empty(cap, dtype=torch.int64, device=dev), torch.empty((cap, shape[1]), dtype=torch.float32, device=dev)


def _coo(rows, vals, n, shape):
    """the coalesced sparse COO gradient of the first n rows / values of _coo_buffers' arrays (None for an absent table)"""
    if shape is None:
        return None
    return torch.sparse_coo_tensor(rows[:n].unsqueeze(0), vals[:n], tuple(shape), is_coalesced=True, check_invariants=False)


def _shape(table):
    return None if table is None else tuple(table.shape)


def table_proxy(table):
    """The gradient proxy of a bfloat16 table: a float32 leaf of the table's shape that requires grad and owns no [n_rows, dim]
    storage (one element, strides 0).  Given to sparse_feature_embedding, shallow_encode or shallow_encode_pool in the
    table's place, it receives the table's f32 gradient as a sparse COO tensor in .grad, summed over every use in the graph
    as autograd sums a sparse_grad=True table's; optimizers.minimize hands it to the optimizer, never rounded to bf16."""
    return torch.zeros(1, dtype=torch.float32, device=table.device).as_strided(tuple(table.shape), (0, 0)).requires_grad_()


def _table_dtype(op, named, mixed=None):
    """the storage dtype of the tables named [(name, table)], float32 when there are none: raises EulerError unless each is a
    2-D float32 or bfloat16 tensor, then unless all have one dtype (mixed(dtypes): that error's text, where the op words it)"""
    for nm, t in named:
        if not torch.is_tensor(t) or t.dtype not in _lib.TORCH_DTYPES or t.dim() != 2:
            raise EulerError("%s: %s must be a 2-D float32 or bfloat16 tensor" % (op, nm))
    dtypes = [t.dtype for _, t in named]
    if len(set(dtypes)) > 1:
        raise EulerError(mixed(dtypes) if mixed else "%s: the tables must have one dtype, got %s" % (op, [str(d) for d in dtypes]))
    return dtypes[0] if dtypes else torch.float32


def _check_tables(op, named, proxies=None):
    """the storage dtype of the embedding tables named [(name, table)] (None entries skipped): raise unless all are 2-D
    float32 or bfloat16 tensors of one dtype, no bf16 table requires grad, and proxies (None, or one entry per named table:
    None or a gradient proxy) gives proxies to bf16 tables only, each a float32 leaf of its table's shape that requires grad"""
    present = [(nm, t) for nm, t in named if t is not None]
    dt = _table_dtype(op, present)
    if dt == torch.bfloat16 and any(t.requires_grad for _, t in present):
        raise EulerError("%s: a bfloat16 table takes no autograd gradient (torch would round it to bf16); give it a gradient "
                         "proxy (table_proxy) and train it with optimizers.minimize" % op)
    proxies = [None] * len(named) if proxies is None else list(proxies)
    if len(proxies) != len(named):
        raise EulerError("%s: proxies needs one entry per table (%d), got %d" % (op, len(named), len(proxies)))
    for (nm, t), q in zip(named, proxies):
        if q is None:
            continue
        if t is None or t.dtype != torch.bfloat16:
            raise EulerError("%s: a gradient proxy stands in for a bfloat16 table only (%s)" % (op, nm))
        if not torch.is_tensor(q) or q.dtype != torch.float32 or tuple(q.shape) != tuple(t.shape) or not q.requires_grad \
                or q.device != t.device:
            raise EulerError("%s: the proxy of %s must be a float32 tensor of the table's shape %s on its device that requires "
                             "grad" % (op, nm, tuple(t.shape)))
    return dt, proxies


# ------------------------------------------------------------------------------------ sparse-feature embedding
_COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}


def _raw_embedding(nodes, fid, table, default_value, comb):
    """one eu_sparse_embedding_lookup (eu_sparse_embedding_lookup_dtype for a bf16 table): out f32[M, dim]"""
    n_rows, dim = table.shape
    out = torch.empty((nodes.numel(), dim), dtype=torch.float32, device=table.device)
    if table.dtype == torch.bfloat16:
        _call("eu_sparse_embedding_lookup_dtype", nodes, nodes.numel(), fid, default_value, table, n_rows, dim, comb, 1, out)
    else:
        _call("eu_sparse_embedding_lookup", nodes, nodes.numel(), fid, default_value, table, n_rows, dim, comb, out)
    return out


class _SparseEmbedding(torch.autograd.Function):
    """eu_sparse_embedding_lookup / eu_sparse_embedding_lookup_backward.  Saves only the node ids: the backward pass lists the
    entries again from the graph.  The gradient goes to the table, or to its proxy when one is given (then sparse)."""

    @staticmethod
    def forward(ctx, table, proxy, nodes, fid, default_value, comb, sparse_grad):
        out = _raw_embedding(nodes, fid, table, default_value, comb)
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            ctx.save_for_backward(nodes)
        ctx.args = (fid, default_value, comb, table.shape, sparse_grad or proxy is not None)
        return out

    @staticmethod
    def backward(ctx, grad):
        nodes, = ctx.saved_tensors
        fid, default_value, comb, (n_rows, dim), sparse_grad = ctx.args
        grad = grad.contiguous()
        args = (grad, nodes, nodes.numel(), fid, default_value, n_rows, dim, comb)
        if not sparse_grad:
            g_t = torch.empty((n_rows, dim), dtype=torch.float32, device=grad.device)
            _call("eu_sparse_embedding_lookup_backward", *args, g_t)
            return g_t, None, None, None, None, None, None
        rows, vals = _coo_buffers(_sparse_entries(nodes, fid), (n_rows, dim), grad.device)
        n = C.c_int64()
        _call("eu_sparse_embedding_lookup_backward_sparse", *args, rows, vals, C.byref(n))
        g_t = _coo(rows, vals, n.value, (n_rows, dim))
        return ((None, g_t) if ctx.needs_input_grad[1] else (g_t, None)) + (None,) * 5


def _sparse_entries(nodes, fid):
    """the entries get_sparse_feature lists for nodes in slot fid (a node without values counts one): one lengths pass and
    one read back"""
    return _ragged_lengths("eu_get_sparse_feature", nodes.numel(), nodes, nodes.numel(), int(fid), 0)[1]


def sparse_feature_embedding(nodes, feature_name, table, default_value, combiner='sum', sparse_grad=False, proxy=None):
    """SparseEmbedding over get_sparse_feature in one fused device op: row i is tf.nn.embedding_lookup_sparse(table, sp_ids,
    None, combiner) (layers.py:152-169) of the SparseTensor get_sparse_feature(nodes, [feature_name], [default_value]) returns,
    i.e. the rows of table f32[n_rows, dim] named by node i's uint64 values of the slot, in stored order, or the one row
    default_value for a node without values; combined by 'sum', 'mean' or 'sqrtn'.  The sum runs left to right from the first
    row, mean / sqrtn divide once (include/euler_b200.h).  Every value of the slot and default_value must lie in [0, n_rows):
    the call raises otherwise, before any device work.  The gradient reaches table only (deterministic, no atomics): a dense
    f32[n_rows, dim] gradient, or, with sparse_grad=True, a coalesced sparse COO gradient of the rows the batch touches (as
    nn.Embedding(sparse=True) gives), the same values without an [n_rows, dim] buffer.  The forward does not synchronise; the
    backward synchronises once (dense) or three times (sparse: sizing the COO, the entry count, the row count).
    A bfloat16 table is read widened exactly to f32, so the output is the f32 op's on the widened table.  It takes no
    gradient itself (one that requires grad raises); its gradient goes to `proxy` (table_proxy), a float32 leaf of the
    table's shape, as the coalesced f32 sparse COO gradient the f32 table gets with sparse_grad=True."""
    if combiner not in _COMBINERS:
        raise EulerError("sparse_feature_embedding: combiner must be one of %s, got %r" % (sorted(_COMBINERS), combiner))
    dt, (proxy,) = _check_tables("sparse_feature_embedding", [("table", table)], [proxy])
    fid = _slot(feature_name, get_graph().sparse_feature_id)
    nodes = _t(nodes, torch.int64).reshape(-1)
    return _SparseEmbedding.apply(_t(table, dt), proxy, nodes, fid, int(default_value), _COMBINERS[combiner], bool(sparse_grad))


# ------------------------------------------------------------------------------------ ShallowEncoder's input row
SHALLOW_COMBINERS = {'concat': 0, 'add': 1}


def _shallow_problem(nodes, id_table, dense, sparse, comb):
    """eu_shallow_problem of resolved inputs: dense [(fid, dim)], sparse [(fid, table, default, combiner code)]"""
    p = _lib.ShallowProblem()
    p.combiner, p.M, p.nodes = comb, nodes.numel(), nodes.data_ptr()
    if id_table is not None:
        p.id_table, p.n_id_rows, p.id_dim = id_table.data_ptr(), id_table.shape[0], id_table.shape[1]
    p.n_dense, p.n_sparse = len(dense), len(sparse)
    for j, (fid, dim) in enumerate(dense):
        p.dense[j].fid, p.dense[j].dim = fid, dim
    for k, (fid, table, default, c) in enumerate(sparse):
        q = p.sparse[k]
        q.fid, q.dim, q.combiner, q.default_value = fid, table.shape[1], c, default
        q.n_rows, q.table = table.shape[0], table.data_ptr()
    first = id_table if id_table is not None else (sparse[0][1] if sparse else None)
    p.table_dtype = _lib.TORCH_DTYPES[first.dtype] if first is not None else 0
    return p


def _shallow_inputs(who, nodes, id_table, dense, sparse, comb, sparse_grad, proxies):
    """shallow_encode's arguments checked and resolved: (nodes i64[M], _ShallowEncode's cfg, the id table, the slots'
    tables, the proxies in the table order (id table, slots): one per table, None where a table has none)"""
    g = get_graph()
    dense, sparse = list(dense), list(sparse)
    if len(dense) > _lib.SHALLOW_MAX_SLOTS or len(sparse) > _lib.SHALLOW_MAX_SLOTS:
        raise EulerError("%s: at most %d dense and %d sparse slots" % (who, _lib.SHALLOW_MAX_SLOTS, _lib.SHALLOW_MAX_SLOTS))
    tables = ([id_table] if id_table is not None else []) + [s[1] for s in sparse]
    named = [("id_table", id_table)] + [("sparse table %d" % k, s[1]) for k, s in enumerate(sparse)]
    dt, proxies = _check_tables(who, named, proxies)
    d_cfg = tuple((_slot(n, g.dense_feature_id), int(d)) for n, d in dense)
    s_cfg = []
    for s in sparse:
        name, _, dv = s[:3]
        c = s[3] if len(s) > 3 else 'sum'
        if c not in _COMBINERS:
            raise EulerError("%s: sparse combiner must be one of %s, got %r" % (who, sorted(_COMBINERS), c))
        s_cfg.append((_slot(name, g.sparse_feature_id), int(dv), _COMBINERS[c]))
    emb_dims = [t.shape[1] for t in tables]
    if comb == 1 and len(set(emb_dims)) > 1:
        raise EulerError("%s: 'add' needs one dim for every table, got %s" % (who, emb_dims))
    dense_w = sum(d for _, d in d_cfg)
    W = (emb_dims[0] if emb_dims else 0) if comb == 1 else sum(emb_dims) + dense_w
    nodes = _t(nodes, torch.int64).reshape(-1)
    id_t = _t(id_table, dt) if id_table is not None else None
    ts = [_t(s[1], dt) for s in sparse]
    # a proxy's gradient is the sparse COO one
    sparse_grad = bool(sparse_grad) or any(q is not None for q in proxies)
    return nodes, (d_cfg, tuple(s_cfg), comb, W, dense_w if comb == 1 else 0, sparse_grad), id_t, ts, proxies


def _route_grads(ctx, first, grads):
    """the backward's outputs for the tables at inputs first .. first + n - 1 and their proxies right after them: each
    table's gradient goes to its proxy when the proxy needs it, else to the table"""
    n = len(grads)
    to_proxy = [ctx.needs_input_grad[first + n + t] for t in range(n)]
    return tuple(None if p else g for g, p in zip(grads, to_proxy)) + tuple(g if p else None for g, p in zip(grads, to_proxy))


def _shallow_call(sym, p, *args):
    """eu_shallow_encode(_pool) over p, or its _dtype twin when the problem's tables are bf16"""
    if p.table_dtype:
        _call(sym + "_dtype", C.byref(p), p.table_dtype, *args)
    else:
        _call(sym, C.byref(p), *args)


def _shallow_backward(sym, extra, nodes, cfg, grad, id_table, tables):
    """the table gradients of a shallow problem through sym (dense) or sym + '_sparse' (cfg's sparse_grad), `extra` being the
    arguments between the problem and grad_out; in the order (id table, slots), None for an absent id table"""
    dense, sparse_cfg, comb, W, dense_w, sparse_grad = cfg
    sparse = [(fid, t, dv, c) for (fid, dv, c), t in zip(sparse_cfg, tables)]
    all_tables = [id_table] + list(tables)
    grad = grad.contiguous()
    p = _shallow_problem(nodes, id_table, dense, sparse, comb)
    if not sparse_grad:
        grads = [None if t is None else torch.empty_like(t) for t in all_tables]
        _call(sym, C.byref(p), *extra, grad, grads)
        return tuple(grads)
    # the id table has M entries, a slot its get_sparse_feature entries
    entries = [nodes.numel()] + [_sparse_entries(nodes, fid) for fid, _, _, _ in sparse]
    shapes = [_shape(t) for t in all_tables]
    bufs = [_coo_buffers(e, sh, nodes.device) for e, sh in zip(entries, shapes)]
    counts = (C.c_int64 * len(all_tables))()
    _call(sym + "_sparse", C.byref(p), *extra, grad, [r for r, _ in bufs], [v for _, v in bufs], counts)
    return tuple(_coo(r, v, counts[t], shapes[t]) for t, (r, v) in enumerate(bufs))


class _ShallowEncode(torch.autograd.Function):
    """eu_shallow_encode(_dtype) / eu_shallow_encode_backward(_sparse).  Saves the node ids only (and the tables, which are
    inputs): the backward pass lists every table's entries again from the graph.  Inputs after the configuration: the id
    table (None when absent), then one table per sparse slot, then one proxy (or None) per table in that order."""

    @staticmethod
    def forward(ctx, nodes, cfg, id_table, *tables_proxies):
        tables = tables_proxies[:(len(tables_proxies) - 1) // 2]
        dense, sparse_cfg, comb, W, dense_w, sparse_grad = cfg
        sparse = [(fid, t, dv, c) for (fid, dv, c), t in zip(sparse_cfg, tables)]
        M, dev = nodes.numel(), nodes.device
        out = torch.empty((M, W), dtype=torch.float32, device=dev)
        dense_out = torch.empty((M, dense_w), dtype=torch.float32, device=dev) if comb == 1 else None
        p = _shallow_problem(nodes, id_table, dense, sparse, comb)
        _shallow_call("eu_shallow_encode", p, out, dense_out)
        ctx.save_for_backward(nodes, id_table, *tables)
        ctx.cfg = cfg
        if dense_out is None:
            return out
        ctx.mark_non_differentiable(dense_out)
        return out, dense_out

    @staticmethod
    def backward(ctx, grad, *unused):
        nodes, id_table, *tables = ctx.saved_tensors
        grads = _shallow_backward("eu_shallow_encode_backward", (), nodes, ctx.cfg, grad, id_table, tables)
        return (None, None) + _route_grads(ctx, 2, grads)


def shallow_encode(nodes, id_table=None, dense=(), sparse=(), combiner='concat', sparse_grad=False, proxies=None):
    """ShallowEncoder's input row (tf_euler/python/utils/encoders.py:134-171) in one fused device op, for node ids of any shape
    (flattened to M):
        id_table    f32[n_id_rows, id_dim] or None: row nodes[i] (tf.nn.embedding_lookup; an id outside the table raises)
        dense       [(feature_name or slot id, dim)]: get_dense_feature(nodes, [name], [dim]) exactly (pad, clip, absent nodes)
        sparse      [(feature_name or slot id, table, default_value[, combiner])]: sparse_feature_embedding(nodes, name,
                    table, default_value, combiner) exactly (combiner 'sum' by default, as SparseEmbedding's)
    combiner 'concat' returns f32[M, W] = [id | dense_0 .. | sparse_0 ..].  'add' (every table one dim) returns (emb, feats):
    emb f32[M, dim] = id + sparse_0 + .. + sparse_last added left to right, and feats f32[M, sum of dense dims] = the dense
    part concatenated (None without dense slots), which the caller maps through its Dense layer and adds to emb.
    The gradient reaches the tables only (features are not trainable), deterministic, no atomics: dense gradients, or with
    sparse_grad=True coalesced sparse COO gradients of the rows the batch touches.  The forward synchronises once to check the
    ids when an id table is given, and not at all under CUDA-graph capture (include/euler_b200.h); the backward once (dense)
    or 2 + the slots (sparse).
    The tables may instead all be bfloat16, read widened exactly to f32: the rows are the f32 op's on the widened tables.
    A bf16 table takes no gradient itself (one that requires grad raises).  proxies (None, or one entry per table in the
    order id table, then the slots: None or table_proxy(table)) are float32 leaves that take each bf16 table's gradient,
    the coalesced f32 sparse COO gradient an f32 table holding the widened values gets with sparse_grad=True."""
    if combiner not in SHALLOW_COMBINERS:
        raise EulerError("shallow_encode: combiner must be one of %s, got %r" % (sorted(SHALLOW_COMBINERS), combiner))
    comb = SHALLOW_COMBINERS[combiner]
    nodes, cfg, id_t, ts, qs = _shallow_inputs("shallow_encode", nodes, id_table, dense, sparse, comb, sparse_grad, proxies)
    d_cfg = cfg[0]
    res = _ShallowEncode.apply(nodes, cfg, id_t, *ts, *qs)
    if comb == 0:
        return res
    out, feats = res
    return out, (feats if d_cfg else None)


POOLS = {'sum': 0, 'mean': 1}


class _ShallowEncodePool(torch.autograd.Function):
    """eu_shallow_encode_pool(_dtype) / eu_shallow_encode_pool_backward(_sparse): _ShallowEncode's inputs ('concat', the
    proxies included), with the segment length and the pool code.  Saves the node ids only (and the tables, which are
    inputs)."""

    @staticmethod
    def forward(ctx, nodes, cfg, count, pool, id_table, *tables_proxies):
        tables = tables_proxies[:(len(tables_proxies) - 1) // 2]
        dense, sparse_cfg, comb, W = cfg[:4]
        sparse = [(fid, t, dv, c) for (fid, dv, c), t in zip(sparse_cfg, tables)]
        out = torch.empty((nodes.numel() // max(count, 1), W), dtype=torch.float32, device=nodes.device)   # count < 1 is refused below
        p = _shallow_problem(nodes, id_table, dense, sparse, comb)
        _shallow_call("eu_shallow_encode_pool", p, count, pool, out)
        ctx.save_for_backward(nodes, id_table, *tables)
        ctx.cfg = (cfg, count, pool)
        return out

    @staticmethod
    def backward(ctx, grad):
        nodes, id_table, *tables = ctx.saved_tensors
        cfg, count, pool = ctx.cfg
        grads = _shallow_backward("eu_shallow_encode_pool_backward", (count, pool), nodes, cfg, grad, id_table, tables)
        return (None, None, None, None) + _route_grads(ctx, 4, grads)


def shallow_encode_pool(nodes, count, id_table=None, dense=(), sparse=(), pool='mean', sparse_grad=False, proxies=None):
    """The 'concat' rows of shallow_encode pooled over consecutive segments of `count` nodes, in one fused device op: what
    SageEncoder's first layer needs of the deepest hop of sample_fanout (count = the last fanout).  nodes (any shape, M =
    R * count ids when flattened), id_table, dense and sparse are shallow_encode's; returns f32[R, W], row r the 'sum' or
    'mean' of the rows shallow_encode(nodes)[r * count : (r + 1) * count], every node counted (absent ones and default_node
    too, as reduce_mean(axis=1) counts them).  The [M, W] matrix is never written, in either direction.  Fixed order
    (include/euler_b200.h): each column is added left to right from the segment's first row, mean divides once by count.
    Gradients reach the tables only, as shallow_encode's (dense, or coalesced sparse COO with sparse_grad=True), with the
    same synchronisations.  count is at least 1, divides M and is at most 512 (EU_SHALLOW_POOL_MAX_COUNT).  bfloat16
    tables and their proxies as shallow_encode's."""
    if pool not in POOLS:
        raise EulerError("shallow_encode_pool: pool must be one of %s, got %r" % (sorted(POOLS), pool))
    nodes, cfg, id_t, ts, qs = _shallow_inputs("shallow_encode_pool", nodes, id_table, dense, sparse, 0, sparse_grad, proxies)
    return _ShallowEncodePool.apply(nodes, cfg, int(count), POOLS[pool], id_t, *ts, *qs)


# ------------------------------------------------------------------------------------ embedding stores
def _store_table(op, named):
    """the tables a store op updates in place: 2-D, contiguous, on the graph's device, all float32 or all bfloat16; returns
    that dtype.  Each table is checked whole before the next."""
    for i, (nm, t) in enumerate(named):
        try:
            dt = _table_dtype(op, named[:i + 1])
        except EulerError:
            raise EulerError("%s: %s must be 2-D float32 or bfloat16 tensors of one dtype"
                             % (op, " and ".join(nm for nm, _ in named))) from None
        if not t.is_contiguous() or t.device != _dev():
            raise EulerError("%s: %s must be contiguous on %s" % (op, nm, _dev()))
    return dt


def store_exchange(store, grad_store, ids, rows):
    """The store update of ScalableSageEncoder / ScalableGCNEncoder's training step (encoders.py:370-408, 710-748), in place
    and in one device op, for ids i64[M] (any shape) in [0, n_rows) and rows f32[M, dim]:
        store[ids[i]] = rows[i]   the LAST occurrence of a repeated id wins
        taken[i] = grad_store[ids[i]] as it was before the call, for every i; then grad_store[ids[i]] = 0
    store and grad_store are f32[n_rows, dim], or both bfloat16: the store row is then rounded to nearest even and taken is
    the gradient row widened exactly (include/euler_b200.h, eu_store_exchange_dtype).  Returns taken f32[M, dim].  No
    autograd: rows is read detached.  An id outside the tables raises before either is written (one host synchronisation;
    none under CUDA-graph capture)."""
    dt = _store_table("store_exchange", (("store", store), ("grad_store", grad_store)))
    _check_f32("store_exchange", (("rows", rows),), 2)
    ids = _t(ids, torch.int64).reshape(-1)
    n_rows, dim = store.shape
    if tuple(grad_store.shape) != (n_rows, dim) or tuple(rows.shape) != (ids.numel(), dim):
        raise EulerError("store_exchange: need store and grad_store [n_rows, dim], rows [M, dim]; got %s, %s, %s for M = %d"
                         % (tuple(store.shape), tuple(grad_store.shape), tuple(rows.shape), ids.numel()))
    rows = _t(rows.detach(), torch.float32)
    taken = torch.empty((ids.numel(), dim), dtype=torch.float32, device=store.device)
    if dt == torch.bfloat16:
        _call("eu_store_exchange_dtype", store, grad_store, n_rows, dim, ids, ids.numel(), rows, taken, 1)
    else:
        _call("eu_store_exchange", store, grad_store, n_rows, dim, ids, ids.numel(), rows, taken)
    return taken


def store_accumulate(grad_store, ids, grad, count=1, pool='mean', seed=0, step=None, tensor=0):
    """The gradient-store update of ScalableSageEncoder / ScalableGCNEncoder (tf.scatter_add, encoders.py:382-389), in place
    and in one device op: grad_store[ids[e]] += grad[e // count] (divided by count under pool='mean'), for ids i64[M] (any
    shape) in [0, n_rows), grad f32[M / count, dim] and grad_store f32[n_rows, dim].  That is the gradient of
    shallow_encode_pool(ids, count, id_table=store, pool=pool) (count = 1: of shallow_encode(ids, id_table=store)), summed per
    distinct id in that op's fixed order and added to the stored row with one rounding: deterministic, no atomics.  No
    autograd.  An id outside the table raises before it is written (one host synchronisation; none under capture).
    grad_store may be bfloat16 (grad stays float32): the same sum is added to the widened row in f32 and written back by
    stochastic rounding keyed by (seed, step, tensor, element), step an int64 device scalar the caller advances once per
    step, as optim_momentum_'s (include/euler_b200.h, eu_store_accumulate_dtype)."""
    op = "store_accumulate"
    if pool not in POOLS:
        raise EulerError("store_accumulate: pool must be one of %s, got %r" % (sorted(POOLS), pool))
    dt = _store_table(op, (("grad_store", grad_store),))
    _check_f32(op, (("grad", grad),), 2)
    ids = _t(ids, torch.int64).reshape(-1)
    n_rows, dim = grad_store.shape
    count = int(count)
    if count < 1 or ids.numel() % count or tuple(grad.shape) != (ids.numel() // count, dim):
        raise EulerError("store_accumulate: need count >= 1 dividing M = %d and grad [M / count, %d]; got count %d, grad %s"
                         % (ids.numel(), dim, count, tuple(grad.shape)))
    grad = _t(grad.detach(), torch.float32)
    if dt == torch.bfloat16:
        _call("eu_store_accumulate_dtype", grad_store, n_rows, dim, ids, ids.numel(), count, POOLS[pool], grad,
              *_sr_args(op, grad_store, seed, step, tensor))
    else:
        _call("eu_store_accumulate", grad_store, n_rows, dim, ids, ids.numel(), count, POOLS[pool], grad)


# ------------------------------------------------------------------------------------ graph-level minibatches
def _labels_from(fn, *args):
    """the label list a two-call entry point reports (counts, then offsets and bytes), as bytes"""
    n, nb = C.c_int64(), C.c_int64()
    check(fn(*args, 0, C.byref(n), C.byref(nb), None, None))
    ptr = np.zeros(n.value + 1, np.int64)
    buf = np.zeros(max(nb.value, 1), np.uint8)
    check(fn(*args, nb.value, C.byref(n), C.byref(nb), ptr.ctypes.data, buf.ctypes.data))
    raw = buf[:nb.value].tobytes()
    return [raw[ptr[i]:ptr[i + 1]] for i in range(n.value)]


def graph_labels():
    """The graph's label list (Graph::GetGraphLabel, graph.cc:439-457) as bytes, in the reference's order: the values of the
    binary slot 'graph_label', b'' included when a node has none.  Label indices (sample_graph_label) index this list."""
    return _labels_from(_lib.load().eu_graph_labels, get_graph()._h)


def inspect_graph_labels(data_path):
    """The label list of an Euler directory, read on the host without a device (the same list and order as graph_labels)."""
    return _labels_from(_lib.load().eu_graph_labels_inspect, str(data_path).encode())


def sample_graph_label(count):
    """sample_ops.sample_graph_label (kernel sample_graph_label_op.cc): i32[count] label indices into graph_labels(), drawn
    uniformly from this thread's engine (the same stream position as the reference's ThreadLocalRandom under rng='minstd')."""
    count = int(count)
    out = torch.empty(count, dtype=torch.int32, device=_dev())
    _call("eu_sample_graph_label", count, out)
    return out


def get_graph_by_label(labels):
    """sample_ops.get_graph_by_label (tf_euler/kernels/get_graph_by_label_op.cc).  labels: the label indices of
    sample_graph_label (a tensor), or a sequence of label strings (mapped on the host; a label the graph does not know is -1).
    Returns the reference's SparseTensor content as (indices i64[nnz, 2], values i64[nnz], dense_shape (B, max_len)): row i
    lists the node ids of graph i in ascending order; an unknown label or one without nodes gets the single entry (i, 0) = 0."""
    if not isinstance(labels, torch.Tensor):
        index = {v: i for i, v in enumerate(graph_labels())}
        labels = [index.get(v if isinstance(v, bytes) else str(v).encode(), -1) for v in labels]
    labels = _t(labels, torch.int32).reshape(-1)
    B = labels.numel()
    ptr = torch.empty(B + 1, dtype=torch.int64, device=labels.device)
    total, max_len = C.c_int64(), C.c_int64()
    _call("eu_get_graph_by_label", labels, B, 0, ptr, None, None, C.byref(total), C.byref(max_len))
    nnz = total.value
    indices = torch.empty((nnz, 2), dtype=torch.int64, device=labels.device)
    values = torch.empty(nnz, dtype=torch.int64, device=labels.device)
    if nnz:
        _call("eu_get_graph_by_label", labels, B, nnz, ptr, indices, values, None, None)
    return indices, values, (B, max_len.value)


def _raw_readout(x, index, size, logits, q):
    """one eu_graph_attention_readout: (out f32[size, D], alpha f32[N])"""
    N, D = x.shape
    out = torch.empty((size, D), dtype=torch.float32, device=x.device)
    alpha = torch.empty(N, dtype=torch.float32, device=x.device)
    _call("eu_graph_attention_readout", x, index, N, size, D, logits, q, out, alpha)
    return out, alpha


class _GraphReadout(torch.autograd.Function):
    """eu_graph_attention_readout / _backward.  Saves alpha [N], never an [N, D] temporary."""

    @staticmethod
    def forward(ctx, x, weight, index, size, by_query):
        out, alpha = _raw_readout(x, index, size, None if by_query else weight, weight if by_query else None)
        ctx.save_for_backward(x, weight, index, alpha)
        ctx.size, ctx.by_query = size, by_query
        return out

    @staticmethod
    def backward(ctx, grad):
        x, weight, index, alpha = ctx.saved_tensors
        N, D = x.shape
        grad = grad.contiguous()
        g_x = torch.empty_like(x)
        g_w = torch.empty_like(weight)
        by_query = ctx.by_query
        _call("eu_graph_attention_readout_backward", grad, x, index, N, ctx.size, D, weight if by_query else None, alpha, g_x,
              None if by_query else g_w, g_w if by_query else None)
        return g_x, g_w, None, None, None


def graph_attention_readout(x, index, size, logits=None, q=None):
    """The attention readout of the graph pools in one fused device op (tf_euler/python/graph_pool/):
        x f32[N, D]          the rows of every graph of the batch
        index [N]            each row's graph, in [0, size)
        logits f32[N] or [N, 1]   AttentionPool's gate, or
        q f32[size, D]       Set2SetPool's query: the logit of row n is <x_n, q[index_n]>
    out[b] = sum over the rows n of graph b of alpha_n * x_n, alpha = scatter_softmax of the logits over each graph; a graph
    without rows gets a zero row.  The sums are fixed-order chunked sums (include/euler_b200.h): for graphs of at most 256 rows
    and a non-decreasing index they equal scatter_softmax / scatter_add composed from the ops above bit for bit.  The backward
    pass is deterministic.  Synchronises once per call (whether index is sorted); an unsorted one costs a radix sort."""
    if (logits is None) == (q is None):
        raise EulerError("graph_attention_readout: give exactly one of logits and q")
    _check_f32("graph_attention_readout", (("x", x),), 2)
    size = int(size)
    x = _f32(x)
    index = _t(index, torch.int32).reshape(-1)
    if index.numel() != x.shape[0]:
        raise EulerError("graph_attention_readout: index has %d rows, x %d" % (index.numel(), x.shape[0]))
    if q is not None:
        w = _f32(q)
        if tuple(w.shape) != (size, x.shape[1]):
            raise EulerError("graph_attention_readout: q must be [size, D] = %s, got %s" % ((size, x.shape[1]), tuple(w.shape)))
    else:
        w = _t(logits, torch.float32).reshape(-1)
        if w.numel() != x.shape[0]:
            raise EulerError("graph_attention_readout: logits has %d rows, x %d" % (w.numel(), x.shape[0]))
    return _GraphReadout.apply(x, w, index, size, q is not None)


# ------------------------------------------------------------------------------------ unsupervised skip-gram step
SKIPGRAM_METRICS = ('mrr', 'hit1', 'hit3', 'hit10', 'mr')


def skipgram_metric(rank, name):
    """metrics.py's ranking metrics (utils/metrics.py mrr_score, hitk_score, mr_score) from rank [B], the position of each row's
    last positive among its logits:
        mrr   mean of 1 / (rank + 1), in float32
        hitK  mean of (rank < K), K in 1, 3, 10
        mr    tf.reduce_mean of the int64 ranks: an INTEGER mean (the sum divided by B, rounded toward zero), int64, as upstream
    A batch of no rows gives NaN for mrr and hitK and 0 for mr."""
    if name == 'mrr':
        return torch.reciprocal((rank + 1).to(torch.float32)).mean()
    if name in ('hit1', 'hit3', 'hit10'):
        return (rank < int(name[3:])).to(torch.float32).mean()
    if name == 'mr':
        r = rank.to(torch.int64)
        return torch.div(r.sum(), max(r.numel(), 1), rounding_mode='trunc')
    raise EulerError("skipgram metric must be one of %s, got %r" % (SKIPGRAM_METRICS, name))


def _raw_skipgram(src, pos, negs, target, context):
    """one eu_skipgram_loss (eu_skipgram_loss_dtype for bf16 tables): (logits f32[B, P + K], rank i32[B], loss f32[])"""
    B, P = pos.shape
    K = negs.shape[1]
    n_rows, dim = target.shape
    logits = torch.empty((B, P + K), dtype=torch.float32, device=target.device)
    rank = torch.empty(B, dtype=torch.int32, device=target.device)
    loss = torch.empty((), dtype=torch.float32, device=target.device)
    if target.dtype == torch.bfloat16:
        _call("eu_skipgram_loss_dtype", src, pos, negs, B, P, K, target, context, n_rows, dim, 1, logits, rank, loss)
    else:
        _call("eu_skipgram_loss", src, pos, negs, B, P, K, target, context, n_rows, dim, logits, rank, loss)
    return logits, rank, loss


def _raw_skipgram_sparse_grads(src, pos, negs, target, context, logits, g, shared):
    """one eu_skipgram_loss_backward_sparse(_dtype): [(rows i64[D], values f32[D, dim])] of the target table and, unless
    shared, of the context table, coalesced; g is the loss's upstream gradient (a device f32[1])"""
    B, P = pos.shape
    K = negs.shape[1]
    n_rows, dim = target.shape
    shape_t, shape_c = (n_rows, dim), None if shared else (n_rows, dim)
    rows_t, vals_t = _coo_buffers(B * (P + K + 1) if shared else B, shape_t, target.device)
    rows_c, vals_c = _coo_buffers(B * (P + K), shape_c, target.device)
    n_t, n_c = C.c_int64(), C.c_int64()
    args = (g, src, pos, negs, B, P, K, target, context, n_rows, dim)
    outs = (logits, rows_t, vals_t, C.byref(n_t), rows_c, vals_c, C.byref(n_c))
    if target.dtype == torch.bfloat16:
        _call("eu_skipgram_loss_backward_sparse_dtype", *args, 1, *outs)
    else:
        _call("eu_skipgram_loss_backward_sparse", *args, *outs)
    grads = [(rows_t[:n_t.value], vals_t[:n_t.value])]
    return grads if shared else grads + [(rows_c[:n_c.value], vals_c[:n_c.value])]


class _SkipgramLoss(torch.autograd.Function):
    """eu_skipgram_loss / eu_skipgram_loss_backward(_sparse).  Saves the ids and the logits (and the tables themselves, which
    are inputs): no [B, P + K, dim] rows are kept.  shared: target and context are one table, whose gradient is computed as
    one list and returned for the target input only."""

    @staticmethod
    def forward(ctx, target, context, src, pos, negs, shared, sparse_grad):
        logits, rank, loss = _raw_skipgram(src, pos, negs, target, context)
        ctx.save_for_backward(target, context, src, pos, negs, logits)
        ctx.shared, ctx.sparse_grad = shared, sparse_grad
        ctx.mark_non_differentiable(rank)
        return loss, rank

    @staticmethod
    def backward(ctx, g_loss, g_rank):
        target, context, src, pos, negs, logits = ctx.saved_tensors
        B, P = pos.shape
        K = negs.shape[1]
        n_rows, dim = target.shape
        dev = target.device
        g = g_loss.to(device=dev, dtype=torch.float32).reshape(1).contiguous()
        args = (g, src, pos, negs, B, P, K, target, context, n_rows, dim, logits)
        if not ctx.sparse_grad:
            g_t = torch.empty((n_rows, dim), dtype=torch.float32, device=dev)
            g_c = g_t if ctx.shared else torch.empty((n_rows, dim), dtype=torch.float32, device=dev)
            _call("eu_skipgram_loss_backward", *args, g_t, g_c)
            return g_t, None if ctx.shared else g_c, None, None, None, None, None
        # a shared table takes the target and the context entries in one list
        shape_t, shape_c = (n_rows, dim), None if ctx.shared else (n_rows, dim)
        rows_t, vals_t = _coo_buffers(B * (P + K + 1) if ctx.shared else B, shape_t, dev)
        rows_c, vals_c = _coo_buffers(B * (P + K), shape_c, dev)
        n_t, n_c = C.c_int64(), C.c_int64()
        _call("eu_skipgram_loss_backward_sparse", *args, rows_t, vals_t, C.byref(n_t), rows_c, vals_c, C.byref(n_c))
        return _coo(rows_t, vals_t, n_t.value, shape_t), _coo(rows_c, vals_c, n_c.value, shape_c), None, None, None, None, None


def _skipgram_args(op, src, pos, negs, target, context, metric):
    """(src [B], pos [B, P], negs [B, K], target, context, shared) on the device, or EulerError: the checks of
    skipgram_xent_loss"""
    if metric not in SKIPGRAM_METRICS:
        raise EulerError("%s: metric must be one of %s, got %r" % (op, SKIPGRAM_METRICS, metric))
    shared = context is target
    _table_dtype(op, (('target', target), ('context', context)),
                 lambda d: "%s: target (%s) and context (%s) must have one dtype" % (op, d[0], d[1]))
    if target.shape != context.shape:
        raise EulerError("%s: target %s and context %s must have one shape" % (op, tuple(target.shape), tuple(context.shape)))
    src = _t(src, torch.int64).reshape(-1)
    B = src.numel()
    pos, negs = _t(pos, torch.int64), _t(negs, torch.int64)
    if pos.dim() == 1:
        pos = pos.unsqueeze(1)
    if pos.dim() != 2 or negs.dim() != 2 or pos.shape[0] != B or negs.shape[0] != B or pos.shape[1] < 1:
        raise EulerError("%s: pos must be [B, P >= 1] and negs [B, K] with B = %d, got %s and %s"
                         % (op, B, tuple(pos.shape), tuple(negs.shape)))
    target = _t(target, target.dtype)
    context = target if shared else _t(context, context.dtype)
    return src, pos.contiguous(), negs.contiguous(), target, context, shared


def skipgram_xent_loss(src, pos, negs, target, context, metric='mrr', sparse_grad=False):
    """The skip-gram step of UnsuperviseModel.__call__ (mp_utils/base.py:50-91; PosNegLogits, xent_loss, utils/metrics.py) in
    one fused device op, for id embeddings:
        src [B] or [B, 1]    target-table rows        pos [B, P] or [B]   context-table rows of the positives (P >= 1)
        negs [B, K]          context-table rows of the negatives (K >= 0)
        target, context      f32[n_rows, dim] tables; passing one tensor twice is LINE's first order (one shared table)
    Returns (loss, metric): loss is the mean sigmoid cross-entropy over the B (P + K) logits (positives labelled 1), metric the
    ranking metric `metric` (skipgram_metric) of each row's last positive among its P + K logits, ties ranked as TF's stable
    top_k ranks them.  Ids index the tables directly, as tf.nn.embedding_lookup does; one outside [0, n_rows) raises.
    The gradient reaches the tables only: dense f32[n_rows, dim] gradients, or, with sparse_grad=True, coalesced sparse COO
    gradients of the rows the batch touches (as nn.Embedding(sparse=True) gives).  Deterministic, no atomics; the forward and the
    backward synchronise once each.
    bfloat16 tables (both of one dtype) are read widened exactly to f32, so the loss and metric are the f32 op's on the widened
    tables.  They take no gradient through autograd, which would round their f32 gradient to nearest bf16: a bf16 table that
    requires grad raises.  Train them with skipgram_xent_loss_sparse_grads and an optimizer's apply_sparse
    (UnsuperviseModel.train_step)."""
    src, pos, negs, target, context, shared = _skipgram_args("skipgram_xent_loss", src, pos, negs, target, context, metric)
    if target.dtype == torch.bfloat16 and (target.requires_grad or context.requires_grad):
        raise EulerError("skipgram_xent_loss: a bfloat16 table takes no autograd gradient (torch would round it to bf16); "
                         "train it with skipgram_xent_loss_sparse_grads and an optimizer's apply_sparse")
    loss, rank = _SkipgramLoss.apply(target, context, src, pos, negs, shared, bool(sparse_grad))
    return loss, skipgram_metric(rank, metric)


def skipgram_xent_loss_sparse_grads(src, pos, negs, target, context, metric='mrr'):
    """skipgram_xent_loss's forward and its sparse backward for an upstream gradient of 1, without autograd, for tables of
    float32 or bfloat16 (read widened exactly to f32).  Returns (loss, metric, grads): grads is [(rows i64[D], values
    f32[D, dim])], the coalesced f32 gradient of the target table, then of the context table unless it is the target
    table -- the bits skipgram_xent_loss(..., sparse_grad=True).backward() gives f32 tables holding the widened values.  They
    go to an optimizer's apply_sparse as they are, never rounded to bf16.  Synchronises twice (the forward, the backward)."""
    src, pos, negs, target, context, shared = _skipgram_args("skipgram_xent_loss_sparse_grads", src, pos, negs, target, context,
                                                             metric)
    target, context = target.detach(), context.detach()
    logits, rank, loss = _raw_skipgram(src, pos, negs, target, context)
    g = torch.ones(1, dtype=torch.float32, device=target.device)
    grads = _raw_skipgram_sparse_grads(src, pos, negs, target, context, logits, g, shared)
    return loss, skipgram_metric(rank, metric), grads


# ------------------------------------------------------------------------------------ graph auto-encoder step
class _GaeLoss(torch.autograd.Function):
    """eu_gae_loss / eu_gae_loss_backward over the sets (src, pos, negs) of mu, log_var (or None) and noise (or None).  Saves
    the inputs and the [B, 2K] logits; the reparameterised rows are never written."""

    @staticmethod
    def forward(ctx, radius, emb, pos, neg, lv_e, lv_p, lv_n, nz_e, nz_p, nz_n):
        B, K, D = pos.shape
        mu, lv, nz = [emb, pos, neg], [lv_e, lv_p, lv_n], [nz_e, nz_p, nz_n]
        lv, nz = (lv if lv_e is not None else None), (nz if nz_e is not None else None)
        logits = torch.empty((B, 2 * K), dtype=torch.float32, device=emb.device)
        loss = torch.empty((), dtype=torch.float32, device=emb.device)
        correct = torch.empty((), dtype=torch.int64, device=emb.device)
        _call("eu_gae_loss", B, K, D, mu, lv, nz, radius, logits, loss, correct)
        ctx.save_for_backward(emb, pos, neg, lv_e, lv_p, lv_n, nz_e, nz_p, nz_n, logits)
        ctx.radius = radius
        ctx.mark_non_differentiable(correct, logits)
        return loss, correct, logits

    @staticmethod
    def backward(ctx, g_loss, g_correct, g_logits):
        emb, pos, neg, lv_e, lv_p, lv_n, nz_e, nz_p, nz_n, logits = ctx.saved_tensors
        B, K, D = pos.shape
        var, noisy = lv_e is not None, nz_e is not None
        mu = [emb, pos, neg]
        g = g_loss.to(device=emb.device, dtype=torch.float32).reshape(1).contiguous()
        g_mu = [torch.empty_like(t, memory_format=torch.contiguous_format) for t in mu]
        g_lv = [torch.empty_like(t, memory_format=torch.contiguous_format) for t in mu] if var else None
        _call("eu_gae_loss_backward", g, B, K, D, mu, [lv_e, lv_p, lv_n] if var else None,
              [nz_e, nz_p, nz_n] if noisy else None, ctx.radius, logits, g_mu, g_lv)
        return (None, *g_mu, *(g_lv or [None] * 3), None, None, None)


def gae_loss(emb, pos, neg, log_var=None, noise=None, radius=1.0, return_logits=False):
    """The reconstruction loss and accuracy of BaseGraphAutoEncoder.__call__ (mp_utils/base_gae.py) and, with log_var, of
    VariationalGraphAutoEncoder.__call__ (examples/gae/gae.py), in one fused device op over encoder rows:
        emb f32[B, D] (or [B, 1, D])   the source rows        pos, neg f32[B, K, D]   positive and negative context rows, K >= 1
        log_var                        None (GAE), or the three sets' log-variance rows (same shapes as emb, pos, neg)
        noise                          None (z = mu: VGAE's train=False), or three sets of unit-normal draws (same shapes);
                                       the op forms z = mu + radius * noise * sqrt(exp(log_var)) itself
    Returns (loss, correct) or, with return_logits, (loss, correct, logits f32[B, 2K]): loss is the mean sigmoid cross entropy
    over the 2BK logits <z_src, z_ctx> (positives first, labelled 1), plus the mean KL -0.5 (log_var - exp(log_var) - mu^2 + 1)
    over the B D (2K + 1) elements with log_var; correct (int64) counts floor(sigmoid(logit) + 0.5) == label, so the batch's
    acc is correct / (2BK).  Gradients reach emb, pos, neg and log_var, never noise.  Deterministic, no atomics, and neither
    pass synchronises with the host (include/euler_b200.h, eu_gae_loss)."""
    if radius is None or not math.isfinite(float(radius)):
        raise EulerError("gae_loss: radius must be finite, got %r" % (radius,))
    if noise is not None and log_var is None:
        raise EulerError("gae_loss: noise needs log_var")
    _check_f32("gae_loss", (('emb', emb), ('pos', pos), ('neg', neg)))
    if emb.dim() == 3 and emb.shape[1] == 1:
        emb = emb.reshape(emb.shape[0], emb.shape[2])
    if emb.dim() != 2 or pos.dim() != 3 or pos.shape[0] != emb.shape[0] or pos.shape[1] < 1 or pos.shape[2] != emb.shape[1] \
            or neg.shape != pos.shape:
        raise EulerError("gae_loss: need emb [B, D] and pos, neg [B, K >= 1, D]; got %s, %s and %s"
                         % (tuple(emb.shape), tuple(pos.shape), tuple(neg.shape)))
    sets = [emb, pos, neg]
    extra = []
    for name, group in (('log_var', log_var), ('noise', noise)):
        if group is None:
            extra.append([None] * 3)
            continue
        group = list(group)
        _check_f32("gae_loss", [(name, t) for t in group])
        group = [t.reshape(t.shape[0], t.shape[2]) if i == 0 and t.dim() == 3 and t.shape[1] == 1 else t
                 for i, t in enumerate(group)]
        if len(group) != 3 or any(t.shape != s.shape for t, s in zip(group, sets)):
            raise EulerError("gae_loss: %s must be three sets shaped as emb, pos and neg" % name)
        extra.append([_t(t, torch.float32) for t in group])
    sets = [_t(t, torch.float32) for t in sets]
    loss, correct, logits = _GaeLoss.apply(float(radius), *sets, *extra[0], *extra[1])
    return (loss, correct, logits) if return_logits else (loss, correct)


# ------------------------------------------------------------------------------------ streaming metrics
def _metric_tensors(op, named, dev):
    """raise unless every (name, tensor, dtype, shape) of named is a contiguous tensor of that dtype and shape on dev"""
    for nm, t, dtype, shape in named:
        if not torch.is_tensor(t) or t.dtype != dtype or tuple(t.shape) != shape or t.device != dev or not t.is_contiguous():
            raise EulerError("%s: %s must be a contiguous %s tensor of shape %s on %s" % (op, nm, dtype, shape, dev))


def _metric_batch(op, labels, predictions):
    """labels and predictions flattened: float32 tensors of one numel on one CUDA device"""
    _check_f32(op, (('labels', labels), ('predictions', predictions)))
    if labels.numel() != predictions.numel():
        raise EulerError("%s: labels (%d elements) and predictions (%d) must have one numel"
                         % (op, labels.numel(), predictions.numel()))
    if predictions.device.type != 'cuda' or labels.device != predictions.device:
        raise EulerError("%s: labels and predictions must be on one CUDA device" % op)
    return labels.detach().reshape(-1).contiguous(), predictions.detach().reshape(-1).contiguous()


def metric_auc_update(labels, predictions, tp, fn, tn, fp, refused, value):
    """One step of tf.metrics.auc(labels, predictions, num_thresholds=T) (TF 1.x metrics_impl.py, trapezoidal ROC) on the
    device: the batch's per-threshold counts are added to the state tp, fn, tn, fp (f32[T] each, 2 <= T <= 16384), and value
    (an f32 scalar) becomes the AUC of the new state.  labels and predictions are float32 with one numel; a label is positive
    when nonzero (NaN included) and predictions must lie in [0, 1].  A batch with a prediction outside [0, 1] or NaN is not
    counted (TF raises at that step): the state is untouched, refused (an int64 scalar) += 1, and value reads NaN while
    refused > 0.  No host synchronisation (include/euler_b200.h, eu_metric_auc_update); returns value."""
    op = "metric_auc_update"
    labels, predictions = _metric_batch(op, labels, predictions)
    T = tp.shape[0] if torch.is_tensor(tp) and tp.dim() == 1 else -1
    if not 2 <= T <= _lib.METRIC_AUC_MAX_THRESHOLDS:
        raise EulerError("%s: the state must be f32[T] with 2 <= T <= %d" % (op, _lib.METRIC_AUC_MAX_THRESHOLDS))
    dev = predictions.device
    _metric_tensors(op, [(nm, t, torch.float32, (T,)) for nm, t in (('tp', tp), ('fn', fn), ('tn', tn), ('fp', fp))]
                    + [('refused', refused, torch.int64, ()), ('value', value, torch.float32, ())], dev)
    _call("eu_metric_auc_update", labels, predictions, labels.numel(), T, tp, fn, tn, fp, refused, value)
    return value


_COUNT_KINDS = {'f1': (_lib.METRIC_F1, 3), 'acc': (_lib.METRIC_ACC, 2)}


def metric_count_update(kind, state, value, labels=None, predictions=None, correct=None, total=None):
    """One step of utils/metrics.py's f1_score (kind 'f1': state f32[3] = tp, fn, fp) or acc_score (kind 'acc': state
    f32[2] = total, count) with TF 1.x tf.metrics semantics, on the device: the batch's counts are added to state and value
    (an f32 scalar) becomes the metric of the new state.  The batch is either labels and predictions (float32, one numel;
    predictions are floor(p + 0.5) in float32) or, for 'acc' only, correct (an int64 device scalar, e.g. gae_loss's count)
    over total predictions (a host int).  No host synchronisation (include/euler_b200.h, eu_metric_count_update); returns
    value."""
    op = "metric_count_update"
    if kind not in _COUNT_KINDS:
        raise EulerError("%s: kind must be one of %s, got %r" % (op, sorted(_COUNT_KINDS), kind))
    code, width = _COUNT_KINDS[kind]
    if correct is None:
        if total is not None:
            raise EulerError("%s: total goes with correct" % op)
        labels, predictions = _metric_batch(op, labels, predictions)
        dev, n = predictions.device, labels.numel()
    else:
        if kind != 'acc' or labels is not None or predictions is not None:
            raise EulerError("%s: correct counts are taken for 'acc' only, without labels and predictions" % op)
        if not torch.is_tensor(correct) or correct.dtype != torch.int64 or correct.numel() != 1 or correct.device.type != 'cuda':
            raise EulerError("%s: correct must be an int64 CUDA scalar" % op)
        if total is None or int(total) < 0:
            raise EulerError("%s: total must be a count >= 0, got %r" % (op, total))
        dev, n, correct = correct.device, int(total), correct.detach().reshape(()).contiguous()
    _metric_tensors(op, [('state', state, torch.float32, (width,)), ('value', value, torch.float32, ())], dev)
    _call("eu_metric_count_update", code, labels, predictions, n, correct, state, value)
    return value


# ------------------------------------------------------------------------------------ optimizers
def _optim_args(op, var, slots, grad):
    """the library's (N, D, values, rows, R) for one update of var and its slots (same shape, float32, contiguous, on the
    graph's device): a dense grad of var's shape is taken as f32[N, D] over var's elements; a sparse COO grad of var's shape
    with one sparse dimension (coalesced here when it is not) as its rows i64[R] and values f32[R, D], D the elements of a row
    of var.  var and its slots may instead all be bfloat16 (the gradient stays float32).  Raises EulerError before any
    device work."""
    dev = _dev()
    dt = var.dtype if torch.is_tensor(var) and var.dtype == torch.bfloat16 else torch.float32
    for nm, t in (('var', var),) + slots:
        if not torch.is_tensor(t) or t.dtype != dt or t.device != dev or not t.is_contiguous() or t.is_sparse:
            raise EulerError("%s: %s must be a contiguous %s tensor on %s" % (op, nm, dt, dev))
        if t.shape != var.shape:
            raise EulerError("%s: %s has shape %s, var %s" % (op, nm, tuple(t.shape), tuple(var.shape)))
    if not torch.is_tensor(grad) or grad.dtype != torch.float32 or grad.device != dev or grad.shape != var.shape:
        raise EulerError("%s: grad must be a float32 tensor of var's shape %s on %s" % (op, tuple(var.shape), dev))
    grad = grad.detach()
    if not grad.is_sparse:
        n = var.numel()
        D = 4 if n % 4 == 0 else 1   # element-wise: a row width of 4 lets an aligned update take float4s
        return n // D, D, grad.contiguous(), None, _lib.OPTIM_DENSE
    if grad.layout != torch.sparse_coo or grad.sparse_dim() != 1 or var.dim() < 1:
        raise EulerError("%s: a sparse grad must be a COO tensor with one sparse dimension (rows of var)" % op)
    if not grad.is_coalesced():
        grad = grad.coalesce()
    N = var.shape[0]
    D = var.numel() // N if N else math.prod(var.shape[1:])
    rows = grad._indices()[0].contiguous()
    return N, D, grad._values().reshape(rows.numel(), D).contiguous(), rows, rows.numel()


def _sr_args(op, var, seed, step, tensor):
    """the trailing (dtype, seed, step, tensor) of an eu_optim_*_dtype call: step must be an int64 device scalar for bf16"""
    if var.dtype != torch.bfloat16:
        return 0, 0, None, 0
    _metric_tensors(op, [('step', step, torch.int64, ())], var.device)
    if not 0 <= int(seed) < 2 ** 64 or not 0 <= int(tensor) < 2 ** 31:
        raise EulerError("%s: seed must lie in [0, 2^64) and tensor in [0, 2^31), got %r and %r" % (op, seed, tensor))
    return 1, int(seed), step, int(tensor)


def optim_momentum_(var, accum, grad, lr, momentum, seed=0, step=None, tensor=0):
    """One step of TF 1.x MomentumOptimizer (non-Nesterov) on var in place, no autograd: accum = accum * momentum + g,
    var = var - lr * accum, each op one f32 rounding.  A dense grad updates every element (apply_momentum); a sparse COO grad
    (sparse_apply_momentum) only its rows, after coalesce() when it is not coalesced.  var, accum: contiguous float32 of one
    shape on the graph's device.  No host synchronisation for a dense or coalesced grad (include/euler_b200.h,
    eu_optim_momentum); shape, dtype and device mismatches raise EulerError and write nothing.  Returns var.
    var and accum may both be bfloat16 (grad stays float32): each value is widened exactly, updated in f32, and written back
    by stochastic rounding keyed by (seed, step, tensor, element), step an int64 device scalar the caller advances once per
    step (include/euler_b200.h, eu_optim_momentum_dtype)."""
    op = "optim_momentum_"
    N, D, g, rows, R = _optim_args(op, var, (('accum', accum),), grad)
    if var.dtype == torch.bfloat16:
        _call("eu_optim_momentum_dtype", var, accum, N, D, g, rows, R, float(lr), float(momentum), *_sr_args(op, var, seed, step, tensor))
    else:
        _call("eu_optim_momentum", var, accum, N, D, g, rows, R, float(lr), float(momentum))
    return var


def optim_adagrad_(var, accum, grad, lr, seed=0, step=None, tensor=0):
    """One step of TF 1.x AdagradOptimizer on var in place, no autograd: accum = accum + g * g, var = var - (lr * g) *
    (1 / sqrt(accum)), each op one f32 rounding.  Dense grads update every element (apply_adagrad), sparse COO grads their
    rows only (sparse_apply_adagrad), as optim_momentum_ (include/euler_b200.h, eu_optim_adagrad).  Returns var.  bfloat16
    var and accum as optim_momentum_."""
    op = "optim_adagrad_"
    N, D, g, rows, R = _optim_args(op, var, (('accum', accum),), grad)
    if var.dtype == torch.bfloat16:
        _call("eu_optim_adagrad_dtype", var, accum, N, D, g, rows, R, float(lr), *_sr_args(op, var, seed, step, tensor))
    else:
        _call("eu_optim_adagrad", var, accum, N, D, g, rows, R, float(lr))
    return var


def optim_adam_(var, m, v, grad, powers, lr, beta1, beta2, epsilon, seed=0, step=None, tensor=0):
    """One step of TF 1.x AdamOptimizer on var in place, no autograd, with alpha = (lr * sqrt(1 - powers[1])) /
    (1 - powers[0]) computed on the device from powers (float32[2]: beta1_power, beta2_power, on var's device).  A dense grad
    runs ApplyAdam: m = m + (g - m) * (1 - b1), v = v + (g * g - v) * (1 - b2), var = var - (m * alpha) / (sqrt(v) + eps).  A
    sparse COO grad (coalesced first when it is not) runs _apply_sparse_shared over EVERY row: m = m * b1 and v = v * b2, plus
    g * (1 - b1) and (g * g) * (1 - b2) on the grad's rows, then var = var - (alpha * m) / (sqrt(v) + eps).  Each op is one f32
    rounding.  The powers are not advanced here: the caller multiplies each by its beta once per step, after every variable
    (TF's _finish).  Checks and synchronisation as optim_momentum_ (include/euler_b200.h, eu_optim_adam).  Returns var.
    bfloat16 var, m and v as optim_momentum_; a sparse step rounds every row it writes."""
    op = "optim_adam_"
    N, D, g, rows, R = _optim_args(op, var, (('m', m), ('v', v)), grad)
    _metric_tensors(op, [('powers', powers, torch.float32, (2,))], var.device)
    hp = (float(lr), float(beta1), float(beta2), float(epsilon))
    if var.dtype == torch.bfloat16:
        _call("eu_optim_adam_dtype", var, m, v, N, D, g, rows, R, powers, *hp, *_sr_args(op, var, seed, step, tensor))
    else:
        _call("eu_optim_adam", var, m, v, N, D, g, rows, R, powers, *hp)
    return var


# ------------------------------------------------------------------------------------ knowledge-graph embedding step
KG_MODELS = {'transe': 0, 'transh': 1, 'transr': 2, 'transd': 3, 'distmult': 4}
KG_CORRUPT = {'front': 1, 'tail': 2, 'both': 3}
# the tables each model takes, in order, and the slot of eu_kg_problem.table each one fills
_KG_SLOTS = {0: (0, 1), 1: (0, 1, 3), 2: (0, 1, 3), 3: (0, 1, 2, 3), 4: (0, 1)}


def _kg_problem(model, l1, corrupt, margin, src, dst, rel, neg, slots, ent_dim, rel_dim):
    p = _lib.KgProblem()
    p.model, p.l1, p.corrupt, p.margin = model, int(bool(l1)), corrupt, float(margin)
    p.B, p.K = src.numel(), neg.shape[1]
    p.ent_dim, p.rel_dim = ent_dim, rel_dim
    p.n_ent, p.n_rel = slots[0].shape[0], slots[1].shape[0]
    p.src, p.dst, p.rel, p.neg = src.data_ptr(), dst.data_ptr(), rel.data_ptr(), neg.data_ptr()
    for t, tb in enumerate(slots):
        if tb is not None:
            p.table[t] = tb.data_ptr()
    return p


def _raw_kg(ent, relt, eaux, raux, src, dst, rel, neg, cfg):
    """one eu_kg_loss (eu_kg_loss_dtype for bf16 tables): (scores f32[B, 1 + C K], rank i32[B], loss f32[],
    [src_emb, rel_emb, dst_emb] or None)"""
    model, l1, corrupt, margin, ent_dim, rel_dim, sparse_grad, with_emb = cfg
    B, K = neg.shape
    dev = ent.device
    scores = torch.empty((B, 1 + (2 if corrupt == 3 else 1) * K), dtype=torch.float32, device=dev)
    rank = torch.empty(B, dtype=torch.int32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    embs = [torch.empty((B, rel_dim), dtype=torch.float32, device=dev) for _ in range(3)] if with_emb else None
    p = _kg_problem(model, l1, corrupt, margin, src, dst, rel, neg, (ent, relt, eaux, raux), ent_dim, rel_dim)
    if ent.dtype == torch.bfloat16:
        _call("eu_kg_loss_dtype", C.byref(p), _lib.TORCH_DTYPES[ent.dtype], scores, rank, loss, *(embs or [None] * 3))
    else:
        _call("eu_kg_loss", C.byref(p), scores, rank, loss, *(embs or [None] * 3))
    return scores, rank, loss, embs


def _raw_kg_sparse_grads(slots, src, dst, rel, neg, cfg, scores, g):
    """one eu_kg_loss_backward_sparse(_dtype) over the four table slots: per slot (rows i64[cap], values f32[cap, width]) or
    (None, None), _coo_buffers' arrays, and the counts of their rows filled"""
    model, l1, corrupt, margin, ent_dim, rel_dim, _, _ = cfg
    B, K = neg.shape
    p = _kg_problem(model, l1, corrupt, margin, src, dst, rel, neg, slots, ent_dim, rel_dim)
    entries = (B * (K + 2), B, B * (K + 2), B)
    bufs = [_coo_buffers(e, _shape(t), slots[0].device) for e, t in zip(entries, slots)]
    counts = (C.c_int64 * 4)()
    outs = ([r for r, _ in bufs], [v for _, v in bufs], counts)
    if slots[0].dtype == torch.bfloat16:
        _call("eu_kg_loss_backward_sparse_dtype", C.byref(p), _lib.TORCH_DTYPES[slots[0].dtype], g, scores, *outs)
    else:
        _call("eu_kg_loss_backward_sparse", C.byref(p), g, scores, *outs)
    return bufs, list(counts)


class _KgLoss(torch.autograd.Function):
    """eu_kg_loss / eu_kg_loss_backward(_sparse).  Saves the ids and the scores (and the tables, which are inputs): no
    [B, K, dim] rows are kept.  The four table slots are entity, relation, entity-side and relation-side auxiliary (None when
    the model has none)."""

    @staticmethod
    def forward(ctx, ent, relt, eaux, raux, src, dst, rel, neg, cfg):
        scores, rank, loss, embs = _raw_kg(ent, relt, eaux, raux, src, dst, rel, neg, cfg)
        ctx.save_for_backward(ent, relt, eaux, raux, src, dst, rel, neg, scores)
        ctx.cfg = cfg
        ctx.mark_non_differentiable(rank, *(embs or []))
        if embs:
            return (loss, rank) + tuple(embs)
        return loss, rank

    @staticmethod
    def backward(ctx, g_loss, *unused):
        ent, relt, eaux, raux, src, dst, rel, neg, scores = ctx.saved_tensors
        model, l1, corrupt, margin, ent_dim, rel_dim, sparse_grad, _ = ctx.cfg
        slots = (ent, relt, eaux, raux)
        dev = ent.device
        g = g_loss.to(device=dev, dtype=torch.float32).reshape(1).contiguous()
        if not sparse_grad:
            p = _kg_problem(model, l1, corrupt, margin, src, dst, rel, neg, slots, ent_dim, rel_dim)
            grads = [None if t is None else torch.empty_like(t) for t in slots]
            _call("eu_kg_loss_backward", C.byref(p), g, scores, grads)
            return tuple(grads) + (None,) * 5
        bufs, counts = _raw_kg_sparse_grads(slots, src, dst, rel, neg, ctx.cfg, scores, g)
        return tuple(_coo(r, v, counts[t], _shape(slots[t])) for t, (r, v) in enumerate(bufs)) + (None,) * 5


def _kg_args(op, src, dst, neg, rel, tables, model, corrupt, metric):
    """(model index, the four table slots, src, dst, rel [B], neg [B, K]) on the device, or EulerError: the checks of
    kg_margin_loss"""
    name = str(model).lower()
    if name not in KG_MODELS:
        raise EulerError("%s: model must be one of %s, got %r" % (op, sorted(KG_MODELS), model))
    if corrupt not in KG_CORRUPT:
        raise EulerError("%s: corrupt must be one of %s, got %r" % (op, sorted(KG_CORRUPT), corrupt))
    if metric not in SKIPGRAM_METRICS:
        raise EulerError("%s: metric must be one of %s, got %r" % (op, SKIPGRAM_METRICS, metric))
    m = KG_MODELS[name]
    want = _KG_SLOTS[m]
    tables = list(tables)
    if len(tables) != len(want):
        raise EulerError("%s: %s takes %d tables, got %d" % (op, name, len(want), len(tables)))
    _table_dtype(op, [("table %d" % k, tb) for k, tb in enumerate(tables)])
    slots = [None] * 4
    for t, tb in zip(want, tables):
        slots[t] = _t(tb, tb.dtype)
    ent_dim, rel_dim = slots[0].shape[1], slots[1].shape[1]
    aux_w = {1: ent_dim, 2: ent_dim * rel_dim, 3: rel_dim}.get(m)
    if (slots[2] is not None and tuple(slots[2].shape) != tuple(slots[0].shape)) or \
       (slots[3] is not None and (slots[3].shape[0] != slots[1].shape[0] or slots[3].shape[1] != aux_w)):
        raise EulerError("%s: the auxiliary tables of %s must match the entity / relation tables" % (op, name))
    src = _t(src, torch.int64).reshape(-1)
    dst = _t(dst, torch.int64).reshape(-1)
    rel = _t(rel, torch.int64).reshape(-1)
    neg = _t(neg, torch.int64)
    B = src.numel()
    if dst.numel() != B or rel.numel() != B or neg.dim() != 2 or neg.shape[0] != B:
        raise EulerError("%s: src, dst, rel must have B = %d ids and neg be [B, K], got %s, %s, %s"
                         % (op, B, dst.numel(), rel.numel(), tuple(neg.shape)))
    return m, slots, src, dst, rel, neg


def kg_margin_loss(src, dst, neg, rel, tables, model, l1=True, corrupt='both', margin=1.0, metric='mrr', sparse_grad=False,
                   with_embeddings=False):
    """The step after the ids of Euler's knowledge-graph models (examples/TransX TransX.call, examples/distmult) in one fused
    device op:
        src, dst [B] or [B, 1]   entity ids of the true triples      rel [B] or [B, 1]   their relation ids (int64)
        neg [B, K]               entity ids of the corruptions (K >= 1)
        tables                   f32 or bf16 tables by model: 'transe' / 'distmult' (entity, relation); 'transh' (entity,
                                 relation, hyper); 'transr' (entity, relation, transfer_matrix [n_rel, ent_dim * rel_dim]);
                                 'transd' (entity, relation, entity_transfer, relation_transfer)
    Scores each triple and its corruptions ('front': (neg_k, r, d), 'tail': (s, r, neg_k), 'both': front then tail) on the
    mapped rows (include/euler_b200.h, eu_kg_loss), and returns (loss, metric): loss = mean_b max(margin + mean_k neg - pos, 0),
    metric the ranking metric `metric` (skipgram_metric: mrr, hit1, hit3, hit10, mr) of the true triple among its corruptions,
    ties ranked as TF's stable top_k ranks them.  with_embeddings=True appends the mapped (src, rel, dst) rows f32[B, rel_dim]
    (not differentiated).  The gradient reaches the tables only: dense, or with sparse_grad=True coalesced sparse COO gradients
    of the rows the batch touches.  Deterministic, no atomics; the forward and the backward synchronise once each.
    bfloat16 tables (all of one dtype) are read widened exactly to f32, so the loss, metric and embeddings are the f32 op's
    on the widened tables.  They take no gradient through autograd, which would round their f32 gradient to nearest bf16: a
    bf16 table that requires grad raises.  Train them with kg_margin_loss_sparse_grads and an optimizer's apply_sparse
    (knowledge's train_step)."""
    m, slots, src, dst, rel, neg = _kg_args("kg_margin_loss", src, dst, neg, rel, tables, model, corrupt, metric)
    if slots[0].dtype == torch.bfloat16 and any(t is not None and t.requires_grad for t in slots):
        raise EulerError("kg_margin_loss: a bfloat16 table takes no autograd gradient (torch would round it to bf16); "
                         "train it with kg_margin_loss_sparse_grads and an optimizer's apply_sparse")
    cfg = (m, bool(l1), KG_CORRUPT[corrupt], float(margin), slots[0].shape[1], slots[1].shape[1], bool(sparse_grad),
           bool(with_embeddings))
    out = _KgLoss.apply(slots[0], slots[1], slots[2], slots[3], src, dst, rel, neg, cfg)
    res = (out[0], skipgram_metric(out[1], metric))
    return res + tuple(out[2:]) if with_embeddings else res


def kg_margin_loss_sparse_grads(src, dst, neg, rel, tables, model, l1=True, corrupt='both', margin=1.0, metric='mrr',
                                with_embeddings=False):
    """kg_margin_loss's forward and its sparse backward for an upstream gradient of 1, without autograd, for tables of
    float32 or bfloat16 (all of one dtype, read widened exactly to f32).  Returns (loss, metric, grads), plus the mapped
    (src, rel, dst) rows f32[B, rel_dim] with with_embeddings=True: grads is one (rows i64[D], values f32[D, width]) per
    table, in the order the model takes its tables -- the coalesced f32 gradient that kg_margin_loss(..., sparse_grad=True)
    .backward() gives f32 tables holding the widened values.  They go to an optimizer's apply_sparse as they are, never
    rounded to bf16.  Synchronises twice (the forward, the backward)."""
    m, slots, src, dst, rel, neg = _kg_args("kg_margin_loss_sparse_grads", src, dst, neg, rel, tables, model, corrupt, metric)
    slots = [None if t is None else t.detach() for t in slots]
    cfg = (m, bool(l1), KG_CORRUPT[corrupt], float(margin), slots[0].shape[1], slots[1].shape[1], True, bool(with_embeddings))
    scores, rank, loss, embs = _raw_kg(*slots, src, dst, rel, neg, cfg)
    g = torch.ones(1, dtype=torch.float32, device=slots[0].device)
    bufs, counts = _raw_kg_sparse_grads(slots, src, dst, rel, neg, cfg, scores, g)
    grads = [(bufs[t][0][:counts[t]], bufs[t][1][:counts[t]]) for t in _KG_SLOTS[m]]
    res = (loss, skipgram_metric(rank, metric), grads)
    return res + (embs,) if with_embeddings else res
