"""tf_euler's Python op API for the minibatch-construction path, over torch CUDA tensors.

Same names, argument meaning and error behaviour as the reference wrappers
(tf_euler/python/euler_ops/{base,neighbor_ops,walk_ops,sample_ops,feature_ops,mp_ops,type_ops}.py);
each function cites the wrapper it mirrors.  Tensors are torch tensors on the graph's device; every
op enqueues kernels from libeuler_b200.so on the current torch stream.  Nothing here computes on the
CPU and nothing falls back to PyTorch ops: if the library or the GPU is missing, calls raise.
"""
import ctypes as C
import threading

import numpy as np
import torch

from . import _lib
from ._lib import EulerError, check
from .graph import Context, Graph

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


def _t(x, dtype):
    if isinstance(x, torch.Tensor):
        return x.to(device=_dev(), dtype=dtype).contiguous()
    return torch.as_tensor(np.asarray(x), dtype=dtype, device=_dev()).contiguous()


def _i32_host(x):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x).reshape(-1), dtype=np.int32)


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


# ------------------------------------------------------------------------------------ sampling
def sample_neighbor(nodes, edge_types, count, default_node=-1, condition=''):
    """neighbor_ops.sample_neighbor (neighbor_ops.py:39-41).  Returns (neighbors i64[B,count],
    weights f32[B,count], types i32[B,count])."""
    if condition:
        raise EulerError("sample_neighbor: `condition` (index queries) is outside this path")
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    B = nodes.numel()
    ids = torch.empty((B, count), dtype=torch.int64, device=nodes.device)
    w = torch.empty((B, count), dtype=torch.float32, device=nodes.device)
    t = torch.empty((B, count), dtype=torch.int32, device=nodes.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_neighbor(ctx._h, nodes.data_ptr(), B, et.ctypes.data, len(et), count,
                                         default_node, ids.data_ptr(), w.data_ptr(), t.data_ptr()))
    return ids, w, t


def sample_fanout(nodes, edge_types, counts, default_node=-1):
    """neighbor_ops.sample_fanout (neighbor_ops.py:122-158).  edge_types: list (per hop) of 1-D
    type lists of equal length.  Returns (neighbors_list[L+1], weights_list[L], types_list[L]),
    all flattened like the reference."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    L = len(counts)
    ets = [get_edge_type_id(e) for e in edge_types]
    if len(ets) != L or any(len(e) != len(ets[0]) for e in ets):
        raise EulerError("sample_fanout: edge_types must hold one equal-length type list per hop")
    et = np.ascontiguousarray(np.stack(ets) if L else np.zeros((0, 0)), dtype=np.int32)
    cs = np.ascontiguousarray(counts, dtype=np.int32)
    B = nodes.numel()
    ids, ws, ts, rows = [], [], [], B
    for c in counts:
        rows *= int(c)
        ids.append(torch.empty(rows, dtype=torch.int64, device=nodes.device))
        ws.append(torch.empty(rows, dtype=torch.float32, device=nodes.device))
        ts.append(torch.empty(rows, dtype=torch.int32, device=nodes.device))
    P = C.c_void_p * max(L, 1)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_fanout(ctx._h, nodes.data_ptr(), B, et.ctypes.data,
                                       et.shape[1] if L else 0, cs.ctypes.data, L, default_node,
                                       P(*[x.data_ptr() for x in ids]), P(*[x.data_ptr() for x in ws]),
                                       P(*[x.data_ptr() for x in ts])))
    return [nodes] + ids, ws, ts


def sample_fanout_with_feature(nodes, edge_types, count, default_node, dense_feature_names, dense_dimensions,
                               sparse_feature_names, sparse_default_values):
    """neighbor_ops.sample_fanout_with_feature (neighbor_ops.py:49-69; kernel sample_fanout_with_feature_op.cc).  The hops are
    sample_fanout's (the same draws on the same context state); the features of hop i are those of its engine ids, as the
    reference's v_select(nb_i) takes them (a row whose first draw is node 0 is packed as default_node but keeps the features of
    its draws).  Returns, as the reference's wrapper does:
        neighbors        [nodes] + L flattened hops
        weights, types   L tensors shaped [B, c1, ..., ci]
        dense_features   (L+1) * len(dense_feature_names) tensors f32[rows_i, dim], hop-major
        sparse_features  (L+1) * len(sparse_feature_names) (indices, values, dense_shape) triples, hop-major, as get_sparse_feature
    One host synchronisation per call when sparse features are asked for (all ragged totals together), none otherwise."""
    g, lib = get_graph(), _lib.load()
    nodes = _t(nodes, torch.int64).reshape(-1)
    L = len(count)
    ets = [get_edge_type_id(e) for e in edge_types]
    if len(ets) != L or any(len(e) != len(ets[0]) for e in ets):
        raise EulerError("sample_fanout_with_feature: edge_types must hold one equal-length type list per hop")
    if len(dense_feature_names) != len(dense_dimensions) or len(sparse_feature_names) != len(sparse_default_values):
        raise EulerError("sample_fanout_with_feature: one dimension per dense feature and one default per sparse feature")
    et = np.ascontiguousarray(np.stack(ets) if L else np.zeros((0, 0)), dtype=np.int32)
    cs = np.ascontiguousarray(count, dtype=np.int32)
    B, dev = nodes.numel(), nodes.device
    shapes, rows = [], [B]
    for c in count:
        shapes.append((shapes[-1] if shapes else (B,)) + (int(c),))
        rows.append(rows[-1] * int(c))
    ids = [torch.empty(r, dtype=torch.int64, device=dev) for r in rows[1:]]
    eng = [torch.empty(r, dtype=torch.int64, device=dev) for r in rows[1:]]
    ws = [torch.empty(sh, dtype=torch.float32, device=dev) for sh in shapes]
    ts = [torch.empty(sh, dtype=torch.int32, device=dev) for sh in shapes]
    dfid = np.asarray([n if isinstance(n, (int, np.integer)) else g.dense_feature_id(str(n)) for n in dense_feature_names], np.int32)
    ddim = np.asarray(dense_dimensions, np.int32)
    sfid = np.asarray([g.sparse_feature_id(str(n)) for n in sparse_feature_names], np.int32)
    nd, ns = len(dfid), len(sfid)
    dense = [torch.empty((rows[l], int(ddim[j])), dtype=torch.float32, device=dev) for l in range(L + 1) for j in range(nd)]
    ptrs = [torch.empty(rows[l] + 1, dtype=torch.int64, device=dev) for l in range(L + 1) for j in range(ns)]
    total, maxlen = np.zeros(max(len(ptrs), 1), np.int64), np.zeros(max(len(ptrs), 1), np.int64)

    def P(ts_):
        return (C.c_void_p * max(len(ts_), 1))(*[t.data_ptr() for t in ts_])
    ctx = _ctx_on_stream()
    check(lib.eu_sample_fanout_with_feature(ctx._h, nodes.data_ptr(), B, et.ctypes.data, et.shape[1] if L else 0, cs.ctypes.data, L,
                                            default_node, P(ids), P(ws), P(ts), P(eng), nd, dfid.ctypes.data, ddim.ctypes.data,
                                            P(dense), ns, sfid.ctypes.data, P(ptrs), total.ctypes.data, maxlen.ctypes.data))
    sparse = []
    for l in range(L + 1):
        hop_ids = nodes if l == 0 else eng[l - 1]
        for j in range(ns):
            k = l * ns + j
            ptr, tot, dv = ptrs[k], int(total[k]), int(sparse_default_values[j])
            vals = torch.empty(tot, dtype=torch.int64, device=dev)
            if tot:
                check(lib.eu_get_sparse_feature(ctx._h, hop_ids.data_ptr(), rows[l], int(sfid[j]), dv, tot, ptr.data_ptr(),
                                                vals.data_ptr()))
            lens = ptr[1:] - ptr[:-1]
            r = torch.repeat_interleave(torch.arange(rows[l], device=dev), lens, output_size=tot)
            cols = torch.arange(tot, device=dev) - ptr[:-1][r]
            sparse.append((torch.stack([r, cols], dim=1), vals, (rows[l], int(maxlen[k]))))
    return [nodes] + ids, ws, ts, dense, sparse


def sample_fanout_batched(nodes, edge_types, counts, default_node=-1, ctx=None):
    """nb independent sample_fanout calls in one set of kernel launches.  nodes: [nb, B]; batch b runs on engine b
    of `ctx` (Context.set_engines), i.e. it returns exactly what sample_fanout(nodes[b]) returns on a context
    seeded like engine b.  Returns (neighbors_list[L+1], weights_list[L], types_list[L]) with a leading nb dim."""
    nodes = _t(nodes, torch.int64)
    nb, B = nodes.shape
    L = len(counts)
    ets = [get_edge_type_id(e) for e in edge_types]
    et = np.ascontiguousarray(np.stack(ets) if L else np.zeros((0, 0)), dtype=np.int32)
    cs = np.ascontiguousarray(counts, dtype=np.int32)
    ids, ws, ts, rows = [], [], [], B
    for c in counts:
        rows *= int(c)
        ids.append(torch.empty((nb, rows), dtype=torch.int64, device=nodes.device))
        ws.append(torch.empty((nb, rows), dtype=torch.float32, device=nodes.device))
        ts.append(torch.empty((nb, rows), dtype=torch.int32, device=nodes.device))
    P = C.c_void_p * max(L, 1)
    ctx = ctx or _ctx_on_stream()
    check(_lib.load().eu_sample_fanout_batched(ctx._h, nodes.data_ptr(), nb, B, et.ctypes.data,
                                               et.shape[1] if L else 0, cs.ctypes.data, L, default_node,
                                               P(*[x.data_ptr() for x in ids]), P(*[x.data_ptr() for x in ws]),
                                               P(*[x.data_ptr() for x in ts])))
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
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_node(ctx._h, count, types.ctypes.data, len(types), out.data_ptr()))
    return out


def random_walk(nodes, edge_types, p=1.0, q=1.0, default_node=-1):
    """walk_ops.random_walk (walk_ops.py:29-43).  edge_types: list of L 1-D type lists.
    Returns i64[B, L+1]."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    ets = [get_edge_type_id(e) for e in edge_types]
    L = len(ets)
    if any(len(e) != len(ets[0]) for e in ets):
        raise EulerError("random_walk: every step needs the same number of edge types here")
    et = np.ascontiguousarray(np.stack(ets) if L else np.zeros((0, 0)), dtype=np.int32)
    B = nodes.numel()
    out = torch.empty((B, L + 1), dtype=torch.int64, device=nodes.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_random_walk(ctx._h, nodes.data_ptr(), B, et.ctypes.data,
                                     et.shape[1] if L else 0, L, float(p), float(q), default_node,
                                     out.data_ptr()))
    return out


def get_dense_feature(nodes, feature_names, dimensions, thread_num=1):
    """feature_ops.get_dense_feature (feature_ops.py:111-125): list of f32[M, dim_i]; names are
    looked up as "dense_"+name in the graph meta (get_dense_feature_op.cc:83); ints are slot ids."""
    del thread_num  # the reference splits the batch over TF threads; one launch here
    nodes = _t(nodes, torch.int64).reshape(-1)
    g = get_graph()
    outs = []
    ctx = _ctx_on_stream()
    for name, dim in zip(feature_names, dimensions):
        fid = name if isinstance(name, (int, np.integer)) else g.dense_feature_id(name)
        out = torch.empty((nodes.numel(), int(dim)), dtype=torch.float32, device=nodes.device)
        check(_lib.load().eu_get_dense_feature(ctx._h, nodes.data_ptr(), nodes.numel(), int(fid),
                                               int(dim), out.data_ptr()))
        outs.append(out)
    return outs


def _ragged(fn, nodes, fid, *mid):
    """two-phase ragged fetch: lengths, then values"""
    nodes = _t(nodes, torch.int64).reshape(-1)
    n = nodes.numel()
    ctx = _ctx_on_stream()
    indptr = torch.empty(n + 1, dtype=torch.int64, device=nodes.device)
    check(fn(ctx._h, nodes.data_ptr(), n, int(fid), *mid, 0, indptr.data_ptr(), None))
    total = int(indptr[-1].item())
    return nodes, n, ctx, indptr, total


def get_sparse_feature(nodes, feature_names, default_values=None, thread_num=1):
    """feature_ops.get_sparse_feature (feature_ops.py:57-73; kernel get_sparse_feature_op.cc:52-130).  Per feature the
    reference returns a SparseTensor; here the same content as (indices i64[nnz, 2], values i64[nnz], dense_shape (N, max_len)):
    row i lists the uint64 values of the node, a node without values gets the single entry (i, 0) = default value."""
    g, lib = get_graph(), _lib.load()
    names = [str(x) for x in feature_names]
    defaults = [0] * len(names) if default_values is None else [int(x) for x in default_values]
    outs = []
    for name, dv in zip(names, defaults):
        fid = g.sparse_feature_id(name)
        nd, n, ctx, indptr, total = _ragged(lib.eu_get_sparse_feature, nodes, fid, dv)
        vals = torch.empty(total, dtype=torch.int64, device=nd.device)
        if total:
            check(lib.eu_get_sparse_feature(ctx._h, nd.data_ptr(), n, int(fid), dv, total, indptr.data_ptr(), vals.data_ptr()))
        lens = indptr[1:] - indptr[:-1]
        rows = torch.repeat_interleave(torch.arange(n, device=nd.device), lens)
        cols = torch.arange(total, device=nd.device) - indptr[:-1][rows]
        outs.append((torch.stack([rows, cols], dim=1), vals, (n, int(lens.max().item()) if n else 0)))
    return outs


def get_binary_feature(nodes, feature_names, thread_num=1):
    """feature_ops.get_binary_feature (feature_ops.py:158-171): per feature a list of N byte strings (b'' for absent nodes)."""
    g, lib = get_graph(), _lib.load()
    outs = []
    for name in [str(x) for x in feature_names]:
        fid = g.binary_feature_id(name)
        nd, n, ctx, indptr, total = _ragged(lib.eu_get_binary_feature, nodes, fid)
        buf = torch.empty(max(total, 1), dtype=torch.uint8, device=nd.device)
        if total:
            check(lib.eu_get_binary_feature(ctx._h, nd.data_ptr(), n, int(fid), total, indptr.data_ptr(), buf.data_ptr()))
        raw, ptr = bytes(buf[:total].cpu().numpy().tobytes()), indptr.cpu().tolist()
        outs.append([raw[ptr[i]:ptr[i + 1]] for i in range(n)])
    return outs


def sample_edge(count, edge_type):
    """sample_ops.sample_edge (tf_euler/python/euler_ops/sample_ops.py; kernel sample_edge_op.cc): i64[count, 3] rows of
    (src, dst, type), drawn by edge weight among the edges of ONE type (several types return nothing in the reference)."""
    types = get_edge_type_id(edge_type)
    count = int(count)
    out = torch.empty((count, 3), dtype=torch.int64, device=_dev())
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_edge(ctx._h, count, types.ctypes.data, len(types), out.data_ptr()))
    return out


def _edges(edges):
    e = _t(edges, torch.int64)
    if e.dim() != 2 or e.shape[1] != 3:
        raise EulerError("edges must be a matrix with shape [n, 3]")
    return e.contiguous()


def get_edge_dense_feature(edges, feature_names, dimensions, thread_num=1):
    """feature_ops.get_edge_dense_feature: list of f32[E, dim] (zeros for unknown edges / features)"""
    e = _edges(edges)
    g, lib, outs = get_graph(), _lib.load(), []
    ctx = _ctx_on_stream()
    for name, dim in zip(feature_names, dimensions):
        out = torch.empty((e.shape[0], int(dim)), dtype=torch.float32, device=e.device)
        check(lib.eu_get_edge_dense_feature(ctx._h, e.data_ptr(), e.shape[0], g.edge_feature_id("dense", name), int(dim), out.data_ptr()))
        outs.append(out)
    return outs


def get_edge_sparse_feature(edges, feature_names, default_values=None, thread_num=1):
    """feature_ops.get_edge_sparse_feature: per feature (indices i64[nnz, 2], values i64[nnz], dense_shape)"""
    e = _edges(edges)
    g, lib, outs = get_graph(), _lib.load(), []
    names = [str(x) for x in feature_names]
    defaults = [0] * len(names) if default_values is None else [int(x) for x in default_values]
    ctx = _ctx_on_stream()
    n = e.shape[0]
    for name, dv in zip(names, defaults):
        fid = g.edge_feature_id("sparse", name)
        indptr = torch.empty(n + 1, dtype=torch.int64, device=e.device)
        check(lib.eu_get_edge_sparse_feature(ctx._h, e.data_ptr(), n, fid, dv, 0, indptr.data_ptr(), None))
        total = int(indptr[-1].item())
        vals = torch.empty(total, dtype=torch.int64, device=e.device)
        if total:
            check(lib.eu_get_edge_sparse_feature(ctx._h, e.data_ptr(), n, fid, dv, total, indptr.data_ptr(), vals.data_ptr()))
        lens = indptr[1:] - indptr[:-1]
        rows = torch.repeat_interleave(torch.arange(n, device=e.device), lens)
        cols = torch.arange(total, device=e.device) - indptr[:-1][rows]
        outs.append((torch.stack([rows, cols], dim=1), vals, (n, int(lens.max().item()) if n else 0)))
    return outs


def get_edge_binary_feature(edges, feature_names, thread_num=1):
    """feature_ops.get_edge_binary_feature: per feature a list of E byte strings"""
    e = _edges(edges)
    g, lib, outs = get_graph(), _lib.load(), []
    ctx = _ctx_on_stream()
    n = e.shape[0]
    for name in [str(x) for x in feature_names]:
        fid = g.edge_feature_id("binary", name)
        indptr = torch.empty(n + 1, dtype=torch.int64, device=e.device)
        check(lib.eu_get_edge_binary_feature(ctx._h, e.data_ptr(), n, fid, 0, indptr.data_ptr(), None))
        total = int(indptr[-1].item())
        buf = torch.empty(max(total, 1), dtype=torch.uint8, device=e.device)
        if total:
            check(lib.eu_get_edge_binary_feature(ctx._h, e.data_ptr(), n, fid, total, indptr.data_ptr(), buf.data_ptr()))
        raw, ptr = bytes(buf[:total].cpu().numpy().tobytes()), indptr.cpu().tolist()
        outs.append([raw[ptr[i]:ptr[i + 1]] for i in range(n)])
    return outs


def get_full_neighbor(nodes, edge_types):
    """neighbor_ops.get_full_neighbor (tf_euler/python/euler_ops/neighbor_ops.py; kernel get_full_neighbor_op.cc over
    euler::GetFullNeighbor api.cc:208-221).  The reference returns three SparseTensors [N, max_degree] (ids, weights,
    types) whose values are listed node by node; here the same values come back ragged: (indptr i64[N+1], ids i64[nnz],
    weights f32[nnz], types i32[nnz]) -- SparseTensor indices are (i, k - indptr[i]) for k in [indptr[i], indptr[i+1])."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = np.ascontiguousarray(edge_types, dtype=np.int32).reshape(-1)
    ctx = _ctx_on_stream()
    lib = _lib.load()
    n = nodes.numel()
    indptr = torch.empty(n + 1, dtype=torch.int64, device=nodes.device)
    check(lib.eu_get_full_neighbor(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), 0, indptr.data_ptr(), None, None, None))
    total = int(indptr[-1].item())
    ids = torch.empty(total, dtype=torch.int64, device=nodes.device)
    w = torch.empty(total, dtype=torch.float32, device=nodes.device)
    t = torch.empty(total, dtype=torch.int32, device=nodes.device)
    if total:
        check(lib.eu_get_full_neighbor(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), total, indptr.data_ptr(),
                                       ids.data_ptr(), w.data_ptr(), t.data_ptr()))
    return indptr, ids, w, t


def get_sorted_full_neighbor(nodes, edge_types, condition=''):
    """neighbor_ops.get_sorted_full_neighbor (neighbor_ops.py:100-119): get_full_neighbor with every node's entries ordered by
    neighbor id; same ragged return."""
    if condition:
        raise EulerError("get_sorted_full_neighbor: `condition` (index queries) is outside this path")
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    ctx = _ctx_on_stream()
    lib = _lib.load()
    n = nodes.numel()
    indptr = torch.empty(n + 1, dtype=torch.int64, device=nodes.device)
    check(lib.eu_get_sorted_full_neighbor(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), 0, indptr.data_ptr(), None, None, None))
    total = int(indptr[-1].item())
    ids = torch.empty(total, dtype=torch.int64, device=nodes.device)
    w = torch.empty(total, dtype=torch.float32, device=nodes.device)
    t = torch.empty(total, dtype=torch.int32, device=nodes.device)
    if total:
        check(lib.eu_get_sorted_full_neighbor(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), total, indptr.data_ptr(),
                                              ids.data_ptr(), w.data_ptr(), t.data_ptr()))
    return indptr, ids, w, t


def get_top_k_neighbor(nodes, edge_types, k, default_node=-1, condition=''):
    """neighbor_ops.get_top_k_neighbor (neighbor_ops.py:44-46): (ids i64[N,k], weights f32[N,k], types i32[N,k]), the k
    heaviest edges of each node, heaviest first, filled with default_node / 0 / -1."""
    if condition:
        raise EulerError("get_top_k_neighbor: `condition` (index queries) is outside this path")
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    n, k = nodes.numel(), int(k)
    ids = torch.empty((n, k), dtype=torch.int64, device=nodes.device)
    w = torch.empty((n, k), dtype=torch.float32, device=nodes.device)
    t = torch.empty((n, k), dtype=torch.int32, device=nodes.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_get_top_k_neighbor(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), k, default_node,
                                            ids.data_ptr(), w.data_ptr(), t.data_ptr()))
    return ids, w, t


_HOP_APPEND_FRONTIER, _HOP_SELF_LOOPS, _HOP_SORT = 1, 2, 4     # include/euler_b200.h


def _full_hop(nodes, edge_types, flags, rows=True, weights=False, types=False):
    """one eu_full_neighbor_hop: two host syncs, the listing total (output shapes) and the unique count (the frontier's length)"""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    ctx = _ctx_on_stream()
    lib = _lib.load()
    n, dev = nodes.numel(), nodes.device
    indptr = torch.empty(n + 1, dtype=torch.int64, device=dev)
    check(lib.eu_full_neighbor_hop(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), flags, 0, indptr.data_ptr(),
                                   None, None, None, None, None, None, None))
    total = int(indptr[-1].item())
    append = bool(flags & _HOP_APPEND_FRONTIER)
    width = total + (n if flags & _HOP_SELF_LOOPS else 0)
    uniq = torch.empty(total + (n if append else 0), dtype=torch.int64, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    edge_index = torch.empty((2 if rows else 1, width), dtype=torch.int64, device=dev)
    w = torch.empty(total, dtype=torch.float32, device=dev) if weights else None
    t = torch.empty(total, dtype=torch.int32, device=dev) if types else None
    res = torch.empty(n, dtype=torch.int64, device=dev) if append else None
    ptr = lambda x: None if x is None else x.data_ptr()          # noqa: E731
    check(lib.eu_full_neighbor_hop(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), flags, total, indptr.data_ptr(),
                                   uniq.data_ptr(), cnt.data_ptr(), edge_index[0].data_ptr() if rows else None,
                                   edge_index[-1].data_ptr(), ptr(w), ptr(t), ptr(res)))
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
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_neighbor_layerwise(ctx._h, nd.data_ptr(), batch, n, et.ctypes.data, len(et), int(count), default_node,
                                                   1 if weight_func == 'sqrt' else 0, out.data_ptr(), adj.data_ptr()))
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
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sparse_get_adj(ctx._h, nd.data_ptr(), nb.data_ptr(), batch, N, M, et.ctypes.data, len(et), adj.data_ptr()))
    return adj


def _adj_coo(nd, nb, batch, N, M, et):
    """one eu_sparse_get_adj_coo: a host sync for the entry count (the output shape)"""
    lib, dev = _lib.load(), nd.device
    rowptr = torch.empty(batch * N + 1, dtype=torch.int64, device=dev)
    ctx = _ctx_on_stream()
    args = (ctx._h, nd.data_ptr(), nb.data_ptr(), batch, N, M, et.ctypes.data, len(et))
    check(lib.eu_sparse_get_adj_coo(*args, 0, rowptr.data_ptr(), None, None))
    nnz = int(rowptr[-1].item())
    indices = torch.empty((nnz, 3), dtype=torch.int64, device=dev)
    values = torch.empty(nnz, dtype=torch.int64, device=dev)
    if nnz:
        check(lib.eu_sparse_get_adj_coo(*args, nnz, rowptr.data_ptr(), indices.data_ptr(), values.data_ptr()))
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
        ctx = _ctx_on_stream()
        check(_lib.load().eu_sample_neighbor_layerwise(ctx._h, nd.data_ptr(), batch, n, et.ctypes.data, len(et), count, default_node,
                                                       1 if weight_func == 'sqrt' else 0, out.data_ptr(), None))
    return out, _adj_coo(nd.reshape(-1), out.reshape(-1), batch, n, count, et)


def gen_pair(paths, left_win_size, right_win_size):
    """walk_ops.gen_pair (tf_euler/kernels/gen_pair_op.cc): skip-gram pairs i64[B, n_pairs, 2] of walks i64[B, path_len]."""
    paths = _t(paths, torch.int64)
    if paths.dim() != 2:
        raise EulerError("gen_pair: paths must be [batch, path_len]")
    paths = paths.contiguous()
    B, plen = paths.shape
    lib = _lib.load()
    pc = lib.eu_gen_pair_count(plen, int(left_win_size), int(right_win_size))
    out = torch.empty((B, pc, 2), dtype=torch.int64, device=paths.device)
    ctx = _ctx_on_stream()
    check(lib.eu_gen_pair(ctx._h, paths.data_ptr(), B, plen, int(left_win_size), int(right_win_size), out.data_ptr()))
    return out


def sample_neighbor_api(nodes, edge_types, count):
    """euler::SampleNeighbor of the C++ api (api.cc:223-236): NO unique / gather -- a repeated id draws again.  Returns
    engine-form (ids i64[N,count], w, t); rows without a result are (0, 0.0, -1)."""
    nodes = _t(nodes, torch.int64).reshape(-1)
    et = get_edge_type_id(edge_types)
    n, count = nodes.numel(), int(count)
    ids = torch.empty((n, count), dtype=torch.int64, device=nodes.device)
    w = torch.empty((n, count), dtype=torch.float32, device=nodes.device)
    t = torch.empty((n, count), dtype=torch.int32, device=nodes.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_neighbor_raw(ctx._h, nodes.data_ptr(), n, et.ctypes.data, len(et), count,
                                             ids.data_ptr(), w.data_ptr(), t.data_ptr()))
    return ids, w, t


def unique(ids):
    """tf.unique on the device (eu_unique): (values in first-occurrence order, inverse i32 with ids == values[inverse])."""
    ids = _t(ids, torch.int64).reshape(-1)
    n = ids.numel()
    vals = torch.empty(n, dtype=torch.int64, device=ids.device)
    inv = torch.empty(n, dtype=torch.int32, device=ids.device)
    cnt = torch.zeros(1, dtype=torch.int64, device=ids.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_unique(ctx._h, ids.data_ptr(), n, vals.data_ptr(), inv.data_ptr(), cnt.data_ptr()))
    return vals[:int(cnt.item())], inv


def sage_mean_aggregate(neighbor_ids, count, dim):
    """Fused get_dense_feature + scatter_mean for fixed-fanout blocks (SAGEConv's neighbor mean,
    tf_euler/python/convolution/sage_conv.py:33-38 over sage_dataflow.py:43-46 blocks)."""
    ids = _t(neighbor_ids, torch.int64).reshape(-1)
    rows = ids.numel() // int(count)
    out = torch.empty((rows, int(dim)), dtype=torch.float32, device=ids.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sage_mean_aggregate(ctx._h, ids.data_ptr(), rows, int(count), int(dim),
                                             out.data_ptr()))
    return out


# ------------------------------------------------------------------------------------ mp ops
def _raw_gather(params, indices):
    params = params.contiguous()
    out = torch.empty((indices.numel(), params.shape[1]), dtype=torch.float32, device=params.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_gather(ctx._h, params.data_ptr(), params.shape[0], params.shape[1],
                                indices.data_ptr(), indices.numel(), out.data_ptr()))
    return out


def _raw_scatter(name, updates, indices, size):
    updates = updates.contiguous()
    out = torch.empty((int(size), updates.shape[1]), dtype=torch.float32, device=updates.device)
    ctx = _ctx_on_stream()
    check(getattr(_lib.load(), name)(ctx._h, updates.data_ptr(), updates.shape[1], indices.data_ptr(),
                                     indices.numel(), int(size), out.data_ptr()))
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


def gather(params, indices):
    """mp_ops.gather = MPGather (mp_ops.py:27): out[i,:] = params[indices[i],:]."""
    return _Gather.apply(_f32(params), _t(indices, torch.int32).reshape(-1))


def scatter_add(updates, indices, size=None):
    """mp_ops.scatter_add = MPScatterAdd (mp_ops.py:28)."""
    return _ScatterAdd.apply(_f32(updates), _t(indices, torch.int32).reshape(-1), int(size))


def scatter_max(updates, indices, size=None):
    """mp_ops.scatter_max = MPScatterMax (mp_ops.py:29); output initialised to -1e9."""
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
    ctx = _ctx_on_stream()
    check(_lib.load().eu_gat_aggregate(ctx._h, h_src.data_ptr(), s_dst.data_ptr(), s_src.data_ptr(), dst.data_ptr(),
                                       src.data_ptr(), E, n_dst, n_src, H, h_src.shape[1] // H, out.data_ptr(),
                                       alpha.data_ptr() if with_alpha else None))
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
        ec = _ctx_on_stream()
        check(_lib.load().eu_gat_aggregate_backward(ec._h, grad.data_ptr(), h_src.data_ptr(), alpha.data_ptr(), s_dst.data_ptr(),
                                                    s_src.data_ptr(), dst.data_ptr(), src.data_ptr(), dst.numel(), n_dst, n_src,
                                                    H, C, g_h.data_ptr(), g_sd.data_ptr(), g_ss.data_ptr()))
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
    ei = _t(edge_index, torch.int32)
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise EulerError("gat_attention_aggregate: edge_index must be [2, E]")
    dst, src = ei[0].contiguous(), ei[1].contiguous()
    return _GatAggregate.apply(h_src, s_dst, s_src, dst, src, n_dst)


def _raw_agnn(x_src, nrm_dst, nrm_src, beta, dst, src, n_dst, with_alpha):
    """one eu_agnn_aggregate: (out f32[n_dst, dim], alpha f32[E] or None, cos f32[E] or None)"""
    n_src, dim = x_src.shape
    E = dst.numel()
    dev = x_src.device
    out = torch.empty((n_dst, dim), dtype=torch.float32, device=dev)
    alpha = torch.empty(E, dtype=torch.float32, device=dev) if with_alpha else None
    cos = torch.empty(E, dtype=torch.float32, device=dev) if with_alpha else None
    ctx = _ctx_on_stream()
    check(_lib.load().eu_agnn_aggregate(ctx._h, x_src.data_ptr(), nrm_dst.data_ptr(), nrm_src.data_ptr(), beta.data_ptr(),
                                        dst.data_ptr(), src.data_ptr(), E, n_dst, n_src, dim, out.data_ptr(),
                                        alpha.data_ptr() if with_alpha else None, cos.data_ptr() if with_alpha else None))
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
        ec = _ctx_on_stream()
        check(_lib.load().eu_agnn_aggregate_backward(ec._h, grad.data_ptr(), x_src.data_ptr(), nrm_dst.data_ptr(), nrm_src.data_ptr(),
                                                     beta.data_ptr(), alpha.data_ptr(), cos.data_ptr(), dst.data_ptr(),
                                                     src.data_ptr(), dst.numel(), ctx.n_dst, n_src, dim, g_x.data_ptr(),
                                                     g_nd.data_ptr(), g_ns.data_ptr(), g_beta.data_ptr()))
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
    named = (("x_src", x_src), ("nrm_dst", nrm_dst), ("nrm_src", nrm_src), ("beta", beta))
    for nm, t in named:
        if not torch.is_tensor(t) or t.dtype != torch.float32:
            raise EulerError("agnn_attention_aggregate: %s must be a float32 tensor" % nm)
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
    ei = _t(edge_index, torch.int32)
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise EulerError("agnn_attention_aggregate: edge_index must be [2, E]")
    dst, src = ei[0].contiguous(), ei[1].contiguous()
    return _AgnnAggregate.apply(x_src, nrm_dst, nrm_src, b, dst, src, n_dst)


def _raw_relation(x_src, matrix, rel, dst, src, n_dst):
    """one eu_relation_aggregate: out f32[n_dst, D]"""
    n_src, F = x_src.shape
    R, D = matrix.shape[0], matrix.shape[1]
    out = torch.empty((n_dst, D), dtype=torch.float32, device=x_src.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_relation_aggregate(ctx._h, x_src.data_ptr(), matrix.data_ptr(), rel.data_ptr(), dst.data_ptr(),
                                            src.data_ptr(), dst.numel(), n_dst, n_src, R, D, F, out.data_ptr()))
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
        ec = _ctx_on_stream()
        check(_lib.load().eu_relation_aggregate_backward(ec._h, grad.data_ptr(), x_src.data_ptr(), matrix.data_ptr(), rel.data_ptr(),
                                                         dst.data_ptr(), src.data_ptr(), dst.numel(), ctx.n_dst, n_src, R, D, F,
                                                         g_x.data_ptr(), g_m.data_ptr()))
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
    for nm, t in (("x_src", x_src), ("matrix", matrix)):
        if not torch.is_tensor(t) or t.dtype != torch.float32:
            raise EulerError("relation_mean_aggregate: %s must be a float32 tensor" % nm)
    if x_src.dim() != 2 or matrix.dim() != 3:
        raise EulerError("relation_mean_aggregate: need x_src [n_src, F] (2-D) and matrix [R, D, F] (3-D); got %s, %s"
                         % (tuple(x_src.shape), tuple(matrix.shape)))
    R, D, F = matrix.shape
    if R < 1 or D < 1 or F < 1 or x_src.shape != (n_src, F):
        raise EulerError("relation_mean_aggregate: need x_src [n_src, F] = [%d, %d] and a non-empty matrix [R, D, F]; got %s, %s"
                         % (n_src, F, tuple(x_src.shape), tuple(matrix.shape)))
    if not torch.is_tensor(edge_attr) or edge_attr.dtype.is_floating_point or edge_attr.dtype.is_complex:
        raise EulerError("relation_mean_aggregate: edge_attr must be an integer tensor")
    ei = _t(edge_index, torch.int32)
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise EulerError("relation_mean_aggregate: edge_index must be [2, E]")
    if edge_attr.numel() != ei.shape[1]:
        raise EulerError("relation_mean_aggregate: edge_attr has %d entries for %d edges" % (edge_attr.numel(), ei.shape[1]))
    rel = _t(edge_attr, torch.int32).reshape(-1)
    dst, src = ei[0].contiguous(), ei[1].contiguous()
    return _RelationAggregate.apply(_t(x_src, torch.float32), _t(matrix, torch.float32), rel, dst, src, n_dst)


def _raw_dna(q, k, v, n0, n1, dst, src, n_dst, heads, with_alpha):
    """one eu_dna_aggregate: (out f32[n_dst, dim], alpha f32[E, H, H] or None)"""
    n_src, dim = k.shape
    E = dst.numel()
    out = torch.empty((n_dst, dim), dtype=torch.float32, device=q.device)
    alpha = torch.empty((E, heads, heads), dtype=torch.float32, device=q.device) if with_alpha else None
    ctx = _ctx_on_stream()
    check(_lib.load().eu_dna_aggregate(ctx._h, q.data_ptr(), k.data_ptr(), v.data_ptr(), n0.data_ptr(), n1.data_ptr(),
                                       dst.data_ptr(), src.data_ptr(), E, n_dst, n_src, heads, dim // heads, out.data_ptr(),
                                       alpha.data_ptr() if with_alpha else None))
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
        ec = _ctx_on_stream()
        check(_lib.load().eu_dna_aggregate_backward(ec._h, grad.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), n0.data_ptr(),
                                                    n1.data_ptr(), alpha.data_ptr(), dst.data_ptr(), src.data_ptr(), dst.numel(),
                                                    n_dst, n_src, H, dim // H, g_q.data_ptr(), g_k.data_ptr(), g_v.data_ptr()))
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
    for nm, t in (("q", q), ("k", k), ("v", v), ("n0", n0), ("n1", n1)):
        if not torch.is_tensor(t) or t.dtype != torch.float32:
            raise EulerError("dna_attention_aggregate: %s must be a float32 tensor" % nm)
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
    ei = _t(edge_index, torch.int32)
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise EulerError("dna_attention_aggregate: edge_index must be [2, E]")
    dst, src = ei[0].contiguous(), ei[1].contiguous()
    q, k, v = (_t(t, torch.float32) for t in (q, k, v))
    n0, n1 = (_t(t, torch.float32).detach().reshape(-1) for t in (n0, n1))
    return _DnaAggregate.apply(q, k, v, n0, n1, dst, src, n_dst, heads)


_COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}


def _raw_embedding(nodes, fid, table, default_value, comb):
    """one eu_sparse_embedding_lookup: out f32[M, dim]"""
    n_rows, dim = table.shape
    out = torch.empty((nodes.numel(), dim), dtype=torch.float32, device=table.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sparse_embedding_lookup(ctx._h, nodes.data_ptr(), nodes.numel(), fid, default_value, table.data_ptr(), n_rows,
                                                 dim, comb, out.data_ptr()))
    return out


class _SparseEmbedding(torch.autograd.Function):
    """eu_sparse_embedding_lookup / eu_sparse_embedding_lookup_backward.  Saves only the node ids: the backward pass lists the
    entries again from the graph."""

    @staticmethod
    def forward(ctx, table, nodes, fid, default_value, comb):
        out = _raw_embedding(nodes, fid, table, default_value, comb)
        if ctx.needs_input_grad[0]:
            ctx.save_for_backward(nodes)
        ctx.args = (fid, default_value, comb, table.shape)
        return out

    @staticmethod
    def backward(ctx, grad):
        nodes, = ctx.saved_tensors
        fid, default_value, comb, (n_rows, dim) = ctx.args
        grad = grad.contiguous()
        g_t = torch.empty((n_rows, dim), dtype=torch.float32, device=grad.device)
        ec = _ctx_on_stream()
        check(_lib.load().eu_sparse_embedding_lookup_backward(ec._h, grad.data_ptr(), nodes.data_ptr(), nodes.numel(), fid, default_value,
                                                              n_rows, dim, comb, g_t.data_ptr()))
        return g_t, None, None, None, None


def sparse_feature_embedding(nodes, feature_name, table, default_value, combiner='sum'):
    """SparseEmbedding over get_sparse_feature in one fused device op: row i is tf.nn.embedding_lookup_sparse(table, sp_ids,
    None, combiner) (layers.py:152-169) of the SparseTensor get_sparse_feature(nodes, [feature_name], [default_value]) returns,
    i.e. the rows of table f32[n_rows, dim] named by node i's uint64 values of the slot, in stored order, or the one row
    default_value for a node without values; combined by 'sum', 'mean' or 'sqrtn'.  The sum runs left to right from the first
    row, mean / sqrtn divide once (include/euler_b200.h).  Every value of the slot and default_value must lie in [0, n_rows):
    the call raises otherwise, before any device work.  The gradient reaches table only (deterministic, no atomics); the
    forward does not synchronise, the backward synchronises once."""
    if combiner not in _COMBINERS:
        raise EulerError("sparse_feature_embedding: combiner must be one of %s, got %r" % (sorted(_COMBINERS), combiner))
    if not torch.is_tensor(table) or table.dtype != torch.float32 or table.dim() != 2:
        raise EulerError("sparse_feature_embedding: table must be a 2-D float32 tensor")
    fid = feature_name if isinstance(feature_name, (int, np.integer)) else get_graph().sparse_feature_id(str(feature_name))
    nodes = _t(nodes, torch.int64).reshape(-1)
    return _SparseEmbedding.apply(_t(table, torch.float32), nodes, int(fid), int(default_value), _COMBINERS[combiner])


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
    ctx = _ctx_on_stream()
    check(_lib.load().eu_sample_graph_label(ctx._h, count, out.data_ptr()))
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
    lib, ctx = _lib.load(), _ctx_on_stream()
    ptr = torch.empty(B + 1, dtype=torch.int64, device=labels.device)
    total, max_len = C.c_int64(), C.c_int64()
    check(lib.eu_get_graph_by_label(ctx._h, labels.data_ptr(), B, 0, ptr.data_ptr(), None, None, C.byref(total), C.byref(max_len)))
    nnz = total.value
    indices = torch.empty((nnz, 2), dtype=torch.int64, device=labels.device)
    values = torch.empty(nnz, dtype=torch.int64, device=labels.device)
    if nnz:
        check(lib.eu_get_graph_by_label(ctx._h, labels.data_ptr(), B, nnz, ptr.data_ptr(), indices.data_ptr(), values.data_ptr(),
                                        None, None))
    return indices, values, (B, max_len.value)


def _raw_readout(x, index, size, logits, q):
    """one eu_graph_attention_readout: (out f32[size, D], alpha f32[N])"""
    N, D = x.shape
    out = torch.empty((size, D), dtype=torch.float32, device=x.device)
    alpha = torch.empty(N, dtype=torch.float32, device=x.device)
    ctx = _ctx_on_stream()
    check(_lib.load().eu_graph_attention_readout(ctx._h, x.data_ptr(), index.data_ptr(), N, size, D,
                                                 logits.data_ptr() if logits is not None else None,
                                                 q.data_ptr() if q is not None else None, out.data_ptr(), alpha.data_ptr()))
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
        q = weight if ctx.by_query else None
        ec = _ctx_on_stream()
        check(_lib.load().eu_graph_attention_readout_backward(ec._h, grad.data_ptr(), x.data_ptr(), index.data_ptr(), N, ctx.size,
                                                              D, q.data_ptr() if q is not None else None, alpha.data_ptr(),
                                                              g_x.data_ptr(), None if ctx.by_query else g_w.data_ptr(),
                                                              g_w.data_ptr() if ctx.by_query else None))
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
    if not torch.is_tensor(x) or x.dim() != 2 or x.dtype != torch.float32:
        raise EulerError("graph_attention_readout: x must be a 2-D float32 tensor")
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
