"""numpy restatements of tf.nn.embedding_lookup_sparse (layers.SparseEmbedding) over get_sparse_feature's bags, and random
graphs with uint64 feature slots.  (Test infrastructure.)"""
import numpy as np

COMBINERS = ("sum", "mean", "sqrtn")


def bags(ids, u64_ptr, u64_val, S, nodes, fid, default):
    """get_sparse_feature's entries per node: the node's values of slot fid in stored order, or [default] when it has none
    (absent id, empty or unknown slot)"""
    ids = np.asarray(ids, np.uint64)
    order = np.argsort(ids, kind="stable")
    q = np.asarray(nodes, np.int64).reshape(-1).astype(np.uint64)
    pos = np.minimum(np.searchsorted(ids[order], q), len(ids) - 1)
    rows = np.where(ids[order][pos] == q, order[pos], -1)
    out = []
    for r in rows:
        vals = []
        if r >= 0 and 0 <= fid < S:
            vals = [int(v) for v in u64_val[u64_ptr[r * S + fid]:u64_ptr[r * S + fid + 1]]]
        out.append(vals if vals else [int(default)])
    return out


def lookup_f32(table, bag_list, combiner):
    """the op's defined float32 order: the first row, then left-to-right adds; mean / sqrtn divide once by fl(n) /
    sqrtf(fl(n))"""
    table = np.asarray(table, np.float32)
    out = np.empty((len(bag_list), table.shape[1]), np.float32)
    for i, b in enumerate(bag_list):
        acc = table[b[0]].copy()
        for v in b[1:]:
            acc = (acc + table[v]).astype(np.float32)
        n = np.float32(len(b))
        if combiner == "mean":
            acc = (acc / n).astype(np.float32)
        elif combiner == "sqrtn":
            acc = (acc / np.sqrt(n)).astype(np.float32)
        out[i] = acc
    return out


def lookup_f64(table, bag_list, combiner):
    table = np.asarray(table, np.float64)
    out = np.empty((len(bag_list), table.shape[1]))
    for i, b in enumerate(bag_list):
        acc = table[b].sum(axis=0)
        out[i] = acc / {"sum": 1.0, "mean": len(b), "sqrtn": np.sqrt(len(b))}[combiner]
    return out


def grad_f64(grad_out, bag_list, n_rows, combiner):
    """d(sum(out * grad_out)) / d table, in float64"""
    g = np.zeros((n_rows, grad_out.shape[1]))
    for i, b in enumerate(bag_list):
        s = {"sum": 1.0, "mean": len(b), "sqrtn": np.sqrt(len(b))}[combiner]
        for v in b:
            g[v] += np.asarray(grad_out[i], np.float64) / s
    return g


def tf_pack(eng, default_node):
    """SampleFanoutWithFeature's packing of one hop (sample_fanout_with_feature_op.cc:196-218): eng = the engine's ids
    [rows, count], 0 (DEFAULT_UINT64) where a row has no result.  A row whose FIRST id is 0 keeps the default fill --
    default_node, weight 0, type -1 -- even when that 0 is a real draw of node 0; every other row is copied."""
    eng = np.asarray(eng, np.int64)
    keep = eng[:, :1] != 0
    return np.where(keep, eng, np.int64(default_node)), keep[:, 0]


def slot_graph(seed, n, lens_of_slot, vals_of_slot, node0=False, feat_dim=0):
    """A small random graph (tests/graphs.random_graph) with len(lens_of_slot) uint64 slots.  lens_of_slot[s](rng, n) gives
    the per-node lengths of slot s, vals_of_slot[s](rng, k) k values.  node0 = True makes the first node's id 0."""
    import graphs
    g = graphs.random_graph(seed=seed, n=n, T=1, avg_deg=4, id_base=0 if node0 else 1, feat_dim=feat_dim)
    rng = np.random.RandomState(seed + 1)
    S = len(lens_of_slot)
    lens = np.stack([np.asarray(f(rng, n), np.int64) for f in lens_of_slot], axis=1)   # [n, S]
    ptr = np.zeros(n * S + 1, np.int64)
    ptr[1:] = np.cumsum(lens.reshape(-1))
    vals = np.empty(int(ptr[-1]), np.uint64)
    for r in range(n):
        for s in range(S):
            b, e = ptr[r * S + s], ptr[r * S + s + 1]
            vals[b:e] = np.asarray(vals_of_slot[s](rng, int(e - b)), np.uint64)
    g.update(u64_ptr=ptr, u64_val=vals, S=S)
    return g


def cuda_slot_graph(g):
    import euler_b200
    return euler_b200.Graph.from_csr(g["ids"], g["grp_ptr"], g["nbr"], n_edge_types=g["T"], node_type=g["node_type"],
                                     node_w=g["node_w"], cum_w=g["cum_w"], feat=g.get("feat"), u64_ptr=g["u64_ptr"], u64_val=g["u64_val"],
                                     n_u64_slots=g["S"])


def composed_parts(nodes, id_table, dense, sparse):
    """the single ops ShallowEncoder's row is made of, on the device: ([F.embedding(nodes, id_table)] or [],
    get_dense_feature's slots, [sparse_feature_embedding per (name, table, default, combiner)])"""
    import torch
    import torch.nn.functional as F
    import euler_b200
    nd = torch.as_tensor(nodes, device="cuda")
    idp = [F.embedding(nd, id_table)] if id_table is not None else []
    dp = euler_b200.get_dense_feature(nd, [n for n, _ in dense], [d for _, d in dense]) if dense else []
    sp = [euler_b200.sparse_feature_embedding(nd, n, t, dv, c) for n, t, dv, c in sparse]
    return idp, dp, sp


def pool_f32(rows, count, pool):
    """shallow_encode_pool's defined order over shallow_encode's rows [R count, W], in float32 on the host: each column added
    left to right from the segment's first row, mean divided once by fl(count)"""
    x = rows.cpu().numpy().reshape(-1, count, rows.shape[1])
    acc = x[:, 0].copy()
    for j in range(1, count):
        acc = acc + x[:, j]
    return acc / np.float32(count) if pool == "mean" else acc


def shallow_problem(nodes, id_table, dense, sparse, comb=0):
    """the eu_shallow_problem of shallow_encode's arguments (names resolved on the installed graph), for raw library calls"""
    import euler_b200
    from euler_b200 import ops
    g = euler_b200.get_graph()
    res = [(g.sparse_feature_id(n), t, dv, ops._COMBINERS[c]) for n, t, dv, c in sparse]
    return ops._shallow_problem(nodes, id_table, [(g.dense_feature_id(n) if isinstance(n, str) else n, d) for n, d in dense], res, comb)
