"""Multi-GPU path: the graph is hash-partitioned by node id over the ranks of one box (Euler's own
shard scheme) and every hop / feature fetch resolves remote ids with an all-to-all over NVLink.

Reference being replaced (mode=remote): ID_SPLIT -> REMOTE (gRPC Execute of a sub-DAG on each shard
server) -> IDX_MERGE / DATA_MERGE, euler/core/kernels/id_split_op.cc:46-99, remote_op.cc:60-146,
idx_merge_op.cc:32-78, discovery through ZooKeeper.  Here: one process per GPU, torch.distributed
(NCCL) for the exchange, CUDA kernels (csrc/shard.cu) for routing and merging.

Per hop on every rank
    bucket seeds by owner (stable)            eu_shard_bucket
    exchange per-owner counts                 all_to_all (N ints; the only host sync of the hop)
    exchange seeds                            all_to_all_v  (8 B / seed)
    sample the received seeds on this shard   eu_sample_neighbor  (this shard's own engine)
    exchange the rows back                    all_to_all_v  (one 16 B record {id, w | t<<32} per slot)
    merge into request order + TF packing     eu_shard_merge_sample

Determinism / parity: a shard processes the concatenation of the requests of rank 0, 1, ... (each in
batch order) as ONE sampleNB call on its own engine, so duplicate seeds -- also across requesters --
share one sample row and the draw order is fixed.  The reference runs every request on whichever
server thread picks it up (thread_local engines, random.cc:22), i.e. it has no defined order here;
tests/test_sharded_*.py pin this definition against the oracle.

The exchange and the per-shard ops are injected (`ops`, `xchg`) so the same orchestration runs over
gloo on CPU in the tests.
"""
import ctypes as C

import numpy as np


def owner_of(ids, num_partitions, shard_num, self_shard=None):
    """euler/core/kernels/id_split_op.cc:46-49 (ids as uint64).  With self_shard given, ids 0 and 2^64-1
    (engine placeholder / default fill: they exist on no shard) stay on the requesting rank."""
    a = np.asarray(ids).astype(np.uint64)
    own = (a % np.uint64(num_partitions)) % np.uint64(shard_num)
    if self_shard is not None:
        own = np.where((a == 0) | (a == np.uint64(0xFFFFFFFFFFFFFFFF)), np.uint64(self_shard), own)
    return own


class ClientRng:
    """The requesting side's engine: std::minstd_rand0 + libstdc++ generate_canonical<double,53>, the thread-local
    generator of euler/common/random.cc:22-28 (the same stream arithmetic as csrc/common.cuh::minstd_uniform)."""
    M, A = 2147483647, 16807

    def __init__(self, seed=1):
        self.x = int(seed) % self.M or 1

    def uniform(self):
        import math
        R = 2147483646.0
        self.x = self.x * self.A % self.M
        s = float(self.x - 1)
        self.x = self.x * self.A % self.M
        s = s + float(self.x - 1) * R
        r = s / (R * R)
        return math.nextafter(1.0, 0.0) if r >= 1.0 else r


def split_sample_count(count, node_types, shard_weight, rng):
    """SAMPLE_NODE_SPLIT (euler/core/kernels/sample_node_split_op.cc:38-85): how many of `count` draws each shard serves.
    shard_weight: f32[n_types + 1][N + 1] = QueryProxy::GetShardNodeWeight() (row n_types = all types, column N = total).
    floor(count * w_shard / w_total) in f32 each, the remainder handed out one by one to non-empty shards picked with the
    CLIENT's engine (one uniform per leftover draw, :79-83)."""
    import math
    w = np.asarray(shard_weight, np.float32)
    N = w.shape[1] - 1
    types = [int(t) for t in node_types]
    if -1 in types:
        if len(types) > 1:
            raise ValueError("sample_node: -1 (all types) cannot be mixed with other node types")   # EULER_LOG(FATAL) :61-63
        types = [w.shape[0] - 1]
    split, nonzero, remain = [], [], int(count)
    for i in range(N):
        s0, s1 = np.float32(0), np.float32(0)
        for t in types:
            s0 = np.float32(s0 + w[t][i])
            s1 = np.float32(s1 + w[t][N])
        if abs(float(s1)) < 1e-7:
            raise ValueError("sample_node: node type sum weight is zero")                              # :69-71
        c = int(math.floor(float(np.float32(np.float32(np.float32(count) * s0) / s1))))
        split.append(c)
        if s0 > 0:
            nonzero.append(i)
        remain -= c
    while remain > 0:
        split[nonzero[int(math.floor(rng.uniform() * len(nonzero)))]] += 1
        remain -= 1
    return split


def shard_weight_table(per_shard_type_sums):
    """per_shard_type_sums: [N][n_types] node-weight sums (f64).  Returns f32[n_types + 1][N + 1] laid out like
    GetShardNodeWeight(): row t = type t, last row = all types; column s = shard s, last column = total."""
    a = np.asarray(per_shard_type_sums, np.float64)          # [N, n_types]
    N, nt = a.shape
    out = np.zeros((nt + 1, N + 1), np.float64)
    out[:nt, :N] = a.T
    out[nt, :N] = a.sum(axis=1)
    out[:, N] = out[:, :N].sum(axis=1)
    return out.astype(np.float32)


class TorchExchange:
    """all-to-all over a torch.distributed process group (NCCL for CUDA tensors, gloo for CPU)."""

    def __init__(self, group=None):
        import torch.distributed as dist
        self.dist, self.group = dist, group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)

    def counts(self, send_counts_t):
        """send_counts_t: int64[world] tensor (device of the backend).  Returns (send, recv) lists."""
        import torch
        recv = torch.empty_like(send_counts_t)
        self.dist.all_to_all_single(recv, send_counts_t, group=self.group)
        both = torch.stack([send_counts_t, recv]).cpu()   # the hop's single host sync
        return both[0].tolist(), both[1].tolist()

    def a2a(self, t, send, recv, width=1):
        """t: [sum(send) * width] flat tensor; returns [sum(recv) * width]."""
        import torch
        out = torch.empty(int(sum(recv)) * width, dtype=t.dtype, device=t.device)
        self.dist.all_to_all_single(out, t, [int(r) * width for r in recv], [int(s) * width for s in send],
                                    group=self.group)
        return out


class CudaShardOps:
    """Per-shard work on this rank's GPU through the C ABI."""

    def __init__(self, graph, rng="minstd", seed=1):
        import torch
        from . import _lib
        from .graph import Context
        self.torch, self.lib, self.check = torch, _lib.load(), _lib.check
        self.graph = graph
        self.dev = torch.device("cuda", graph.device)
        self.ctx = Context(graph, rng, seed)

    def _stream(self):
        self.ctx.set_stream(self.torch.cuda.current_stream(self.dev).cuda_stream)
        return self.ctx._h

    def to_dev(self, a, dtype):
        t = self.torch
        if isinstance(a, t.Tensor):
            return a.to(device=self.dev, dtype=dtype).contiguous()
        return t.as_tensor(np.asarray(a), dtype=dtype, device=self.dev).contiguous()

    def bucket(self, ids, P, N, me):
        t = self.torch
        rows = ids.numel()
        sorted_ids = t.empty(rows, dtype=t.int64, device=self.dev)
        src = t.empty(rows, dtype=t.int32, device=self.dev)
        counts = t.empty(N, dtype=t.int64, device=self.dev)
        offs = t.empty(N + 1, dtype=t.int64, device=self.dev)
        self.check(self.lib.eu_shard_bucket(self._stream(), ids.data_ptr(), rows, P, N, me, sorted_ids.data_ptr(),
                                            src.data_ptr(), counts.data_ptr(), offs.data_ptr()))
        return sorted_ids, src, counts

    def sample_local(self, seeds, etypes, count):
        """Engine-form rows for the received seeds: ids with 0 placeholders, w 0, t -1 on empty rows."""
        t = self.torch
        n = seeds.numel()
        et = np.ascontiguousarray(etypes, dtype=np.int32)
        ids = t.empty(n * count, dtype=t.int64, device=self.dev)
        w = t.empty(n * count, dtype=t.float32, device=self.dev)
        ty = t.empty(n * count, dtype=t.int32, device=self.dev)
        self.check(self.lib.eu_sample_neighbor(self._stream(), seeds.data_ptr(), n, et.ctypes.data, len(et), count, 0,
                                               ids.data_ptr(), w.data_ptr(), ty.data_ptr()))
        packed = t.empty(n * count * 2, dtype=t.int64, device=self.dev)
        self.check(self.lib.eu_shard_pack_sample(self._stream(), ids.data_ptr(), w.data_ptr(), ty.data_ptr(), n * count,
                                                 packed.data_ptr()))
        return packed

    def merge_sample(self, packed, src, rows, count, default_node):
        t = self.torch
        eng = t.empty(rows * count, dtype=t.int64, device=self.dev)
        o_ids = t.empty(rows * count, dtype=t.int64, device=self.dev)
        o_w = t.empty(rows * count, dtype=t.float32, device=self.dev)
        o_t = t.empty(rows * count, dtype=t.int32, device=self.dev)
        self.check(self.lib.eu_shard_merge_sample(self._stream(), packed.data_ptr(),
                                                  src.data_ptr(), rows, count, default_node, eng.data_ptr(),
                                                  o_ids.data_ptr(), o_w.data_ptr(), o_t.data_ptr()))
        return eng, o_ids, o_w, o_t

    def node_weight_sums(self):
        """per node type: sum of this shard's node weights (f64), the shard's column of GetShardNodeWeight()"""
        ex = self.graph.export(with_feat=False)
        nt = int(self.graph.num_node_types)
        return np.bincount(ex["node_type"], weights=ex["node_w"].astype(np.float64), minlength=nt)

    def sample_node_local(self, n, node_types):
        t = self.torch
        out = t.empty(n, dtype=t.int64, device=self.dev)
        types = np.ascontiguousarray(node_types, dtype=np.int32)
        if n:
            self.check(self.lib.eu_sample_node(self._stream(), n, types.ctypes.data, len(types), out.data_ptr()))
        return out

    def feature_local(self, ids, fid, dim):
        t = self.torch
        out = t.empty(ids.numel() * dim, dtype=t.float32, device=self.dev)
        self.check(self.lib.eu_get_dense_feature(self._stream(), ids.data_ptr(), ids.numel(), fid, dim, out.data_ptr()))
        return out

    def merge_rows(self, rows_in, src, rows, dim):
        t = self.torch
        out = t.empty((rows, dim), dtype=t.float32, device=self.dev)
        self.check(self.lib.eu_shard_merge_rows(self._stream(), rows_in.data_ptr(), src.data_ptr(), rows, dim,
                                                out.data_ptr()))
        return out

    def seed(self, s):
        self.ctx.seed(s)


class ShardedGraph:
    """tf_euler's sampling / feature ops over a graph partitioned across the ranks of `xchg`."""

    def __init__(self, ops, xchg, num_partitions=None, feature_ops=None):
        """feature_ops: per-rank ops over a graph that holds EVERY node's dense features (replicated feature table: 5 GB at
        BASELINE configs[1] against 80 GB of HBM); when given, get_dense_feature runs locally and only the sampling hops
        use the exchange (DESIGN.md section 8, item 1).  None = Euler's scheme: features live with their rows."""
        self.ops, self.xchg = ops, xchg
        self.N = xchg.world
        self.P = num_partitions or self.N   # partitions a multiple of shards -> owner = id % N
        self._shard_w = None
        self.feature_ops = feature_ops

    def sample_neighbor(self, nodes, edge_types, count, default_node=-1):
        eng, ids, w, t = self._hop(self.ops.to_dev(nodes, _i64(self.ops)), edge_types, count, default_node)
        shape = (-1, count)
        return ids.reshape(shape), w.reshape(shape), t.reshape(shape)

    def sample_fanout(self, nodes, edge_types, counts, default_node=-1):
        """neighbor_ops.sample_fanout (tf_euler/python/euler_ops/neighbor_ops.py:122-158): the next hop's
        seeds are the ENGINE ids of this hop (0 placeholders), tf_euler/kernels/sample_fanout_op.cc:36-43."""
        frontier = self.ops.to_dev(nodes, _i64(self.ops)).reshape(-1)
        ids, ws, ts = [frontier], [], []
        for et, c in zip(edge_types, counts):
            frontier, o_ids, o_w, o_t = self._hop(frontier, et, int(c), default_node)
            ids.append(o_ids); ws.append(o_w); ts.append(o_t)
        return ids, ws, ts

    def _hop(self, frontier, etypes, count, default_node):
        ops, x = self.ops, self.xchg
        rows = frontier.numel()
        sorted_ids, src, counts = ops.bucket(frontier, self.P, self.N, x.rank)
        send, recv = x.counts(counts)
        inbox = x.a2a(sorted_ids, send, recv)
        packed = ops.sample_local(inbox, etypes, count)            # 16-byte records {id, w | t << 32}
        back = x.a2a(packed, recv, send, count * 2)
        return ops.merge_sample(back, src, rows, count, default_node)

    def random_walk(self, nodes, edge_types, p=1.0, q=1.0, default_node=-1):
        """walk_ops.random_walk over shards for p = q = 1 (TraditionalRandomWalk, tf_euler/kernels/random_walk_op.cc:170-232):
        L chained sampleNB(count = 1) hops whose frontier is the ENGINE id (0 placeholder), one exchange per step; returns
        [B, L+1] with default_node where the walk has died.  The biased node2vec step needs the parent's adjacency on the
        walker's shard and is not sharded yet."""
        if abs(float(p) - 1.0) > 1e-6 or abs(float(q) - 1.0) > 1e-6:
            raise NotImplementedError("sharded random_walk: only p = q = 1 (node2vec across shards is not built)")
        ops = self.ops
        frontier = ops.to_dev(nodes, _i64(ops)).reshape(-1)
        cols = [frontier]
        for et in edge_types:
            frontier, o_ids, _, _ = self._hop(frontier, et, 1, default_node)
            cols.append(o_ids)
        return ops.torch.stack(cols, dim=1)

    def sample_node(self, count, node_types, client_rng):
        """sample_ops.sample_node over shards (SAMPLE_NODE_SPLIT -> per-shard API_SAMPLE_NODE -> merge in shard order,
        euler/core/kernels/sample_node_split_op.cc:38-110): this rank's `count` draws are split over the shards in
        proportion to their node-weight sums; every shard serves the requests of rank 0..N-1 in rank order on its own
        engine; the result is the concatenation in shard order.  Collective: every rank calls it with the same
        node_types.  client_rng: this rank's ClientRng (the remainder draws)."""
        ops, x = self.ops, self.xchg
        if self._shard_w is None:
            import torch
            mine = torch.as_tensor(np.asarray(ops.node_weight_sums(), np.float64))
            mine = ops.to_dev(mine, torch.float64)
            allw = [torch.empty_like(mine) for _ in range(self.N)]
            x.dist.all_gather(allw, mine, group=x.group)
            self._shard_w = shard_weight_table(np.stack([a.cpu().numpy() for a in allw]))
        split = split_sample_count(count, node_types, self._shard_w, client_rng)
        send, recv = x.counts(ops.to_dev(np.asarray(split, np.int64), _i64(ops)))
        served = [ops.sample_node_local(int(n), node_types) for n in recv]        # rank order, one call per requester
        cat = ops.torch.cat(served) if served else ops.to_dev(np.zeros(0, np.int64), _i64(ops))
        return x.a2a(cat, recv, send)

    def get_dense_feature(self, nodes, fid, dim):
        ops, x = self.ops, self.xchg
        _f32_features("ShardedGraph.get_dense_feature", getattr(ops, "graph", None), getattr(self.feature_ops, "graph", None))
        ids = ops.to_dev(nodes, _i64(ops)).reshape(-1)
        rows = ids.numel()
        if self.feature_ops is not None:     # replicated feature table: no exchange
            return self.feature_ops.feature_local(ids, fid, dim).reshape(rows, dim)
        sorted_ids, src, counts = ops.bucket(ids, self.P, self.N, x.rank)
        send, recv = x.counts(counts)
        inbox = x.a2a(sorted_ids, send, recv)
        feats = ops.feature_local(inbox, fid, dim)
        back = x.a2a(feats, recv, send, dim)
        return ops.merge_rows(back, src, rows, dim)


class PeerShardedGraph:
    """The same ops as ShardedGraph with the exchange done by the kernels themselves over NVLink peer memory
    (csrc/p2p.cu): no NCCL call and no host sync per hop, so a whole step can be captured in a CUDA graph.
    torch.distributed is used once, at construction, to all_gather the cudaIpc handles."""

    def __init__(self, graph, rank, world, max_rows, max_count, max_feat_rows, max_dim, rng="minstd", seed=1,
                 num_partitions=None, group=None, engines=1, feature_graph=None):
        """max_rows / max_feat_rows count ALL batches of a batched call; engines = the largest nb used.
        feature_graph: a Graph on this rank's GPU that holds EVERY node's dense features (replicated feature table: 51 GB at
        the 50M-node / dim-256 headline config against 80 GB of HBM per H100).  When given, get_dense_feature and sage_mean are the
        single-GPU kernels on it and only the sampling hops cross NVLink; None = Euler's scheme (features live with their
        rows and are fetched / aggregated by the owners)."""
        import torch
        import torch.distributed as dist
        from . import _lib
        from .graph import Context
        self.torch, self.lib, self.check = torch, _lib.load(), _lib.check
        self.graph, self.rank, self.N = graph, rank, world
        self.P = num_partitions or world
        self.dev = torch.device("cuda", graph.device)
        self.ctx = Context(graph, rng, seed)
        if engines > 1:
            self.ctx.set_engines(engines)
        self.ctx.reserve(world * max_rows + 1024)
        self.feature_graph = feature_graph
        self.fctx = Context(feature_graph, rng, seed + 7) if feature_graph is not None else None
        self._h = C.c_void_p()
        handle = (C.c_char * 64)()
        self.check(self.lib.eu_sym_create(self.ctx._h, rank, world, max_rows, max_count, max_feat_rows, max_dim,
                                          C.byref(self._h), handle))
        handles = [None] * world
        dist.all_gather_object(handles, bytes(handle.raw), group=group)
        blob = b"".join(handles)
        self.check(self.lib.eu_sym_connect(self._h, blob))
        dist.barrier(group=group)
        ptrs = [C.c_void_p() for _ in range(5)]
        self.check(self.lib.eu_sym_outputs(self._h, *[C.byref(p) for p in ptrs]))
        mk = self._view
        n_out = max_rows * max_count
        self.o_eng = mk(ptrs[0].value, n_out, torch.int64)
        self.o_ids = mk(ptrs[1].value, n_out, torch.int64)
        self.o_w = mk(ptrs[2].value, n_out, torch.float32)
        self.o_t = mk(ptrs[3].value, n_out, torch.int32)
        self.o_rows = mk(ptrs[4].value, max_feat_rows * max_dim, torch.float32)

    def _view(self, ptr, n, dtype):
        """zero-copy tensor over library-owned device memory"""
        t = self.torch
        nbytes = max(n, 1) * t.empty(0, dtype=dtype).element_size()
        st = t._C._construct_storage_from_data_pointer(ptr, self.dev, nbytes)
        return t.empty(0, dtype=dtype, device=self.dev).set_(st, 0, (max(n, 1),))

    def _stream(self):
        self.ctx.set_stream(self.torch.cuda.current_stream(self.dev).cuda_stream)

    def error(self):
        """nonzero if a bounded wait of this exchange group timed out (or the ranks disagreed on a batch shape): the region is
        poisoned on EVERY rank -- results since then are invalid and the object must be closed.  Synchronises."""
        e = C.c_int(0)
        self.check(self.lib.eu_sym_error(self._h, C.byref(e)))
        return e.value

    def raise_on_error(self):
        if self.error():
            raise EulerErrorSharded("peer exchange poisoned: a rank did not answer within EU_SYM_TIMEOUT_S (default 30 s) "
                                    "or issued a different batch shape; results of this PeerShardedGraph are invalid")

    def hop(self, frontier, etypes, count, default_node=-1, packed=True, nb=1):
        """frontier: device i64 tensor, [nb * rows] (batch-major).  Returns (eng, ids, w, t) VIEWS into the symmetric
        outputs (overwritten by the next hop; eng is what the next hop consumes), each [nb * rows * count]."""
        self._stream()
        et = np.ascontiguousarray(etypes, dtype=np.int32)
        total = frontier.numel()
        assert total % nb == 0
        self.check(self.lib.eu_sym_sample_hop_batched(self._h, frontier.data_ptr(), int(nb), total // nb, et.ctypes.data, len(et),
                                                      int(count), default_node, self.P, int(packed)))
        n = total * int(count)
        return self.o_eng[:n], self.o_ids[:n], self.o_w[:n], self.o_t[:n]

    def sample_fanout_batched(self, nodes, edge_types, counts, default_node=-1, check=True):
        """nodes: [nb, B].  Batch g == sample_fanout of nodes[g] with every shard on its engine g.  Returns lists of
        [nb, B * prod(counts[:l])] tensors."""
        t = self.torch
        nodes = nodes if isinstance(nodes, t.Tensor) else t.as_tensor(np.asarray(nodes), dtype=t.int64)
        nodes = nodes.to(device=self.dev, dtype=t.int64).contiguous()
        nb = nodes.shape[0]
        frontier = nodes.reshape(-1)
        ids, ws, ts = [nodes], [], []
        for et, c in zip(edge_types, counts):
            eng, o_ids, o_w, o_t = self.hop(frontier, et, c, default_node, nb=nb)
            ids.append(o_ids.clone().reshape(nb, -1)); ws.append(o_w.clone().reshape(nb, -1)); ts.append(o_t.clone().reshape(nb, -1))
            frontier = eng.clone()
        if check:
            self.raise_on_error()
        return ids, ws, ts

    def sample_fanout(self, nodes, edge_types, counts, default_node=-1, check=True):
        """check=True synchronises and raises if the exchange was poisoned (pass False inside a CUDA-graph capture and call
        raise_on_error() at your own sync point)."""
        t = self.torch
        frontier = nodes if isinstance(nodes, t.Tensor) else t.as_tensor(np.asarray(nodes), dtype=t.int64, device=self.dev)
        frontier = frontier.to(device=self.dev, dtype=t.int64).reshape(-1).contiguous()
        ids, ws, ts = [frontier], [], []
        for et, c in zip(edge_types, counts):
            eng, o_ids, o_w, o_t = self.hop(frontier, et, c, default_node)
            ids.append(o_ids.clone()); ws.append(o_w.clone()); ts.append(o_t.clone())
            frontier = eng.clone()
        if check:
            self.raise_on_error()
        return ids, ws, ts

    def get_dense_feature(self, nodes, fid, dim, clone=True, out=None):
        t = self.torch
        _f32_features("PeerShardedGraph.get_dense_feature", self.graph, self.feature_graph)
        ids = nodes.to(device=self.dev, dtype=t.int64).reshape(-1).contiguous()
        if self.fctx is not None:      # replicated feature table: the single-GPU kernel, nothing crosses NVLink
            if out is None:
                out = t.empty(ids.numel(), dim, dtype=t.float32, device=self.dev)
            self.fctx.set_stream(t.cuda.current_stream(self.dev).cuda_stream)
            self.check(self.lib.eu_get_dense_feature(self.fctx._h, ids.data_ptr(), ids.numel(), int(fid), int(dim), out.data_ptr()))
            return out
        self._stream()
        self.check(self.lib.eu_sym_get_dense_feature(self._h, ids.data_ptr(), ids.numel(), int(fid), int(dim), self.P))
        out = self.o_rows[:ids.numel() * dim].reshape(ids.numel(), dim)
        return out.clone() if clone else out

    def sage_mean(self, nbr_ids, rows, count, dim, out=None):
        """fused sharded mean aggregation of a fixed-fanout block (owners sum their rows; eu_sym_sage_mean)"""
        t = self.torch
        _f32_features("PeerShardedGraph.sage_mean", self.graph, self.feature_graph)
        ids = nbr_ids.to(device=self.dev, dtype=t.int64).reshape(-1).contiguous()
        assert ids.numel() == rows * count
        if out is None:
            out = t.empty(rows, dim, dtype=t.float32, device=self.dev)
        if self.fctx is not None:      # replicated feature table: eu_sage_mean_aggregate, bit-identical to the single-GPU path
            self.fctx.set_stream(t.cuda.current_stream(self.dev).cuda_stream)
            self.check(self.lib.eu_sage_mean_aggregate(self.fctx._h, ids.data_ptr(), int(rows), int(count), int(dim), out.data_ptr()))
            return out
        self._stream()
        self.check(self.lib.eu_sym_sage_mean(self._h, ids.data_ptr(), int(rows), int(count), int(dim), self.P, out.data_ptr()))
        return out

    def close(self):
        """destroys the symmetric region; raises if the exchange had been poisoned (results before the close are invalid)"""
        if self._h:
            self.torch.cuda.synchronize()
            bad = self.error()
            self.lib.eu_sym_destroy(self._h)
            self._h = None
            if self.fctx is not None:
                self.fctx.close()
            if bad:
                raise EulerErrorSharded("peer exchange was poisoned (timeout or batch-shape mismatch) before close()")


class EulerErrorSharded(RuntimeError):
    pass


def _f32_features(what, *graphs):
    """The sharded feature paths read float32 feature tables held in HBM only: a bfloat16 or host-placed graph is refused on
    every rank alike, before any exchange or write."""
    from ._lib import EulerError
    for g in graphs:
        if g is not None and getattr(g, "feat_dtype", "float32") != "float32":
            raise EulerError("%s: the sharded feature paths read float32 feature tables only (this graph stores %s)"
                             % (what, g.feat_dtype))
        if g is not None and getattr(g, "feat_place", "device") != "device":
            raise EulerError("%s: the sharded feature paths read feature tables held in HBM only (this graph's is placed on "
                             "the %s)" % (what, g.feat_place))


def _i64(ops):
    return ops.torch.int64 if hasattr(ops, "torch") else np.int64
