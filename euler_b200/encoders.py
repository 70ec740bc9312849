"""SparseEmbedding (tf_euler/python/utils/layers.py:152-169), the embedding the sparse-feature encoders apply to uint64
feature slots (ShallowEncoder, encoders.py:151-160; SageEncoderNew, encoders.py:590-612), and ShallowEncoder
(encoders.py:32-171), the input layer of the node encoders: an id embedding, dense feature slots and sparse-feature
embeddings, concatenated or added.  And SageEncoder / ShuffleSageEncoder (encoders.py:411-541), GraphSAGE over
sample_fanout's sample tree with that input layer and the aggregators of aggregators.py.  And GCNEncoder / GenieEncoder
(encoders.py:174-291), the full-neighbourhood encoders over get_multi_hop_neighbor's hops and the aggregators of
sparse_aggregators.py.  And ScalableSageEncoder / ScalableGCNEncoder (encoders.py:294-408, 629-748), which train every layer
from one hop over per-layer embedding stores (_ScalableStores).  And LGCEncoder (encoders.py:872-922), LGCN's convolutions over
each node's row and the k largest values of every feature column among its sampled neighbours.

Callers size the table as the encoders do: SparseEmbedding(max_id + 1, dim) for values in [0, max_id] and
default = max_id + 1 for nodes without values, so the table has max_id + 2 rows and the default row is the last one.

Upstream quirk: ShallowEncoder's use_hash_embedding=True names layers.HashEmbedding / layers.HashSparseEmbedding
(encoders.py:108-119), which the reference tree does not define, so that option fails there; it raises here too.
"""
import functools

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, ops
from .ops import sparse_feature_embedding
from .unsupervised import Embedding, check_table_dtype


def _truncated_normal_(t, stddev):
    """tf.truncated_normal_initializer: normal draws, those beyond two standard deviations drawn again"""
    torch.nn.init.trunc_normal_(t, mean=0.0, std=stddev, a=-2 * stddev, b=2 * stddev)
    return t


class SparseEmbedding(torch.nn.Module):
    """layers.SparseEmbedding(max_id, dim, initializer=None, combiner='sum'): a table f32[max_id + 1, dim] initialised
    truncated-normal with stddev 0.0002 (layers.py:157-165).

    __call__(sparse) takes the (indices, values, dense_shape) triple ops.get_sparse_feature returns and restates
    tf.nn.embedding_lookup_sparse(table, sp_ids, None, combiner) in torch: the reference path, composed of a gather and a
    segment sum.  lookup(nodes, feature_name, default_value) goes from node ids to the same rows in one fused device op
    (ops.sparse_feature_embedding).  dtype=torch.bfloat16 initialises the table in f32 and rounds it once to nearest; such a
    table takes no autograd gradient (ShallowEncoder trains it through a proxy)."""

    def __init__(self, max_id, dim, combiner='sum', device=None, dtype=torch.float32):
        super().__init__()
        if combiner not in ('sum', 'mean', 'sqrtn'):
            raise ValueError("combiner must be 'sum', 'mean' or 'sqrtn'")
        self.combiner = combiner
        table = _truncated_normal_(torch.empty(max_id + 1, dim, device=device), 0.0002)
        if dtype == torch.float32:
            self.embeddings = torch.nn.Parameter(table)
        else:
            self.embeddings = torch.nn.Parameter(table.to(dtype), requires_grad=False)

    def forward(self, sparse):
        indices, values, dense_shape = sparse
        rows = indices[:, 0].long()
        n = int(dense_shape[0])
        emb = self.embeddings[values.long()]
        out = torch.zeros((n, emb.shape[1]), dtype=emb.dtype, device=emb.device).index_add(0, rows, emb)
        if self.combiner == 'sum':
            return out
        cnt = torch.zeros(n, dtype=emb.dtype, device=emb.device).index_add(0, rows, torch.ones_like(rows, dtype=emb.dtype))
        den = cnt if self.combiner == 'mean' else cnt.sqrt()
        return out / den.clamp(min=1)[:, None]

    def lookup(self, nodes, feature_name, default_value):
        return sparse_feature_embedding(nodes, feature_name, self.embeddings, default_value, self.combiner)


class Dense(torch.nn.Module):
    """layers.Dense(dim, activation=None, use_bias) (utils/layers.py:70-116) over inputs of in_dim columns: a kernel
    [in_dim, dim] initialised by tf.uniform_unit_scaling_initializer(factor=0.36), uniform in +-0.36 sqrt(3 / in_dim), and
    with use_bias a bias [dim] initialised to 0.0002; activation(x @ kernel + bias).  use_bias defaults to False here (the
    encoders' use); upstream's default is True, which the pool aggregators rely on and pass explicitly."""

    def __init__(self, in_dim, dim, activation=None, use_bias=False, device=None):
        super().__init__()
        bound = 0.36 * (3.0 / max(in_dim, 1)) ** 0.5
        self.kernel = torch.nn.Parameter(torch.empty(in_dim, dim, device=device).uniform_(-bound, bound))
        self.bias = torch.nn.Parameter(torch.full((dim,), 0.0002, device=device)) if use_bias else None
        self.activation = activation

    def forward(self, x):
        out = x @ self.kernel
        if self.bias is not None:
            out = out + self.bias
        return self.activation(out) if self.activation else out


class ShallowEncoder(torch.nn.Module):
    """encoders.ShallowEncoder (tf_euler/python/utils/encoders.py:32-171), with upstream's constructor arguments and
    ValueErrors.  Each node's row is built from
        max_id != -1               an id embedding: unsupervised.Embedding(max_id + 1, dim), a table of max_id + 2 rows
        feature_idx != -1          the dense slots feature_idx with widths feature_dim (get_dense_feature)
        sparse_feature_idx != -1   one SparseEmbedding(max_id_s + 1, dim) per uint64 slot, default value max_id_s + 1
    combined by 'concat' (then the Dense layer when dim is given) or 'add' (every table dim columns; the dense features go
    through the Dense layer first).  Dense is layers.Dense(dim, use_bias=False) (Dense above), built when dim is given.
    output_dim follows upstream; __call__(inputs) takes node ids of any shape and returns inputs.shape + (output_dim,).

    fused=True (the default) builds the row in one device op, ops.shallow_encode: 'concat' writes [id | dense | sparse]
    exactly as the composition does; 'add' computes (id + sparse_0 + ..) + Dense(features), which differs from upstream's
    add_n order id + Dense(features) + sparse_0 + .. only in float rounding.  sparse_grad=True gives the tables coalesced
    sparse COO gradients (use an optimizer that takes them, e.g. torch.optim.SGD or SparseAdam).  fused=False runs the literal
    composition: Embedding, get_dense_feature, get_sparse_feature + SparseEmbedding.__call__, then cat or add_n.

    table_dtype=torch.bfloat16 (fused only) stores the id table and every SparseEmbedding table in bfloat16, initialised in
    f32 and rounded once to nearest: half the HBM, and the optimizer keeps its slots in bf16 too.  The rows are the f32
    op's on the widened tables.  A bf16 table takes no autograd gradient; each has a proxy (ops.table_proxy, not a
    parameter and not in the state_dict) that receives its f32 sparse gradient, and optimizers.minimize hands those to
    the optimizer in the same step as the dense parameters."""

    def __init__(self, dim=None, feature_idx='f1', feature_dim=0, max_id=-1, sparse_feature_idx=-1, sparse_feature_max_id=-1,
                 embedding_dim=16, use_hash_embedding=False, combiner='concat', fused=True, sparse_grad=False, device=None,
                 table_dtype=torch.float32):
        super().__init__()
        check_table_dtype(table_dtype, fused)
        if combiner not in ['add', 'concat']:
            raise ValueError('combiner must be \'add\' or \'concat\'.')
        if combiner == 'add' and dim is None:
            raise ValueError('add must be used with dim provided.')
        use_feature = feature_idx != -1
        use_id = max_id != -1
        use_sparse_feature = sparse_feature_idx != -1
        if not isinstance(feature_idx, list) and use_feature:
            feature_idx = [feature_idx]
        if isinstance(feature_dim, int) and use_feature:
            feature_dim = [feature_dim]
        if use_feature and len(feature_idx) != len(feature_dim):
            raise ValueError('feature_dim must be the same length as feature'
                             '_idx.idx:%s, dim:%s' % (str(feature_idx), str(feature_dim)))
        if isinstance(sparse_feature_idx, int) and use_sparse_feature:
            sparse_feature_idx = [sparse_feature_idx]
        if isinstance(sparse_feature_max_id, int) and use_sparse_feature:
            sparse_feature_max_id = [sparse_feature_max_id]
        if use_sparse_feature and len(sparse_feature_idx) != len(sparse_feature_max_id):
            raise ValueError('sparse_feature_idx must be the same length as'
                             'sparse_feature_max_id.')
        embedding_num = (1 if use_id else 0) + (len(sparse_feature_idx) if use_sparse_feature else 0)
        if combiner == 'add':
            embedding_dim = dim
        if isinstance(embedding_dim, int) and embedding_num:
            embedding_dim = [embedding_dim] * embedding_num
        if embedding_num and len(embedding_dim) != embedding_num:
            raise ValueError('length of embedding_num must be int(use_id) + '
                             'len(sparse_feature_idx)')
        if isinstance(use_hash_embedding, bool) and embedding_num:
            use_hash_embedding = [use_hash_embedding] * embedding_num
        if embedding_num and len(use_hash_embedding) != embedding_num:
            raise ValueError('length of use_hash_embedding must be int(use_id)'
                             ' + len(sparse_feature_idx)')
        if embedding_num and any(use_hash_embedding):
            raise NotImplementedError('use_hash_embedding: layers.HashEmbedding / HashSparseEmbedding are not defined upstream')

        self.dim = dim
        self.use_id = use_id
        self.use_feature = use_feature
        self.use_sparse_feature = use_sparse_feature
        self.combiner = combiner
        self.feature_idx = feature_idx
        self.feature_dim = feature_dim
        self.sparse_feature_idx = sparse_feature_idx
        self.sparse_feature_max_id = sparse_feature_max_id
        self.embedding_dim = embedding_dim
        self.fused = fused
        self.sparse_grad = sparse_grad
        self.table_dtype = table_dtype
        self._proxies = {}   # table index (0: id, 1 + s: slot s) -> its proxy; plain attributes, not module state

        dims = list(embedding_dim) if embedding_num else []
        if use_id:
            self.embedding = Embedding(max_id + 1, dims.pop(0), device=device, dtype=table_dtype)
        if use_sparse_feature:
            self.sparse_embeddings = torch.nn.ModuleList(
                [SparseEmbedding(m + 1, d, device=device, dtype=table_dtype) for m, d in zip(sparse_feature_max_id, dims)])
        if dim:
            feat_w = sum(feature_dim) if use_feature else 0
            in_dim = feat_w if combiner == 'add' else feat_w + (sum(embedding_dim) if embedding_num else 0)
            self.dense = Dense(in_dim, dim, device=device)

    @property
    def output_dim(self):
        if self.dim is not None:
            return self.dim
        output_dim = 0
        if self.use_feature:
            output_dim += sum(self.feature_dim)
        if self.use_id or self.use_sparse_feature:
            output_dim += sum(self.embedding_dim)
        return output_dim

    def _default_values(self):
        return [m + 1 for m in self.sparse_feature_max_id]

    def forward(self, inputs):
        shape = tuple(inputs.shape)
        nodes = inputs.reshape(-1)
        out = self._fused(nodes) if self.fused else self._composed(nodes)
        return out.reshape(shape + (self.output_dim,))

    def _op_inputs(self):
        """(id_table, dense, sparse, proxies) as ops.shallow_encode takes them"""
        id_table = self.embedding.embeddings if self.use_id else None
        dense = list(zip(self.feature_idx, self.feature_dim)) if self.use_feature else []
        sparse = [(name, e.embeddings, dv, e.combiner) for name, e, dv in
                  zip(self.sparse_feature_idx, self.sparse_embeddings, self._default_values())] if self.use_sparse_feature else []
        return id_table, dense, sparse, self._proxy_list([id_table] + [s[1] for s in sparse])

    def _proxy_list(self, tables):
        """one proxy per table (None for an absent or f32 table), made on the table's device at first use"""
        out = []
        for t, table in enumerate(tables):
            q = None
            if table is not None and table.dtype == torch.bfloat16:
                q = self._proxies.get(t)
                if q is None or q.device != table.device or tuple(q.shape) != tuple(table.shape):
                    q = self._proxies[t] = ops.table_proxy(table)
            out.append(q)
        return out

    def table_proxies(self):
        """[(table, proxy)] of every bfloat16 table: what optimizers.minimize steps"""
        id_table, _, sparse, proxies = self._op_inputs()
        return [(t, q) for t, q in zip([id_table] + [s[1] for s in sparse], proxies) if q is not None]

    @property
    def poolable(self):
        """whether pooled() applies: the row is the fused op's 'concat' row itself, with no Dense layer after it"""
        return self.fused and self.combiner == 'concat' and not self.dim

    def pooled(self, nodes, count, pool):
        """the 'sum' or 'mean' of this encoder's rows over consecutive segments of `count` nodes, f32[nodes.numel() / count,
        output_dim], in one device op that never writes the rows (ops.shallow_encode_pool); needs poolable"""
        id_table, dense, sparse, proxies = self._op_inputs()
        return ops.shallow_encode_pool(nodes, count, id_table, dense, sparse, pool, self.sparse_grad, proxies)

    def _fused(self, nodes):
        id_table, dense, sparse, proxies = self._op_inputs()
        if self.combiner == 'concat':
            emb = ops.shallow_encode(nodes, id_table, dense, sparse, 'concat', self.sparse_grad, proxies)
            return self.dense(emb) if self.dim else emb
        emb, feats = ops.shallow_encode(nodes, id_table, dense, sparse, 'add', self.sparse_grad, proxies)
        if feats is None:
            return emb
        feats = self.dense(feats)
        return feats if id_table is None and not sparse else emb + feats

    def _composed(self, nodes):
        embeddings = []
        if self.use_id:
            embeddings.append(F.embedding(nodes, self.embedding.embeddings, sparse=self.sparse_grad))
        if self.use_feature:
            features = torch.cat(ops.get_dense_feature(nodes, self.feature_idx, self.feature_dim), -1)
            if self.combiner == 'add':
                features = self.dense(features)
            embeddings.append(features)
        if self.use_sparse_feature:
            sparse_features = ops.get_sparse_feature(nodes, self.sparse_feature_idx, default_values=self._default_values())
            embeddings.extend([e(sp) for e, sp in zip(self.sparse_embeddings, sparse_features)])
        if self.combiner == 'add':
            return functools.reduce(torch.add, embeddings)
        embedding = torch.cat(embeddings, -1)
        return self.dense(embedding) if self.dim else embedding


class SageEncoder(torch.nn.Module):
    """encoders.SageEncoder (tf_euler/python/utils/encoders.py:411-493): GraphSAGE over the sample tree of
    sample_fanout(inputs, metapath, fanouts, default_node=max_id + 1), with upstream's constructor arguments, ValueErrors and
    dims.  The node encoder is ShallowEncoder(feature_idx, feature_dim, max_id if use_id else -1, sparse_feature_idx, ..)
    with 'concat' and no dim (or shared_node_encoder), the aggregators aggregators.get(aggregator)(dim, relu on all but the last
    layer, concat=concat) (or shared_aggregators).  use_feature is deprecated upstream and has no effect; use_residual is
    ignored, as upstream's SageEncoder ignores it.  __call__(inputs) returns inputs.shape + (dim,).

    fused=True (the default): the deepest hop, which only ever reaches layer 0's aggregator as the neighbours of hop L - 1, is
    not encoded row by row when that aggregator is linear in its neighbours ('mean', 'gcn': it has forward_pooled) and the
    node encoder can pool (ShallowEncoder.poolable, and a fanout within the op's bound): the aggregator then receives
    ops.shallow_encode_pool's [n, W] rows and the [n * fanout, W] matrix is never written, forward or backward.  Every other
    combination takes the composition.  fused=False is the literal composition everywhere: the node encoder's composed path
    per hop, then upstream's layer / hop loop.  sparse_grad=True gives the node encoder's tables sparse COO gradients.
    table_dtype is the node encoder's (ShallowEncoder; bfloat16 trains with optimizers.minimize)."""

    @staticmethod
    def create_aggregators(in_dim, dim, num_layers, aggregator, **kwargs):
        """upstream's create_aggregators, with the input width of layer 0 (every later layer reads dim columns)"""
        from . import aggregators
        aggregator_class = aggregators.get(aggregator)
        return torch.nn.ModuleList([
            aggregator_class(in_dim if layer == 0 else dim, dim, activation=torch.relu if layer < num_layers - 1 else None, **kwargs)
            for layer in range(num_layers)])

    def __init__(self, metapath, fanouts, dim, aggregator='mean', concat=False, shared_aggregators=None, feature_idx=-1,
                 feature_dim=0, max_id=-1, use_feature=None, use_id=None, sparse_feature_idx=-1, sparse_feature_max_id=-1,
                 embedding_dim=16, use_hash_embedding=False, use_residual=False, shared_node_encoder=None, fused=True,
                 sparse_grad=False, device=None, table_dtype=torch.float32):
        super().__init__()
        if len(metapath) != len(fanouts):
            raise ValueError('Len of metapath must be the same as fanouts.')
        self.metapath = metapath
        self.fanouts = list(fanouts)
        self.num_layers = len(metapath)
        self.concat = concat
        self.fused = fused
        if shared_node_encoder:
            self._node_encoder = shared_node_encoder
        else:
            self._node_encoder = ShallowEncoder(
                feature_idx=feature_idx, feature_dim=feature_dim, max_id=max_id if use_id else -1,
                sparse_feature_idx=sparse_feature_idx, sparse_feature_max_id=sparse_feature_max_id, embedding_dim=embedding_dim,
                use_hash_embedding=use_hash_embedding, fused=fused, sparse_grad=sparse_grad, device=device,
                table_dtype=table_dtype)
        self.dims = [self._node_encoder.output_dim] + [dim] * self.num_layers
        if shared_aggregators is not None:
            self.aggregators = shared_aggregators
        else:
            self.aggregators = self.create_aggregators(self.dims[0], dim, self.num_layers, aggregator, concat=concat, device=device)
        self._max_id = max_id

    def node_encoder(self, inputs):
        return self._node_encoder(inputs)

    def _pools_deepest_hop(self):
        fanout = self.fanouts[-1]
        return (self.fused and hasattr(self.aggregators[0], 'forward_pooled') and getattr(self._node_encoder, 'poolable', False)
                and 1 <= fanout <= _lib.SHALLOW_POOL_MAX_COUNT)

    def sample(self, inputs):
        return ops.sample_fanout(inputs, self.metapath, self.fanouts, default_node=self._max_id + 1)[0]

    def agg(self, inputs, samples):
        """upstream's layer / hop loop over the ids of the sample tree (samples[hop], flat)"""
        L = self.num_layers
        pooled = None
        if self._pools_deepest_hop():
            pooled = self._node_encoder.pooled(samples[L], self.fanouts[-1], self.aggregators[0].pooled_input)
        hidden = [self.node_encoder(sample) for sample in (samples[:L] if pooled is not None else samples)]
        for layer in range(L):
            aggregator = self.aggregators[layer]
            next_hidden = []
            for hop in range(L - layer):
                if layer == 0 and hop == L - 1 and pooled is not None:
                    h = aggregator.forward_pooled(hidden[hop], pooled, self.fanouts[hop])
                else:
                    h = aggregator((hidden[hop], hidden[hop + 1].reshape(-1, self.fanouts[hop], self.dims[layer])))
                next_hidden.append(h)
            hidden = next_hidden
        return hidden[0].reshape(tuple(inputs.shape) + (self.dims[-1],))

    def forward(self, inputs):
        return self.agg(inputs, self.sample(inputs))


class ShuffleSageEncoder(SageEncoder):
    """encoders.ShuffleSageEncoder (encoders.py:496-541), DGI's encoder: returns [h, h_neg], h_neg aggregated over the same
    sample tree with its rows shuffled.  Upstream's shuffle_tensors lays the encoded rows out as [batch, tree position, dim]
    (the 1 + f1 + f1 f2 + .. positions of each seed's tree), permutes the positions by one permutation for the whole batch,
    flattens and splits by the hops' sizes.  The node encoder is row-wise, so that equals encoding the sample ids moved the
    same way (shuffle_samples), which keeps the deepest hop of the negative pass on the pooled op.  forward takes the
    torch.Generator of the permutation."""

    def shuffle_samples(self, samples, generator=None):
        batch = samples[0].numel()
        tree = torch.cat([s.reshape(batch, -1) for s in samples], 1)
        perm = torch.randperm(tree.shape[1], generator=generator).to(tree.device)
        return list(torch.split(tree[:, perm].reshape(-1), [s.numel() for s in samples]))

    def forward(self, inputs, generator=None):
        samples = self.sample(inputs)
        return [self.agg(inputs, samples), self.agg(inputs, self.shuffle_samples(samples, generator))]


class GCNEncoder(torch.nn.Module):
    """encoders.GCNEncoder (tf_euler/python/utils/encoders.py:174-233): the full-neighbourhood encoder over
    get_multi_hop_neighbor(inputs, metapath), with upstream's constructor arguments and head_num handling (an int, or a list
    of one per layer).  The node encoder is ShallowEncoder(dim if use_residual else None, .., combiner='add' if use_residual
    else 'concat'); layer l is sparse_aggregators.get(aggregator)(width of its inputs, dim, relu on all but the last layer,
    head_num=head_num[l]).  Layer 0 reads the node encoder's output_dim columns, every later layer the previous layer's
    output width (head_num * (dim // head_num) for 'attention'); self.dims lists them.  With use_residual each hop's output
    is hidden[hop] + aggregator(..).  __call__(inputs) returns inputs.shape + (width of the last layer,).

    Difference from upstream: under use_residual an aggregator whose width is not dim ('attention' with dim not a multiple of
    head_num) fails upstream when the residual is added, at run time; here it raises ValueError at construction.

    fused=True (the default) gives the aggregators their device paths (sparse_aggregators: ops.adjacency_mean for 'gcn' /
    'mean', ops.gat_attention_aggregate for 'attention') and the node encoder its fused op; fused=False is the literal
    composition everywhere.  sparse_grad=True gives the node encoder's tables sparse COO gradients.  table_dtype is the node
    encoder's (ShallowEncoder; bfloat16 trains with optimizers.minimize, and infer reads the bf16 tables as they are)."""

    def __init__(self, metapath, dim, aggregator='mean', feature_idx=-1, feature_dim=0, max_id=-1, use_id=False,
                 sparse_feature_idx=-1, sparse_feature_max_id=-1, embedding_dim=16, use_hash_embedding=False,
                 use_residual=False, head_num=4, fused=True, sparse_grad=False, device=None, table_dtype=torch.float32):
        super().__init__()
        from . import sparse_aggregators
        self.metapath = metapath
        self.num_layers = len(metapath)
        if isinstance(head_num, int):
            self.head_num = [head_num] * self.num_layers
        elif isinstance(head_num, list):
            assert len(head_num) == self.num_layers
            self.head_num = head_num
        else:
            raise ValueError('head_num error: expect int or'
                             ' list, got {}'.format(str(head_num)))
        self.use_residual = use_residual
        self._node_encoder = ShallowEncoder(
            dim=dim if use_residual else None, feature_idx=feature_idx, feature_dim=feature_dim,
            max_id=max_id if use_id else -1, sparse_feature_idx=sparse_feature_idx, sparse_feature_max_id=sparse_feature_max_id,
            embedding_dim=embedding_dim, use_hash_embedding=use_hash_embedding, combiner='add' if use_residual else 'concat',
            fused=fused, sparse_grad=sparse_grad, device=device, table_dtype=table_dtype)
        aggregator_class = sparse_aggregators.get(aggregator)
        self.dims = [self._node_encoder.output_dim]
        aggs = []
        for layer in range(self.num_layers):
            activation = torch.relu if layer < self.num_layers - 1 else None
            aggs.append(aggregator_class(self.dims[-1], dim, activation=activation, head_num=self.head_num[layer], fused=fused,
                                         device=device))
            self.dims.append(aggs[-1].output_dim)
        if use_residual and any(d != dim for d in self.dims[1:]):
            raise ValueError('use_residual needs every aggregator to be dim = %d wide, got widths %s' % (dim, self.dims[1:]))
        self.aggregators = torch.nn.ModuleList(aggs)

    def node_encoder(self, inputs):
        return self._node_encoder(inputs)

    def _layers(self, hidden, adjs, each_layer=None):
        """upstream's layer / hop loop; each_layer(layer, hidden[0]) after every layer"""
        for layer in range(self.num_layers):
            aggregator = self.aggregators[layer]
            next_hidden = []
            for hop in range(self.num_layers - layer):
                h = aggregator((hidden[hop], hidden[hop + 1], adjs[hop]))
                next_hidden.append(hidden[hop] + h if self.use_residual else h)
            hidden = next_hidden
            if each_layer:
                each_layer(layer, hidden[0])
        return hidden[0]

    def forward(self, inputs):
        nodes, adjs = ops.get_multi_hop_neighbor(inputs, self.metapath)
        out = self._layers([self.node_encoder(node) for node in nodes], adjs)
        return out.reshape(tuple(inputs.shape) + (self.dims[-1],))

    @torch.no_grad()
    def infer(self, ids=None, chunk_rows=1 << 20):
        """forward(ids) for many ids at once, computed layer by layer over the whole graph: f32[len(ids), dims[-1]], or
        every node in engine-row order (ops.graph_node_ids()) when ids is None.  The encoder draws nothing, so a node's
        layer-l value depends only on its neighbours' layer-(l-1) values and each layer is one pass over the graph's edges
        (ops.graph_adjacency) instead of one L-hop neighbourhood per batch.  Equals forward(ids) up to float rounding (the
        neighbour sums run in listing order, forward's in its column order; the GEMMs have other shapes).  An id that is
        not a node is encoded as forward encodes it: its node-encoder row, then every layer with no neighbours.

        The plan (infer_plan) keeps, per layer below the last, one table of every node for each distinct metapath window;
        the last layer runs at hop 0 on the requested rows only.  Peak memory is the node-encoder table, the tables of two
        consecutive layers, the metapath's adjacencies (12 B per listed entry) and one chunk of chunk_rows rows: f32 tables
        of 128 columns over 10M nodes are 5.1 GB each.  chunk_rows does not change the result's bits."""
        return self._infer(ids, chunk_rows)

    def _infer(self, ids, chunk_rows, each_layer=None):
        """infer's device inputs: the metapath's whole-graph adjacencies, the requested rows and the node-encoder table over
        every node and every absent id, all with one column numbering; then _infer_layers"""
        if chunk_rows < 1:
            raise ValueError('chunk_rows must be at least 1, got %d' % chunk_rows)
        L, n = self.num_layers, ops.get_graph().num_nodes
        hops = [_hop_key(t) for t in self.metapath]
        built = {}
        for h in (range(L) if L > 1 else []):
            if hops[h] not in built:
                built[hops[h]] = ops.graph_adjacency(self.metapath[h])
        if ids is None:
            if hops[0] not in built:
                built[hops[0]] = ops.graph_adjacency(self.metapath[0])
            final, absent_ids = built[hops[0]], []
        else:
            ids = ops._t(ids, torch.int64).reshape(-1)
            rows = ops.graph_node_rows(ids)
            final = ops.graph_adjacency(self.metapath[0], rows=rows)
            absent_ids = [ids[rows < 0]]
        # one numbering for every table: the n engine rows, then the distinct absent ids (none on most graphs)
        absent = torch.unique(torch.cat([a[3] for a in list(built.values()) + [final]] + absent_ids))
        N = n + absent.numel()

        def renumber(adj, n_rows):
            indptr, cols, _, extra = adj
            if extra.numel():
                mapped = n + torch.searchsorted(absent, extra)
                cols = torch.where(cols < n, cols, mapped[(cols - n).clamp(min=0)])
            if n_rows > indptr.numel() - 1:   # absent ids list nothing
                indptr = torch.cat([indptr, indptr[-1:].expand(n_rows - indptr.numel() + 1)])
            return indptr, cols

        adjs = {key: renumber(adj, N) for key, adj in built.items()}
        if ids is None:
            final, self_cols = adjs[hops[0]], None
            final = (final[0][:n + 1], final[1])
        else:
            final = renumber(final, 0)
            self_cols = torch.where(rows >= 0, rows, n + torch.searchsorted(absent, ids))
        node_ids = torch.cat([ops.graph_node_ids(), absent])
        table = None
        for a in range(0, N, chunk_rows):
            rows_a = self.node_encoder(node_ids[a:a + chunk_rows])
            if table is None:
                table = rows_a.new_empty((N, rows_a.shape[1]))
            table[a:a + rows_a.shape[0]] = rows_a
        return self._infer_layers(table, [adjs.get(k) for k in hops], final, self_cols, chunk_rows, each_layer)

    def _infer_layers(self, table, adjs, final, self_cols, chunk_rows, each_layer=None):
        """infer's layer / hop plan over the node-encoder table [N, dims[0]] (row r = column r of the adjacencies):
        adjs[h] = (indptr i64[N+1], cols) of metapath hop h over all N rows (used when L > 1), final = (indptr i64[B+1], cols)
        of hop 0 at the B requested rows, whose own rows are self_cols (None: rows 0 .. B-1).  each_layer(layer, rows) gets
        the requested rows' hop-0 values before layer 0 (layer = -1) and after every layer.  Plain torch around the
        aggregators: with fused=False it runs on CPU tensors and in float64."""
        L = self.num_layers
        hops = [_hop_key(t) for t in self.metapath]
        B = final[0].numel() - 1

        def at_requested(t):
            return t[:B] if self_cols is None else t[self_cols]

        tables = {(): table}   # metapath window -> the table of every row at the hops of that window
        if each_layer:
            each_layer(-1, at_requested(table))
        for layer, plan in enumerate(infer_plan(self.metapath)):
            tables = {win: self._infer_layer(layer, tables[win[:-1]], tables[win[1:]], adjs[h[0]], None, chunk_rows)
                      for win, h in plan.items()}
            if each_layer:
                each_layer(layer, at_requested(tables[tuple(hops[:layer + 1])]))
        out = self._infer_layer(L - 1, tables[tuple(hops[:L - 1])], tables[tuple(hops[1:])], final, self_cols, chunk_rows)
        if each_layer:
            each_layer(L - 1, out)
        return out

    def _infer_layer(self, layer, self_table, neigh_table, adj, self_cols, chunk_rows):
        """aggregator `layer` (and the residual) at every row of adj, chunk_rows rows at a time; row i's own row is
        self_table[self_cols[i]] (self_cols None: self_table[i])"""
        indptr, cols = adj
        R = indptr.numel() - 1
        starts = list(range(0, R, chunk_rows)) + [R]
        offs = indptr[torch.as_tensor(starts, device=indptr.device)].tolist()
        out = None
        for a, b, oa, ob in zip(starts[:-1], starts[1:], offs[:-1], offs[1:]):
            own = self_table[a:b] if self_cols is None else self_table[self_cols[a:b]]
            h = self.aggregators[layer]((own, neigh_table, (indptr[a:b + 1] - oa, cols[oa:ob])))
            h = own + h if self.use_residual else h
            if out is None:
                out = h.new_empty((R, h.shape[1]))
            out[a:b] = h
        return out if out is not None else self_table.new_empty((0, self.dims[layer + 1]))


def _hop_key(types):
    """one metapath hop's edge-type list as a hashable key (the order is kept: it is the listing order)"""
    return tuple((types.reshape(-1) if torch.is_tensor(types) else np.asarray(types).reshape(-1)).tolist())


def infer_plan(metapath):
    """The tables GCNEncoder.infer builds for a metapath of L hops: per layer l < L - 1, {window: hops}, one table per
    distinct window.  Layer l's table at hop h (h = 0 .. L-1-l) is built from layer l-1's tables at hops h and h + 1 over
    metapath[h] (layer -1's is the node-encoder table, window ()), so it depends on metapath[h .. h+l]: its window is those
    type lists, and hops whose windows are equal share one table.  The last layer runs at hop 0 only, at the requested
    rows, so it has no table here."""
    L = len(metapath)
    keys = [_hop_key(t) for t in metapath]
    plan = []
    for layer in range(L - 1):
        tables = {}
        for h in range(L - layer):
            tables.setdefault(tuple(keys[h:h + layer + 1]), []).append(h)
        plan.append(tables)
    return plan


class GenieEncoder(GCNEncoder):
    """encoders.GenieEncoder (encoders.py:236-291), GeniePath's encoder: GCNEncoder's layers ('attention' by default), then
    depth_fc[0] of the seeds' node-encoder rows and depth_fc[l + 1] of layer l's seed rows (depth_fc: Dense(dim) with a bias,
    upstream's layers.Dense default), run as a sequence of L + 1 steps through TF's LSTMCell(dim) (graph_pool.LSTMCell) from a
    zero state.  __call__(inputs) returns inputs.shape + (dim,).

    Upstream returns outputs[:, 0, :] (encoders.py:287), the LSTM's output at the FIRST step: the result depends on the seeds'
    own node-encoder rows only, and the aggregators, the later depth_fc layers and the later steps never reach it (they get
    no gradient).  This restates that exactly, for parity with the geniepath example; it computes every layer and step, as
    upstream does."""

    def __init__(self, metapath, dim, aggregator='attention', feature_idx=-1, feature_dim=0, max_id=-1, use_id=False,
                 sparse_feature_idx=-1, sparse_feature_max_id=-1, embedding_dim=16, use_hash_embedding=False,
                 use_residual=False, head_num=4, fused=True, sparse_grad=False, device=None, table_dtype=torch.float32):
        super().__init__(metapath, dim, aggregator, feature_idx, feature_dim, max_id, use_id, sparse_feature_idx,
                         sparse_feature_max_id, embedding_dim, use_hash_embedding, use_residual, head_num, fused=fused,
                         sparse_grad=sparse_grad, device=device, table_dtype=table_dtype)
        from .graph_pool import LSTMCell
        self.dim = dim
        self.depth_fc = torch.nn.ModuleList([Dense(d, dim, use_bias=True, device=device) for d in self.dims])
        self.lstm_cell = LSTMCell(dim, dim)
        if device is not None:
            self.lstm_cell.to(device)

    def forward(self, inputs):
        nodes, adjs = ops.get_multi_hop_neighbor(inputs, self.metapath)
        hidden = [self.node_encoder(node) for node in nodes]
        h_t = [self.depth_fc[0](hidden[0])]
        self._layers(hidden, adjs, lambda layer, h: h_t.append(self.depth_fc[layer + 1](h)))
        return self._steps(h_t).reshape(tuple(inputs.shape) + (self.dim,))

    def _steps(self, h_t):
        """the LSTM over the L + 1 depth_fc outputs from a zero state; upstream's output at the first step"""
        zero = h_t[0].new_zeros((h_t[0].shape[0], self.dim))
        state, outputs = (zero, zero), []
        for x in h_t:
            out, state = self.lstm_cell(x, state)
            outputs.append(out)
        return outputs[0]

    @torch.no_grad()
    def infer(self, ids=None, chunk_rows=1 << 20):
        """forward(ids) computed layer by layer over the whole graph, as GCNEncoder.infer: every layer's hop-0 rows at the
        requested ids through depth_fc, then the LSTM steps, returning the first step's output as forward does.
        f32[len(ids), dim], or every node in engine-row order when ids is None."""
        h_t = []
        self._infer(ids, chunk_rows, lambda layer, rows: h_t.append(self.depth_fc[layer + 1](rows)))
        return self._steps(h_t)


def _exchange_composed(store, grad_store, ids, rows):
    """ops.store_exchange as the literal composition (any dtype and device): the pre-clear gather, then index_put_ of the
    ids deduplicated in Python, keeping each id's last occurrence"""
    taken = grad_store[ids]
    last = {v: i for i, v in enumerate(ids.tolist())}
    keys = torch.as_tensor(list(last.keys()), dtype=torch.int64, device=store.device)
    store.index_put_((keys,), rows.detach()[torch.as_tensor(list(last.values()), dtype=torch.int64, device=store.device)])
    grad_store.index_put_((keys,), torch.zeros((), dtype=grad_store.dtype, device=grad_store.device))
    return taken


def _scalable_f32(table_dtype):
    """the scalable encoders train their node-encoder tables in f32 only (train_step steps them through .grad)"""
    if table_dtype != torch.float32:
        raise ValueError("the scalable encoders train float32 tables only, got table_dtype=%r" % (table_dtype,))


def _scalable_store_args(store_dtype, store_seed, fused):
    """the stores' dtype and stochastic-rounding seed, checked before anything is allocated: float32, or bfloat16 with the
    fused store ops (the literal composition would round every accumulation to nearest)"""
    if store_dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("store_dtype must be torch.float32 or torch.bfloat16, got %r" % (store_dtype,))
    if store_dtype == torch.bfloat16 and not fused:
        raise ValueError("store_dtype=torch.bfloat16 needs fused=True")
    if not isinstance(store_seed, (int, np.integer)) or not 0 <= int(store_seed) < 2 ** 64:
        raise ValueError("store_seed must be an integer in [0, 2^64), got %r" % (store_seed,))


class _ScalableStores(torch.nn.Module):
    """The per-layer stores of ScalableSageEncoder / ScalableGCNEncoder and the training step over them.

    One step (the order upstream leaves open, fixed here):
      1. forward(inputs, training=True) samples one hop, encodes the node rows and runs every layer; layer l >= 1 reads its
         neighbours' rows from stores[l - 1] as they were at the start of the step (a leaf tensor that requires grad).
      2. After the last layer, one exchange per store: stores[l][node] = node_embeddings[l] (detached, the last occurrence of
         a repeated node wins), taken_l = gradient_stores[l][node] as it was, then those rows zeroed; store_loss =
         sum over l of sum(node_embeddings[l] * taken_l).  Reading and clearing before the backward pass means that a node
         that is also a neighbour in this step keeps the gradient it receives in this step.
      3. train_step(loss, optimizer) adds d(loss + store_loss) / d(each layer's neighbour store rows) into gradient_stores
         (every id gets the fixed-order sum of its entries, added with one rounding), computes d loss / d params for
         `optimizer` and d store_loss / d params for store_optimizer from the same parameters, then steps both.

    store_dtype=torch.bfloat16 keeps every store and gradient store in bfloat16, half the bytes (fused only).  Each store is
    initialised in f32 exactly as an f32 one and rounded once to nearest; the gradient stores are zeros.  Reads widen
    exactly, so the forward is the f32 encoder's on the widened stores; the exchange rounds the written store rows to
    nearest, and each accumulation is written by stochastic rounding keyed by (store_seed, store_sr_step, layer, element).
    store_sr_step, an int64 device counter (a non-persistent buffer), advances once per train_step, after every layer.
    """

    def _init_stores(self, widths, max_id, store_learning_rate, store_init_maxval, generator, device,
                     store_dtype=torch.float32, store_seed=0):
        self.max_id = max_id
        self.store_learning_rate = store_learning_rate
        self.store_init_maxval = store_init_maxval
        self.store_dtype = store_dtype
        self.store_seed = int(store_seed)
        self._n_stores = len(widths)
        for l, w in enumerate(widths):
            # upstream's tables are LOCAL_VARIABLES, which its Saver does not checkpoint: non-persistent buffers
            store = torch.empty((max_id + 2, w), device=device).uniform_(0, store_init_maxval, generator=generator)
            self.register_buffer('store_%d' % l, store.to(store_dtype), persistent=False)
            del store   # a bf16 store's f32 initialisation is freed before its gradient store is made
            self.register_buffer('gradient_store_%d' % l, torch.zeros((max_id + 2, w), dtype=store_dtype, device=device),
                                 persistent=False)
        self.register_buffer('store_sr_step', torch.zeros((), dtype=torch.int64, device=device), persistent=False)
        self.store_optimizer = torch.optim.Adam(self.parameters(), lr=store_learning_rate)
        self.store_loss = None
        self._neigh_rows = []

    @property
    def stores(self):
        return [getattr(self, 'store_%d' % l) for l in range(self._n_stores)]

    @property
    def gradient_stores(self):
        return [getattr(self, 'gradient_store_%d' % l) for l in range(self._n_stores)]

    def _store_rows(self, l, neighbor, count=1, pool=None):
        """stores[l]'s rows of the neighbours as a leaf that requires grad: pooled over segments of `count` ('sum' or
        'mean', [n / count, w]) when pool is given, else gathered ([n, w]); recorded for train_step"""
        store = self.stores[l]
        with torch.no_grad():
            if not self.fused:
                rows = store[neighbor]
            elif pool is not None:
                rows = ops.shallow_encode_pool(neighbor, count, id_table=store, pool=pool)
            else:
                rows = ops.shallow_encode(neighbor, id_table=store)
        rows.requires_grad_()
        self._neigh_rows.append((l, neighbor, rows, count, pool))
        return rows

    def _exchange(self, node, node_embeddings):
        """step 2: the stores' exchanges in layer order, and store_loss"""
        losses = []
        for store, grad_store, h in zip(self.stores, self.gradient_stores, node_embeddings):
            if self.fused:
                taken = ops.store_exchange(store, grad_store, node, h.detach())
            else:
                with torch.no_grad():
                    taken = _exchange_composed(store, grad_store, node, h)
            losses.append((h * taken).sum())
        self.store_loss = functools.reduce(torch.add, losses) if losses else torch.zeros((), device=node.device)

    def train_step(self, loss, optimizer):
        """step 3 for the last forward(training=True): accumulate the neighbour store rows' gradients of loss + store_loss
        into gradient_stores, then step `optimizer` on d loss and store_optimizer (Adam, store_learning_rate) on
        d store_loss, both taken from the parameters before either step.  Sparse table gradients (sparse_grad=True) reach
        store_optimizer densified."""
        neigh, self._neigh_rows = self._neigh_rows, []
        params = [p for p in self.parameters() if p.requires_grad]
        store_grads = [None] * len(params)
        if self.store_loss.requires_grad:
            store_grads = torch.autograd.grad(self.store_loss, params, retain_graph=True, allow_unused=True)
        bf16 = self.store_dtype == torch.bfloat16
        if neigh:
            grads = torch.autograd.grad(loss + self.store_loss, [r for _, _, r, _, _ in neigh], retain_graph=True, allow_unused=True)
            for (l, neighbor, _, count, pool), g in zip(neigh, grads):
                if g is None:
                    continue
                if self.fused:
                    sr = dict(seed=self.store_seed, step=self.store_sr_step, tensor=l) if bf16 else {}
                    ops.store_accumulate(self.gradient_stores[l], neighbor, g, count, pool or 'sum', **sr)
                else:
                    self.gradient_stores[l].index_add_(0, neighbor, g)
        if bf16:
            self.store_sr_step.add_(1)
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        self.store_optimizer.zero_grad()
        for p, g in zip(params, store_grads):
            p.grad = None if g is None else (g.to_dense() if g.is_sparse else g)
        self.store_optimizer.step()


class ScalableSageEncoder(SageEncoder, _ScalableStores):
    """encoders.ScalableSageEncoder (tf_euler/python/utils/encoders.py:629-748): SageEncoder over metapath [edge_type] *
    num_layers and fanouts [fanout] * num_layers, trained from ONE hop.  With training=False, forward is SageEncoder's.
    With training=True it samples sample_fanout(inputs, [edge_type], [fanout], default_node=max_id + 1) once; layer 0
    aggregates the hop's node-encoder rows, layer l >= 1 the neighbours' rows of stores[l - 1] (f32[max_id + 2, dims[l]],
    initialised uniform(0, store_init_maxval) from `generator`; gradient_stores alike, zeros).  The step's order and
    train_step are _ScalableStores'; store_optimizer is torch.optim.Adam(self.parameters(), store_learning_rate).
    store_dtype=torch.bfloat16 (with store_seed) keeps the stores in bfloat16, by _ScalableStores' rules.

    fused=True (the default): layer 0 pools the hop through ShallowEncoder.pooled by SageEncoder's rule; layers >= 1 read
    the stores through ops.shallow_encode_pool(neighbor, fanout, id_table=store) when the aggregator has forward_pooled
    ('mean', 'gcn'), else ops.shallow_encode and a reshape ('meanpool', 'maxpool'); the exchanges are ops.store_exchange and
    the accumulations ops.store_accumulate, deterministic.  fused=False is the literal composition: store[ids],
    index_put_ with the ids deduplicated keep-last, index_add_.

    Differences from upstream:
      - upstream's __init__ passes shared_node_encoder, use_residual positionally into SageEncoder's use_residual,
        shared_node_encoder slots, so a shared node encoder is silently ignored there; here both keywords mean what they say.
      - the stores are initialised from `generator`, not TF's seeded random_uniform_initializer(seed=1) stream.
      - store_optimizer is torch's Adam, which applies epsilon to sqrt(v_hat), where TF's applies "epsilon hat" to sqrt(v).
    """

    def __init__(self, edge_type, fanout, num_layers, dim, aggregator='mean', concat=False, shared_aggregators=None,
                 feature_idx=-1, feature_dim=0, max_id=-1, use_feature=True, use_id=False, sparse_feature_idx=-1,
                 sparse_feature_max_id=-1, embedding_dim=16, use_hash_embedding=False, shared_node_encoder=None,
                 use_residual=False, store_learning_rate=0.001, store_init_maxval=0.05, fused=True, sparse_grad=False,
                 device=None, generator=None, table_dtype=torch.float32, store_dtype=torch.float32, store_seed=0):
        _scalable_f32(table_dtype)
        _scalable_store_args(store_dtype, store_seed, fused)
        super().__init__([edge_type] * num_layers, [fanout] * num_layers, dim, aggregator, concat, shared_aggregators,
                         feature_idx, feature_dim, max_id, use_feature, use_id, sparse_feature_idx, sparse_feature_max_id,
                         embedding_dim, use_hash_embedding, use_residual=use_residual,
                         shared_node_encoder=shared_node_encoder, fused=fused, sparse_grad=sparse_grad, device=device)
        self.edge_type = edge_type
        self.fanout = fanout
        self._init_stores(self.dims[1:-1], max_id, store_learning_rate, store_init_maxval, generator, device, store_dtype,
                          store_seed)

    def _pools_store(self, aggregator):
        return self.fused and hasattr(aggregator, 'forward_pooled') and 1 <= self.fanout <= _lib.SHALLOW_POOL_MAX_COUNT

    def forward(self, inputs, training=False):
        if not training:
            return super().forward(inputs)
        f, L = self.fanout, self.num_layers
        node, neighbor = ops.sample_fanout(inputs, [self.edge_type], [f], default_node=self.max_id + 1)[0]
        self._neigh_rows = []
        a = self.aggregators[0]
        if self._pools_deepest_hop():
            h = a.forward_pooled(self.node_encoder(node), self._node_encoder.pooled(neighbor, f, a.pooled_input), f)
        else:
            h = a((self.node_encoder(node), self.node_encoder(neighbor).reshape(-1, f, self.dims[0])))
        node_embeddings = [h]
        for layer in range(1, L):
            a = self.aggregators[layer]
            if self._pools_store(a):
                h = a.forward_pooled(h, self._store_rows(layer - 1, neighbor, f, a.pooled_input), f)
            else:
                h = a((h, self._store_rows(layer - 1, neighbor).reshape(-1, f, self.dims[layer])))
            node_embeddings.append(h)
        self._exchange(node, node_embeddings[:-1])
        return h.reshape(tuple(inputs.shape) + (self.dims[-1],))


class ScalableGCNEncoder(GCNEncoder, _ScalableStores):
    """encoders.ScalableGCNEncoder (tf_euler/python/utils/encoders.py:294-408): GCNEncoder over metapath [edge_type] *
    num_layers, trained from ONE full hop.  With training=False, forward is GCNEncoder's.  With training=True,
    (node, neighbor), (adj,) = get_multi_hop_neighbor(inputs, [edge_type]); layer 0 aggregates the node-encoder rows of both,
    layer l >= 1 the distinct neighbours' rows of stores[l - 1] (f32[max_id + 2, dim], uniform(0, store_init_maxval) from
    `generator`; gradient_stores alike, zeros), each layer's output plus its input under use_residual.  The step's order and
    train_step are _ScalableStores'.  fused=True reads the stores through ops.shallow_encode and updates them through
    ops.store_exchange / ops.store_accumulate, the aggregators taking their own fused paths; fused=False is the literal
    composition (store[ids], index_put_ keep-last, index_add_).  store_dtype=torch.bfloat16 (with store_seed) keeps the
    stores in bfloat16, by _ScalableStores' rules.

    Differences from upstream:
      - an aggregator whose output is stored must be dim wide, the stores' width; 'attention' with dim % head_num != 0 is
        not, and fails upstream at the first store write: here the constructor raises ValueError.
      - store initialisation and Adam's epsilon as ScalableSageEncoder's.
    """

    def __init__(self, edge_type, num_layers, dim, aggregator='mean', feature_idx=-1, feature_dim=0, max_id=-1, use_id=False,
                 sparse_feature_idx=-1, sparse_feature_max_id=-1, embedding_dim=16, use_hash_embedding=False,
                 use_residual=False, store_learning_rate=0.001, store_init_maxval=0.05, head_num=4, fused=True,
                 sparse_grad=False, device=None, generator=None, table_dtype=torch.float32, store_dtype=torch.float32,
                 store_seed=0):
        _scalable_f32(table_dtype)
        _scalable_store_args(store_dtype, store_seed, fused)
        super().__init__([edge_type] * num_layers, dim, aggregator, feature_idx, feature_dim, max_id, use_id,
                         sparse_feature_idx, sparse_feature_max_id, embedding_dim, use_hash_embedding, use_residual,
                         head_num, fused=fused, sparse_grad=sparse_grad, device=device)
        if any(w != dim for w in self.dims[1:-1]):
            raise ValueError('the stores are dim = %d wide; the stored layers are %s wide' % (dim, self.dims[1:-1]))
        self.dim = dim
        self.edge_type = edge_type
        self.fused = fused
        self._init_stores([dim] * (num_layers - 1), max_id, store_learning_rate, store_init_maxval, generator, device,
                          store_dtype, store_seed)

    def forward(self, inputs, training=False):
        if not training:
            return super().forward(inputs)
        (node, neighbor), (adj,) = ops.get_multi_hop_neighbor(inputs, [self.edge_type])
        self._neigh_rows = []
        h, nb = self.node_encoder(node), self.node_encoder(neighbor)
        node_embeddings = []
        for layer in range(self.num_layers):
            out = self.aggregators[layer]((h, nb, adj))
            h = h + out if self.use_residual else out
            node_embeddings.append(h)
            if layer < self.num_layers - 1:
                nb = self._store_rows(layer, neighbor)
        self._exchange(node, node_embeddings[:-1])
        return h.reshape(tuple(inputs.shape) + (self.dims[-1],))


class LGCEncoder(torch.nn.Module):
    """encoders.LGCEncoder (tf_euler/python/utils/encoders.py:872-922), "Large-Scale Learnable Graph Convolutional Networks"
    (https://arxiv.org/pdf/1808.03965.pdf), with upstream's constructor arguments.  __call__(inputs) takes node ids of any
    shape, flattened to [B], and returns f32[B, out_dim]:
        1. neighbors = sample_neighbor(inputs, edge_type, nb_num), default_node -1
        2. x = [the node's feature row; for every column, the k largest of that column over the nb_num neighbours'
           rows, descending] -- f32[B, k + 1, feature_dim], slot feature_idx (an absent neighbour's row is zeros)
        3. two tf.layers.conv1d over the k + 1 rows (channels last upstream, transposed for torch.nn.Conv1d): kernel size
           k // 2 + 1, 'valid' padding, a bias, no activation; feature_dim -> hidden_dim -> out_dim, glorot-uniform kernels
           and zero biases (TF's defaults); being torch's Conv1d they follow torch.backends.cudnn.allow_tf32 (on by
           default, so TF32 products on an H100)
        4. output row 0
    fused=True (the default) builds x in one device op, ops.neighbor_top_k_feature, without the [B, nb_num, feature_dim]
    neighbour rows; fused=False is the literal composition: two get_dense_feature calls, then cat, transpose and torch.topk.
    The two give the same x, except where +0.0 and -0.0 tie: the op keeps the lower neighbour index first (tf.nn.top_k's
    rule), torch.topk leaves the order of equal values open.  No gradient flows into x (graph data, as upstream).

    Upstream quirks kept: for odd k the two valid convolutions read only rows 0 .. 2 (k // 2) of x, so the k-th largest
    value never reaches the output (it is still selected); upstream's unused concat of the node and all neighbour rows
    (`nbs`) is dropped.  feature_idx=-1, upstream's default, would ask get_dense_feature for slot -1, and a k outside
    [1, nb_num] fails in tf.nn.top_k at run time: both raise ValueError at construction here."""

    def __init__(self, edge_type=[0], feature_idx=-1, feature_dim=0, k=3, hidden_dim=128, nb_num=10, out_dim=64, fused=True,
                 device=None):
        super().__init__()
        if feature_idx == -1:
            raise ValueError('LGCEncoder needs a dense feature slot: feature_idx is -1')
        if not 1 <= k <= nb_num:
            raise ValueError('k must lie in [1, nb_num = %d], got %d' % (nb_num, k))
        self.edge_type = edge_type
        self.feature_idx = feature_idx
        self.feature_dim = feature_dim
        self.k = k
        self.hidden_dim = hidden_dim
        self.out_dim = out_dim
        self.nb_num = nb_num
        self.fused = fused
        width = k // 2 + 1
        self.conv1 = torch.nn.Conv1d(feature_dim, hidden_dim, width, device=device)
        self.conv2 = torch.nn.Conv1d(hidden_dim, out_dim, width, device=device)
        for conv in (self.conv1, self.conv2):
            torch.nn.init.xavier_uniform_(conv.weight)    # TF's glorot: fans width * in and width * out, as torch counts them
            torch.nn.init.zeros_(conv.bias)

    def top_k_rows(self, nodes, neighbors):
        """x of step 2, f32[B, k + 1, feature_dim], from the flat node ids and their neighbours i64[B, nb_num]"""
        if self.fused:
            return ops.neighbor_top_k_feature(nodes, neighbors, self.feature_idx, self.feature_dim, self.k)
        node_feats, = ops.get_dense_feature(nodes, [self.feature_idx], [self.feature_dim])
        neighbor_feats, = ops.get_dense_feature(neighbors.reshape(-1), [self.feature_idx], [self.feature_dim])
        neighbor_feats = neighbor_feats.reshape(-1, self.nb_num, self.feature_dim)
        topk = torch.topk(neighbor_feats.transpose(1, 2), self.k)[0].transpose(1, 2)
        return torch.cat([node_feats.reshape(-1, 1, self.feature_dim), topk], 1)

    def forward(self, inputs):
        nodes = inputs.reshape(-1)
        neighbors = ops.sample_neighbor(nodes, self.edge_type, self.nb_num)[0]
        x = self.top_k_rows(nodes, neighbors)
        out = self.conv2(self.conv1(x.transpose(1, 2)))
        return out[:, :, 0]
