"""GraphSAGE's dense aggregators (tf_euler/python/utils/aggregators.py) in torch, with upstream's constructor arguments and
errors: GCNAggregator, MeanAggregator, MeanPoolAggregator, MaxPoolAggregator and get(name).

Each takes (self_embedding [R, Din], neigh_embedding [R, f, Din]) and returns [R, dim].  The self / neigh layers are
layers.Dense(dim, activation, use_bias=False); the pool aggregators first map every neighbour row through
layers.Dense(dim, relu) with a bias, where dim is the constructor's (not halved by concat=True), as upstream.

MeanAggregator and GCNAggregator are linear in the neighbours before any weight, so they also take the neighbours already
pooled over f (ops.shallow_encode_pool writes exactly that for the deepest hop of a fanout): forward_pooled(self, pooled, f)
with MeanAggregator.pooled_input = 'mean' and GCNAggregator.pooled_input = 'sum'.  The pool aggregators have no such entry: their Dense + relu
comes before the reduction.
"""
import torch

from .encoders import Dense


class GCNAggregator(torch.nn.Module):
    """aggregators.py:25-35: dense(mean over [self | neighbours]); in_dim is the width of the inputs"""
    pooled_input = 'sum'

    def __init__(self, in_dim, dim, activation=torch.relu, device=None, **kwargs):
        super().__init__()
        self.dense = Dense(in_dim, dim, activation=activation, device=device)

    def forward(self, inputs):
        self_embedding, neigh_embedding = inputs
        all_embedding = torch.cat([self_embedding.unsqueeze(1), neigh_embedding], 1)
        return self.dense(all_embedding.mean(1))

    def forward_pooled(self, self_embedding, neigh_sum, fanout):
        """the same from the neighbours' sum over the fanout axis: (self + sum) / (fanout + 1)"""
        return self.dense((self_embedding + neigh_sum) / (fanout + 1))


class BaseAggregator(torch.nn.Module):
    """aggregators.py:38-67: self_layer(self) + neigh_layer(aggregate(neighbours)), or their concatenation (dim halved)"""

    def __init__(self, in_dim, dim, activation=torch.relu, concat=False, device=None, agg_dim=None):
        super().__init__()
        if concat:
            if dim % 2:
                raise ValueError('dim must be divided exactly '
                                 'by 2 if concat is True.')
            dim //= 2
        self.concat = concat
        self.self_layer = Dense(in_dim, dim, activation=activation, device=device)
        self.neigh_layer = Dense(in_dim if agg_dim is None else agg_dim, dim, activation=activation, device=device)

    def forward(self, inputs):
        self_embedding, neigh_embedding = inputs
        return self._combine(self_embedding, self.aggregate(neigh_embedding))

    def _combine(self, self_embedding, agg_embedding):
        from_self = self.self_layer(self_embedding)
        from_neighs = self.neigh_layer(agg_embedding)
        return torch.cat([from_self, from_neighs], 1) if self.concat else from_self + from_neighs

    def aggregate(self, inputs):
        raise NotImplementedError()


class MeanAggregator(BaseAggregator):
    pooled_input = 'mean'

    def aggregate(self, inputs):
        return inputs.mean(1)

    def forward_pooled(self, self_embedding, neigh_mean, fanout):
        """the same from the neighbours' mean over the fanout axis"""
        return self._combine(self_embedding, neigh_mean)


class BasePoolAggregator(BaseAggregator):
    """aggregators.py:75-88: every neighbour row through Dense(dim, relu) (with bias; the constructor's dim, whatever concat
    is), then pool"""

    def __init__(self, in_dim, dim, *args, device=None, **kwargs):
        super().__init__(in_dim, dim, *args, device=device, agg_dim=dim, **kwargs)
        self.layers = torch.nn.ModuleList([Dense(in_dim, dim, activation=torch.relu, use_bias=True, device=device)])

    def aggregate(self, inputs):
        embedding = inputs
        for layer in self.layers:
            embedding = layer(embedding)
        return self.pool(embedding)

    def pool(self, inputs):
        raise NotImplementedError()


class MeanPoolAggregator(BasePoolAggregator):
    def pool(self, inputs):
        return inputs.mean(1)


class MaxPoolAggregator(BasePoolAggregator):
    def pool(self, inputs):
        return inputs.max(1).values


aggregators = {
    'gcn': GCNAggregator,
    'mean': MeanAggregator,
    'meanpool': MeanPoolAggregator,
    'maxpool': MaxPoolAggregator
}


def get(aggregator):
    return aggregators.get(aggregator)
