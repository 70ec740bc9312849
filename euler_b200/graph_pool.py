"""tf_euler's graph readouts (tf_euler/python/graph_pool/) over the euler_b200 mp ops, in torch.

  Pooling        base_pool.py       scatter_(aggr, inputs, index, size), aggr in 'add' | 'mean' | 'max'
  AttentionPool  attention_pool.py  gate = gate_nn(inputs) -> scatter_softmax -> gate * inputs -> scatter_(aggr)
  Set2SetPool    set2set_pool.py    processing_steps of: an LSTM step (TF's MultiRNNCell of LSTMCell) on q*, e = <x_n, q[g(n)]>,
                                    scatter_softmax, r = scatter_(aggr, a * x), q* = [q, r]

AttentionPool with aggr='add' and Set2SetPool's readout with aggr='add' run the fused device op
ops.graph_attention_readout (softmax and weighted sum in one pass, alpha [N] saved for the backward pass); any other aggr
composes the mp ops literally.  The dense layers (the gate, the LSTM kernels) are GEMMs and stay with torch.
"""
import torch

from . import ops


def _size(index, size):
    return int(index.max().item()) + 1 if size is None else int(size)


class Pooling(object):
    """base_pool.Pooling: out[b] = scatter_(aggr) of the rows of graph b"""

    def __init__(self, aggr='add'):
        assert aggr in ['add', 'mean', 'max']
        self.aggr = aggr

    def __call__(self, inputs, index, size=None):
        return ops.scatter_(self.aggr, inputs, index, _size(index, size))


def _glorot_uniform(fan_in, fan_out, device=None):
    """tf.glorot_uniform_initializer, the default kernel initializer of tf.layers.Dense and LSTMCell"""
    bound = (6.0 / (fan_in + fan_out)) ** 0.5
    return torch.empty(fan_in, fan_out, device=device).uniform_(-bound, bound)


class Dense(torch.nn.Module):
    """tf.layers.Dense(units, use_bias=False): a kernel [in, units] initialised glorot-uniform, created on the first call
    from the input's width and device"""

    def __init__(self, units):
        super(Dense, self).__init__()
        self.units = units
        self.register_parameter("kernel", None)

    def forward(self, x):
        if self.kernel is None:
            self.kernel = torch.nn.Parameter(_glorot_uniform(x.shape[1], self.units, device=x.device))
        return x @ self.kernel


class AttentionPool(Pooling):
    """attention_pool.AttentionPool.  gate_nn defaults to tf.layers.Dense(1, use_bias=False) (Dense above); nn, when given,
    maps the rows before they are summed."""

    def __init__(self, gate_nn=None, nn=None, aggr='add'):
        super(AttentionPool, self).__init__(aggr=aggr)
        self.gate_nn = Dense(1) if gate_nn is None else gate_nn
        self.nn = nn

    def __call__(self, inputs, index, size=None):
        size = _size(index, size)
        gate = self.gate_nn(inputs)
        inputs = self.nn(inputs) if self.nn is not None else inputs
        if self.aggr == 'add':
            return ops.graph_attention_readout(inputs, index, size, logits=gate)
        gate = ops.scatter_softmax(gate, index, size)
        return ops.scatter_(self.aggr, gate * inputs, index, size)


class LSTMCell(torch.nn.Module):
    """TF 1.x LSTMCell without peepholes or projection: one kernel [in + units, 4 * units] over concat([input, h]) plus a
    bias, gates split in the order i, j, f, o; c' = sigmoid(f + forget_bias) * c + sigmoid(i) * tanh(j), h' = sigmoid(o) *
    tanh(c') with forget_bias = 1.0.  (torch.nn.LSTM orders its gates i, f, g, o and has no forget bias.)"""

    def __init__(self, input_size, units, forget_bias=1.0):
        super(LSTMCell, self).__init__()
        self.units, self.forget_bias = units, forget_bias
        self.kernel = torch.nn.Parameter(_glorot_uniform(input_size + units, 4 * units))
        self.bias = torch.nn.Parameter(torch.zeros(4 * units))

    def forward(self, x, state):
        c, h = state
        z = torch.cat([x, h], dim=1) @ self.kernel + self.bias
        i, j, f, o = torch.split(z, self.units, dim=1)
        c = torch.sigmoid(f + self.forget_bias) * c + torch.sigmoid(i) * torch.tanh(j)
        h = torch.sigmoid(o) * torch.tanh(c)
        return h, (c, h)


class MultiRNNCell(torch.nn.Module):
    """TF's MultiRNNCell: the cells in order, each fed the previous one's output; the state is one (c, h) per cell"""

    def __init__(self, cells):
        super(MultiRNNCell, self).__init__()
        self.cells = torch.nn.ModuleList(cells)

    def zero_state(self, batch, device):
        return [(torch.zeros(batch, cl.units, device=device), torch.zeros(batch, cl.units, device=device)) for cl in self.cells]

    def forward(self, x, states):
        out = []
        for cell, st in zip(self.cells, states):
            x, st = cell(x, st)
            out.append(st)
        return x, out


class Set2SetPool(Pooling):
    """set2set_pool.Set2SetPool(dim, processing_steps, num_layers): q* starts at zeros [size, 2 dim]; each step runs the
    LSTM (num_layers LSTMCells of dim units) on q*, reads r = sum of softmax(<x_n, q[g(n)]>) * x_n per graph and sets
    q* = [q, r].  Returns q* [size, 2 dim]."""

    def __init__(self, dim, processing_steps, num_layers, aggr='add'):
        super(Set2SetPool, self).__init__(aggr=aggr)
        self.dim = dim
        self.processing_steps = processing_steps
        self.num_layers = num_layers
        self.lstm = MultiRNNCell([LSTMCell(2 * dim if k == 0 else dim, dim) for k in range(num_layers)])

    def __call__(self, inputs, index, size=None):
        size = _size(index, size)
        dev = inputs.device
        self.lstm.to(dev)
        cell_in = torch.zeros(size, self.dim * 2, dtype=torch.float32, device=dev)
        state = self.lstm.zero_state(size, dev)
        for _ in range(self.processing_steps):
            q, state = self.lstm(cell_in, state)
            if self.aggr == 'add':
                r = ops.graph_attention_readout(inputs, index, size, q=q)
            else:
                e = (inputs * ops.gather(q, index)).sum(-1, keepdim=True)
                a = ops.scatter_softmax(e, index, size)
                r = ops.scatter_(self.aggr, a * inputs, index, size)
            cell_in = torch.cat([q, r], dim=-1)
        return cell_in
