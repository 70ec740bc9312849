"""tf_euler's optimizers (tf_euler/python/utils/optimizers.py) with TF 1.x semantics, as torch optimizers.

    get('sgd')       MomentumOptimizer(lr, 0.0)
    get('momentum')  MomentumOptimizer(lr, 0.9)
    get('adagrad')   AdagradOptimizer(lr), accumulators starting at 0.1
    get('adam')      AdamOptimizer(lr), beta1 0.9, beta2 0.999, epsilon 1e-8

Each is a torch.optim.Optimizer over parameters whose .grad is dense or a sparse COO tensor with one sparse dimension (the
sparse_grad=True table gradients), so it drops into any `loss.backward(); opt.step()` loop.  A step reproduces TF's update
bit for bit: every op is one float32 rounding in TF's order, hyperparameters are rounded to float32 as TF casts them, a
sparse gradient that is not coalesced is coalesce()d first (TF sums duplicate IndexedSlices), and a parameter whose .grad is
None is skipped (apply_gradients drops None gradients).  The update rules are written out in include/euler_b200.h
(eu_optim_momentum, eu_optim_adagrad, eu_optim_adam).  Where they depart from torch's optimizers:
  - Adam puts epsilon after sqrt(v) and folds the bias corrections into alpha = lr * sqrt(1 - beta2^t) / (1 - beta1^t).
  - Sparse Adam decays m and v and moves var on EVERY row of the table each step, not only the gradient's rows
    (torch.optim.SparseAdam is lazy).
  - Adagrad's accumulator starts at initial_accumulator_value (0.1) and has no epsilon.
Adam's beta1_power and beta2_power (TF's non-slot variables, starting at beta1 and beta2) are one pair per optimizer, advanced
once at the end of every step(), also for parameters without a gradient; state_dict() saves them as 'beta_powers'.

With fused=True (the default) each parameter's update is one device op (ops.optim_momentum_, optim_adagrad_, optim_adam_)
that reads and writes each tensor once and never synchronises with the host, so a step can be captured in a CUDA graph.
With fused=False the step runs TF's op sequence literally in torch, one torch op per TF op, on any device: the reference the
fused ops are checked against.

bfloat16 parameters (the skip-gram id tables of unsupervised.UnsuperviseModel(table_dtype=torch.bfloat16)) are trained by the
fused ops only, with slots of the parameter's dtype.  Each value is widened exactly to f32 and updated in f32, and the var and
every slot are written back by stochastic rounding keyed by (seed, the optimizer's step counter, the parameter's index in the
optimizer, the element): one seed gives the same bits on every run.  The step counter (`sr_step`, int64 on the first bf16
parameter's device) advances once per step, after every parameter, as Adam's powers do; state_dict() saves it.  Torch
autograd would round a bf16 leaf's f32 gradient to nearest bf16, so a bf16 parameter takes its gradient through
apply_sparse(param, rows, values) from f32 rows and values, never through .grad.  fused=False refuses bf16 parameters.
"""
import math

import numpy as np
import torch

from . import ops


def _f32(x):
    """x rounded to float32, as TF casts a Python hyperparameter to the variable's dtype"""
    return float(np.float32(x))


def _one_minus(b):
    """1 - b in float32 arithmetic, TF's (1 - beta_t)"""
    return float(np.float32(1) - np.float32(b))


def _sqrt(x):
    """the correctly rounded float32 sqrt TF computes: torch's CUDA sqrt is one; its CPU kernel may be off by an ulp, so on
    the CPU it is taken from float64, which rounds to the same float32"""
    return torch.sqrt(x) if x.is_cuda else torch.sqrt(x.double()).float()


def _check(name, value, ok, want):
    if not isinstance(value, (int, float)) or isinstance(value, bool) or not ok(float(value)):
        raise ValueError("%s must be %s, got %r" % (name, want, value))


def _finite_nonneg(x):
    return math.isfinite(x) and x >= 0


def _rows(grad):
    """(rows, values) of a sparse COO gradient, coalesced first when it is not"""
    if not grad.is_coalesced():
        grad = grad.coalesce()
    return grad._indices()[0], grad._values()


class _TFOptimizer(torch.optim.Optimizer):
    def __init__(self, params, defaults, fused, seed):
        self.fused = bool(fused)   # add_param_group reads it
        if not isinstance(seed, int) or isinstance(seed, bool) or not 0 <= seed < 2 ** 64:
            raise ValueError("seed must be an int in [0, 2^64), got %r" % (seed,))
        self.seed = seed
        self.sr_step = None   # the stochastic-rounding step counter, made with the first bf16 parameter
        super().__init__(params, defaults)

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        bf16 = [p for p in self.param_groups[-1]['params'] if p.dtype == torch.bfloat16]
        if bf16 and not self.fused:
            self.param_groups.pop()
            raise ValueError("a bfloat16 parameter is trained by the fused update only (fused=True)")
        if bf16 and self.sr_step is None:
            self.sr_step = torch.zeros((), dtype=torch.int64, device=bf16[0].device)

    def _each(self):
        """(index, param, group) of every parameter, in the order the parameters were given"""
        i = 0
        for group in self.param_groups:
            for p in group['params']:
                yield i, p, group
                i += 1

    def _update(self, i, p, grad, group):
        state = self.state[p]
        if not state:
            self._init_state(p, state, group)
        if self.fused:
            self._fused(p, grad, state, group, dict(seed=self.seed, step=self.sr_step, tensor=i))
        elif grad.is_sparse:
            self._literal_sparse(p, *_rows(grad), state, group)
        else:
            self._literal_dense(p, grad, state, group)

    @torch.no_grad()
    def step(self, closure=None, sparse_grads=None):
        """One step over every parameter with a gradient.  sparse_grads (optional) maps parameters to float32 sparse COO
        gradients, which are used instead of their .grad (never rounded to the parameter's dtype: this is how a bfloat16
        table trains beside dense parameters).  Adam's powers and the rounding step counter advance once."""
        sparse_grads = {} if sparse_grads is None else sparse_grads
        mine = {id(p) for _, p, _ in self._each()}
        for p, g in sparse_grads.items():
            if id(p) not in mine:
                raise ValueError("step: a parameter of sparse_grads is not one of this optimizer's")
            if not torch.is_tensor(g) or not g.is_sparse or g.dtype != torch.float32 or tuple(g.shape) != tuple(p.shape):
                raise ValueError("step: sparse_grads must map each parameter to a float32 sparse COO gradient of its shape")
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for i, p, group in self._each():
            grad = sparse_grads.get(p, p.grad)
            if grad is not None:
                self._update(i, p, grad, group)
        self._finish()
        return loss

    @torch.no_grad()
    def apply_sparse(self, param, rows, values):
        """One step from sparse f32 gradients, without .grad: param, rows and values are one parameter, its rows i64[R]
        (sorted and unique, as a coalesced gradient has them) and values f32[R, ...] of the parameter's row shape, or lists
        of equal length with one entry per parameter.  The parameters not listed take no update this step, as a None .grad
        in step().  The values are never rounded to the parameter's dtype: this is how a bfloat16 parameter is trained."""
        if torch.is_tensor(param):
            param, rows, values = [param], [rows], [values]
        if not len(param) == len(rows) == len(values):
            raise ValueError("apply_sparse: param, rows and values must have one length")
        index = {id(p): (i, g) for i, p, g in self._each()}
        for p in param:
            if id(p) not in index:
                raise ValueError("apply_sparse: a parameter is not one of this optimizer's")
        for p, r, v in zip(param, rows, values):
            if not torch.is_tensor(v) or v.dtype != torch.float32:
                raise ValueError("apply_sparse: values must be float32, got %s" % getattr(v, 'dtype', type(v)))
            i, group = index[id(p)]
            grad = torch.sparse_coo_tensor(r.reshape(1, -1), v, tuple(p.shape), is_coalesced=True, check_invariants=False)
            self._update(i, p, grad, group)
        self._finish()

    def _finish(self):
        if self.sr_step is not None:
            self.sr_step.add_(1)

    def state_dict(self):
        sd = super().state_dict()
        if self.sr_step is not None:
            sd['sr_step'] = self.sr_step.clone()
        return sd

    def load_state_dict(self, state_dict):
        sd = dict(state_dict)
        step = sd.pop('sr_step', None)
        super().load_state_dict(sd)
        if step is not None and self.sr_step is not None:
            self.sr_step.copy_(step)


class MomentumOptimizer(_TFOptimizer):
    """tf.train.MomentumOptimizer(learning_rate, momentum), non-Nesterov: accum = accum * momentum + g, var = var - lr *
    accum.  A sparse gradient updates its rows only.  Slot: state['momentum'], starting at zeros."""

    def __init__(self, params, learning_rate, momentum, fused=True, seed=0):
        _check("learning_rate", learning_rate, _finite_nonneg, "a finite number >= 0")
        _check("momentum", momentum, _finite_nonneg, "a finite number >= 0")
        super().__init__(params, dict(lr=learning_rate, momentum=momentum), fused, seed)

    def _init_state(self, p, state, group):
        state['momentum'] = torch.zeros_like(p, memory_format=torch.contiguous_format)

    def _fused(self, p, grad, state, group, sr):
        ops.optim_momentum_(p, state['momentum'], grad, group['lr'], group['momentum'], **sr)

    def _literal_dense(self, p, g, state, group):
        a = state['momentum']
        a.copy_(a * _f32(group['momentum']) + g)
        p.sub_(_f32(group['lr']) * a)

    def _literal_sparse(self, p, rows, g, state, group):
        a = state['momentum']
        a_rows = a[rows] * _f32(group['momentum']) + g
        a.index_copy_(0, rows, a_rows)
        p.index_copy_(0, rows, p[rows] - _f32(group['lr']) * a_rows)


class AdagradOptimizer(_TFOptimizer):
    """tf.train.AdagradOptimizer(learning_rate, initial_accumulator_value=0.1): accum = accum + g * g, var = var - (lr * g)
    * (1 / sqrt(accum)).  A sparse gradient updates its rows only.  Slot: state['accumulator']."""

    def __init__(self, params, learning_rate, initial_accumulator_value=0.1, fused=True, seed=0):
        _check("learning_rate", learning_rate, _finite_nonneg, "a finite number >= 0")
        _check("initial_accumulator_value", initial_accumulator_value, lambda x: math.isfinite(x) and x > 0,
               "a finite number > 0")
        super().__init__(params, dict(lr=learning_rate, initial_accumulator_value=initial_accumulator_value), fused, seed)

    def _init_state(self, p, state, group):
        state['accumulator'] = torch.full_like(p, _f32(group['initial_accumulator_value']),
                                               memory_format=torch.contiguous_format)

    def _fused(self, p, grad, state, group, sr):
        ops.optim_adagrad_(p, state['accumulator'], grad, group['lr'], **sr)

    def _literal_dense(self, p, g, state, group):
        a = state['accumulator']
        a.copy_(a + g * g)
        p.sub_((_f32(group['lr']) * g) * torch.reciprocal(_sqrt(a)))

    def _literal_sparse(self, p, rows, g, state, group):
        a = state['accumulator']
        a_rows = a[rows] + g * g
        a.index_copy_(0, rows, a_rows)
        p.index_copy_(0, rows, p[rows] - (_f32(group['lr']) * g) * torch.reciprocal(_sqrt(a_rows)))


class AdamOptimizer(_TFOptimizer):
    """tf.train.AdamOptimizer(learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8).  alpha = (lr * sqrt(1 -
    beta2_power)) / (1 - beta1_power).  Dense gradient (ApplyAdam): m = m + (g - m) * (1 - beta1), v = v + (g * g - v) *
    (1 - beta2), var = var - (m * alpha) / (sqrt(v) + epsilon).  Sparse gradient (_apply_sparse_shared), every row: m = m *
    beta1 and v = v * beta2, plus g * (1 - beta1) and (g * g) * (1 - beta2) on the gradient's rows, then var = var - (alpha *
    m) / (sqrt(v) + epsilon).  Slots: state['m'], state['v'], starting at zeros.  beta1 and beta2 are one per optimizer, as
    the power pair they advance (`beta_powers`, float32[2] on the first parameter's device)."""

    def __init__(self, params, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, fused=True, seed=0):
        _check("learning_rate", learning_rate, _finite_nonneg, "a finite number >= 0")
        for name, b in (("beta1", beta1), ("beta2", beta2)):
            _check(name, b, lambda x: 0 <= x < 1, "in [0, 1)")
        _check("epsilon", epsilon, _finite_nonneg, "a finite number >= 0")
        super().__init__(params, dict(lr=learning_rate, beta1=beta1, beta2=beta2, epsilon=epsilon), fused, seed)
        dev = self.param_groups[0]['params'][0].device
        self.beta_powers = torch.tensor([_f32(beta1), _f32(beta2)], dtype=torch.float32, device=dev)
        self._betas = self.beta_powers.clone()

    def add_param_group(self, param_group):
        for k in ('beta1', 'beta2'):
            if param_group.get(k, self.defaults[k]) != self.defaults[k]:
                raise ValueError("AdamOptimizer: %s is one per optimizer (TF's %s_power), a group cannot set its own" % (k, k))
        super().add_param_group(param_group)

    def _init_state(self, p, state, group):
        state['m'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        state['v'] = torch.zeros_like(p, memory_format=torch.contiguous_format)

    def _fused(self, p, grad, state, group, sr):
        ops.optim_adam_(p, state['m'], state['v'], grad, self.beta_powers, group['lr'], group['beta1'], group['beta2'],
                        group['epsilon'], **sr)

    def _alpha(self, group):
        b1p, b2p = self.beta_powers[0], self.beta_powers[1]
        return (_f32(group['lr']) * _sqrt(1 - b2p)) / (1 - b1p)

    def _literal_dense(self, p, g, state, group):
        m, v = state['m'], state['v']
        m.copy_(m + (g - m) * _one_minus(group['beta1']))
        v.copy_(v + (g * g - v) * _one_minus(group['beta2']))
        p.sub_((m * self._alpha(group)) / (_sqrt(v) + _f32(group['epsilon'])))

    def _literal_sparse(self, p, rows, g, state, group):
        m, v = state['m'], state['v']
        m.copy_(m * _f32(group['beta1']))
        m.index_copy_(0, rows, m[rows] + g * _one_minus(group['beta1']))
        v.copy_(v * _f32(group['beta2']))
        v.index_copy_(0, rows, v[rows] + (g * g) * _one_minus(group['beta2']))
        p.sub_((self._alpha(group) * m) / (_sqrt(v) + _f32(group['epsilon'])))

    def _finish(self):
        self.beta_powers.mul_(self._betas)
        super()._finish()

    def state_dict(self):
        sd = super().state_dict()
        sd['beta_powers'] = self.beta_powers.clone()
        return sd

    def load_state_dict(self, state_dict):
        sd = dict(state_dict)
        powers = sd.pop('beta_powers')
        super().load_state_dict(sd)
        self.beta_powers.copy_(powers)


def minimize(optimizer, loss, module):
    """One training step of a model whose node encoders may hold bfloat16 tables (encoders.ShallowEncoder(table_dtype=)):
    clears every parameter's .grad and every table proxy's, runs loss.backward(), collects each bf16 table's f32 sparse
    gradient from its proxy (every ShallowEncoder in module.modules(), a shared one once) and steps `optimizer` once with
    them as sparse_grads.  Without a bf16 table it is zero_grad(); loss.backward(); step().  Returns loss."""
    from .encoders import ShallowEncoder
    encoders = [m for m in module.modules() if isinstance(m, ShallowEncoder)]
    pairs = {}
    for e in encoders:
        for table, proxy in e.table_proxies():
            pairs[id(table)] = (table, proxy)
    optimizer.zero_grad()
    for _, proxy in pairs.values():
        proxy.grad = None
    loss.backward()
    sparse_grads = {table: proxy.grad for table, proxy in pairs.values() if proxy.grad is not None}
    optimizer.step(sparse_grads=sparse_grads)
    return loss


OPTIMIZERS = {
    'sgd': lambda params, lr, **kw: MomentumOptimizer(params, lr, 0.0, **kw),
    'momentum': lambda params, lr, **kw: MomentumOptimizer(params, lr, 0.9, **kw),
    'adagrad': AdagradOptimizer,
    'adam': AdamOptimizer,
}


def get(name):
    """optimizers.get: the factory of optimizer `name`, one of 'adagrad', 'adam', 'momentum' and 'sgd', called as
    get(name)(params, lr) (keyword arguments such as fused=False pass through)"""
    if name not in OPTIMIZERS:
        raise ValueError("optimizer must be one of %s, got %r" % (sorted(OPTIMIZERS), name))
    return OPTIMIZERS[name]
