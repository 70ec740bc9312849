"""numpy float32 restatement of TF 1.x's Momentum, Adagrad and Adam updates (training_ops apply_momentum / apply_adagrad /
ApplyAdam and sparse_apply_momentum / sparse_apply_adagrad, AdamOptimizer._apply_sparse_shared), the rules
include/euler_b200.h states.  Every operation is one numpy float32 op, so it rounds once, in TF's order.

A gradient is a dense array of var's shape or a pair (rows int64[R], values float32[R, ...]); a pair with repeated rows is
summed first, duplicates added in order of appearance (TF's _apply_sparse_duplicate_indices).  Each update works in place on
the var and slot arrays it is given."""
import numpy as np

F32 = np.float32


def f32(x):
    return F32(x)


def dedup(rows, values):
    """(sorted unique rows, summed values), as coalesce() gives them: a row's first value, plus each later duplicate in order
    of appearance with one f32 add"""
    rows = np.asarray(rows, np.int64)
    values = np.asarray(values, F32)
    uniq, inv = np.unique(rows, return_inverse=True)
    out = np.zeros((uniq.size,) + values.shape[1:], F32)
    seen = np.zeros(uniq.size, bool)
    for k in range(rows.size):
        out[inv[k]] = out[inv[k]] + values[k] if seen[inv[k]] else values[k]
        seen[inv[k]] = True
    return uniq, out


def momentum(var, accum, grad, lr, mom):
    lr, mom = f32(lr), f32(mom)
    if isinstance(grad, tuple):
        rows, g = dedup(*grad)
        a = accum[rows] * mom + g
        accum[rows] = a
        var[rows] = var[rows] - lr * a
    else:
        accum[...] = accum * mom + np.asarray(grad, F32)
        var[...] = var - lr * accum


def adagrad(var, accum, grad, lr):
    lr = f32(lr)
    if isinstance(grad, tuple):
        rows, g = dedup(*grad)
        a = accum[rows] + g * g
        accum[rows] = a
        var[rows] = var[rows] - (lr * g) * (F32(1) / np.sqrt(a))
    else:
        g = np.asarray(grad, F32)
        accum[...] = accum + g * g
        var[...] = var - (lr * g) * (F32(1) / np.sqrt(accum))


class Adam:
    """one AdamOptimizer: its (beta1_power, beta2_power) pair, starting at (beta1, beta2)"""

    def __init__(self, lr=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8):
        self.lr, self.b1, self.b2, self.eps = f32(lr), f32(beta1), f32(beta2), f32(epsilon)
        self.powers = np.array([self.b1, self.b2], F32)

    def alpha(self):
        b1p, b2p = self.powers
        return (self.lr * np.sqrt(F32(1) - b2p)) / (F32(1) - b1p)

    def update(self, var, m, v, grad):
        """one variable's update at the current powers"""
        alpha, b1, b2, eps = self.alpha(), self.b1, self.b2, self.eps
        if isinstance(grad, tuple):
            rows, g = dedup(*grad)
            m[...] = m * b1
            m[rows] = m[rows] + g * (F32(1) - b1)
            v[...] = v * b2
            v[rows] = v[rows] + (g * g) * (F32(1) - b2)
            var[...] = var - (alpha * m) / (np.sqrt(v) + eps)
        else:
            g = np.asarray(grad, F32)
            m[...] = m + (g - m) * (F32(1) - b1)
            v[...] = v + (g * g - v) * (F32(1) - b2)
            var[...] = var - (m * alpha) / (np.sqrt(v) + eps)

    def finish(self):
        """_finish: each power times its beta, once per step, after every variable"""
        self.powers = (self.powers * np.array([self.b1, self.b2], F32)).astype(F32)

    def step(self, items):
        """one apply_gradients over (var, m, v, grad) items; grad None skips the variable"""
        for var, m, v, grad in items:
            if grad is not None:
                self.update(var, m, v, grad)
        self.finish()


SLOTS = {'sgd': ('momentum',), 'momentum': ('momentum',), 'adagrad': ('accumulator',), 'adam': ('m', 'v')}


def run(name, var, grads, lr, **hp):
    """optimizers.get(name)(params=[var], lr) stepped once per entry of grads (a dense array, a (rows, values) pair, or None
    for a step without a gradient), from fresh slots.  Returns (var, {slot name: array}, Adam's powers or None); var is
    updated in place.  hp: Adagrad's initial_accumulator_value, Adam's beta1, beta2, epsilon."""
    if name == 'adagrad':
        slots = {'accumulator': np.full_like(var, f32(hp.get('initial_accumulator_value', 0.1)))}
    else:
        slots = {k: np.zeros_like(var) for k in SLOTS[name]}
    adam = Adam(lr, **hp) if name == 'adam' else None
    for g in grads:
        if name == 'adam':
            adam.step([(var, slots['m'], slots['v'], g)])
        elif g is None:
            continue
        elif name == 'adagrad':
            adagrad(var, slots['accumulator'], g, lr)
        else:
            momentum(var, slots['momentum'], g, lr, 0.0 if name == 'sgd' else 0.9)
    return var, slots, None if adam is None else adam.powers
