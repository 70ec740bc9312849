"""CPU: euler_b200/optimizers.py's fused=False steps (TF 1.x's op sequence in torch) bit for bit against the numpy float32
restatement (tests/optim_reference.py) over consecutive steps, dense and sparse, with duplicate rows; get, the constructors'
errors, parameters without a gradient, Adam's power pair and state_dict round trips."""
import numpy as np
import pytest
import torch

import graphs  # noqa: F401  (sys.path)
import optim_reference as ref
from euler_b200 import optimizers

F32 = np.float32
NAMES = ['sgd', 'momentum', 'adagrad', 'adam']
LR = {'sgd': 0.1, 'momentum': 0.05, 'adagrad': 0.3, 'adam': 0.01}


def _bits(x):
    return np.ascontiguousarray(np.asarray(x, F32)).view(np.int32)


def _assert_bits(got, want, what):
    np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=what)


def _values(rng, shape):
    """gradient values with zeros, subnormals and large entries among ordinary ones"""
    g = rng.randn(*shape).astype(F32)
    flat = g.reshape(-1)
    k = flat.size
    flat[rng.rand(k) < 0.1] = 0
    flat[rng.rand(k) < 0.05] = F32(3e-39) * rng.choice([-1, 1])
    flat[rng.rand(k) < 0.05] = F32(1e18) * rng.choice([-1, 1])
    return g


def _grads(rng, shape, form, steps=5):
    """per-step gradients for a var of shape: dense arrays, or (rows, values) pairs; 'dup' repeats some rows once, out of
    order (an uncoalesced COO gradient)"""
    out = []
    N = shape[0]
    for s in range(steps):
        if form == 'dense':
            out.append(_values(rng, shape))
            continue
        rows = np.sort(rng.choice(N, size=max(1, N // 2), replace=False))
        if s == 1:
            rows = np.array([0, N - 1], np.int64)
        if form == 'dup':
            rows = rng.permutation(np.concatenate([rows, rows[::2]]))
        out.append((rows.astype(np.int64), _values(rng, (rows.size,) + tuple(shape[1:]))))
    return out


def _torch_grad(g, shape):
    if isinstance(g, tuple):
        rows, vals = g
        return torch.sparse_coo_tensor(torch.from_numpy(rows)[None], torch.from_numpy(vals), shape, check_invariants=True)
    return torch.from_numpy(g)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("form", ['dense', 'sparse', 'dup'])
@pytest.mark.parametrize("shape", [(9, 3), (6, 4), (11,)])
def test_literal_matches_restatement(name, form, shape):
    rng = np.random.RandomState(len(name) * 7 + len(form) + shape[0])
    var0 = (rng.randn(*shape) * 2).astype(F32)
    grads = _grads(rng, shape, form)
    p = torch.nn.Parameter(torch.from_numpy(var0.copy()))
    opt = optimizers.get(name)([p], LR[name], fused=False)
    want_var, want_slots, want_powers = ref.run(name, var0.copy(), grads, LR[name])
    for k, g in enumerate(grads):
        p.grad = _torch_grad(g, shape)
        opt.step()
    _assert_bits(p.detach().numpy(), want_var, "%s %s var" % (name, form))
    for slot, want in want_slots.items():
        _assert_bits(opt.state[p][slot].numpy(), want, "%s %s %s" % (name, form, slot))
    if name == 'adam':
        _assert_bits(opt.beta_powers.numpy(), want_powers, "powers")


def test_adam_hyperparameters_round_to_f32():
    """non-default hyperparameters, each rounded to f32 as TF casts it; Adagrad's initial accumulator likewise"""
    rng = np.random.RandomState(5)
    var0 = rng.randn(5, 2).astype(F32)
    grads = _grads(rng, (5, 2), 'sparse') + _grads(rng, (5, 2), 'dense')
    for name, kw in (('adam', dict(beta1=0.7, beta2=0.95, epsilon=0.1)), ('adagrad', dict(initial_accumulator_value=0.3))):
        p = torch.nn.Parameter(torch.from_numpy(var0.copy()))
        opt = optimizers.get(name)([p], 1 / 3, fused=False, **kw)
        for g in grads:
            p.grad = _torch_grad(g, (5, 2))
            opt.step()
        want, _, _ = ref.run(name, var0.copy(), grads, 1 / 3, **kw)
        _assert_bits(p.detach().numpy(), want, name)


def test_get_names():
    p = [torch.nn.Parameter(torch.zeros(3))]
    assert isinstance(optimizers.get('sgd')(p, 0.1), optimizers.MomentumOptimizer)
    assert optimizers.get('sgd')(p, 0.1).defaults['momentum'] == 0.0
    assert optimizers.get('momentum')(p, 0.1).defaults['momentum'] == 0.9
    assert isinstance(optimizers.get('adagrad')(p, 0.1), optimizers.AdagradOptimizer)
    a = optimizers.get('adam')(p, 0.1)
    assert isinstance(a, optimizers.AdamOptimizer)
    assert (a.defaults['beta1'], a.defaults['beta2'], a.defaults['epsilon']) == (0.9, 0.999, 1e-8)
    assert optimizers.AdagradOptimizer(p, 0.1).defaults['initial_accumulator_value'] == 0.1
    assert optimizers.AdamOptimizer(p).defaults['lr'] == 0.001
    for bad in ('rmsprop', 'Adam', 'lazy_adam', None):
        with pytest.raises(ValueError):
            optimizers.get(bad)
    import euler_b200
    assert euler_b200.optimizers is optimizers


def test_constructor_errors():
    p = [torch.nn.Parameter(torch.zeros(3))]
    with pytest.raises(ValueError):
        optimizers.MomentumOptimizer(p, -0.1, 0.9)
    with pytest.raises(ValueError):
        optimizers.MomentumOptimizer(p, float('nan'), 0.9)
    with pytest.raises(ValueError):
        optimizers.MomentumOptimizer(p, 0.1, -1.0)
    with pytest.raises(ValueError):
        optimizers.MomentumOptimizer(p, '0.1', 0.9)
    with pytest.raises(ValueError):
        optimizers.AdagradOptimizer(p, 0.1, initial_accumulator_value=0.0)
    with pytest.raises(ValueError):
        optimizers.AdagradOptimizer(p, 0.1, initial_accumulator_value=-1)
    for kw in (dict(beta1=1.0), dict(beta2=-0.1), dict(beta1=float('nan')), dict(epsilon=-1e-8), dict(learning_rate=float('inf'))):
        with pytest.raises(ValueError):
            optimizers.AdamOptimizer(p, **kw)
    with pytest.raises(ValueError):   # TF has one beta1_power per optimizer
        optimizers.AdamOptimizer([{'params': p, 'beta1': 0.5}])
    with pytest.raises(ValueError):
        optimizers.AdamOptimizer([])


def test_no_grad_parameter_is_skipped_and_powers_advance_once_per_step():
    rng = np.random.RandomState(2)
    a0, b0 = rng.randn(4, 3).astype(F32), rng.randn(6).astype(F32)
    pa, pb = torch.nn.Parameter(torch.from_numpy(a0.copy())), torch.nn.Parameter(torch.from_numpy(b0.copy()))
    opt = optimizers.AdamOptimizer([pa, pb], 0.01, fused=False)
    adam = ref.Adam(0.01)
    ma, va, mb, vb = (np.zeros_like(x) for x in (a0, a0, b0, b0))
    wa, wb = a0.copy(), b0.copy()
    for s in range(4):
        ga = _values(rng, (4, 3))
        gb = None if s % 2 else _values(rng, (6,))
        pa.grad = torch.from_numpy(ga)
        pb.grad = None if gb is None else torch.from_numpy(gb)
        opt.step()
        adam.step([(wa, ma, va, ga), (wb, mb, vb, gb)])
        _assert_bits(opt.beta_powers.numpy(), adam.powers, "powers step %d" % s)
    _assert_bits(pa.detach().numpy(), wa, "a")
    _assert_bits(pb.detach().numpy(), wb, "b")
    # a step with no gradient at all: nothing moves, the powers still advance
    pa.grad = pb.grad = None
    before = pa.detach().clone()
    opt.step()
    adam.finish()
    assert torch.equal(pa.detach(), before)
    _assert_bits(opt.beta_powers.numpy(), adam.powers, "powers without gradients")
    # momentum and adagrad never create a slot for a parameter that never had a gradient
    q = torch.nn.Parameter(torch.zeros(3))
    for name in ('momentum', 'adagrad'):
        o = optimizers.get(name)([q], 0.1, fused=False)
        o.step()
        assert len(o.state) == 0 and torch.equal(q.detach(), torch.zeros(3))


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_round_trip_resumes_bit_exact(name):
    rng = np.random.RandomState(9)
    var0 = rng.randn(8, 4).astype(F32)
    grads = _grads(rng, (8, 4), 'sparse', steps=3) + _grads(rng, (8, 4), 'dense', steps=3)

    def make():
        p = torch.nn.Parameter(torch.from_numpy(var0.copy()))
        return p, optimizers.get(name)([p], LR[name], fused=False)

    p1, o1 = make()
    for g in grads:
        p1.grad = _torch_grad(g, (8, 4))
        o1.step()
    p2, o2 = make()
    for g in grads[:3]:
        p2.grad = _torch_grad(g, (8, 4))
        o2.step()
    sd = o2.state_dict()
    p3, o3 = make()
    with torch.no_grad():
        p3.copy_(p2)
    o3.load_state_dict(sd)
    if name == 'adam':
        assert torch.equal(sd['beta_powers'], o3.beta_powers) and sd['beta_powers'] is not o3.beta_powers
    for g in grads[3:]:
        p3.grad = _torch_grad(g, (8, 4))
        o3.step()
    _assert_bits(p3.detach().numpy(), p1.detach().numpy(), name)
    if name == 'adam':
        _assert_bits(o3.beta_powers.numpy(), o1.beta_powers.numpy(), "powers")


def test_fused_step_refuses_cpu_parameters():
    """fused=True runs the device op: a CPU parameter is refused, not quietly updated in torch"""
    import euler_b200
    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.ones(4)
    for name in NAMES:
        with pytest.raises(euler_b200.EulerError):
            optimizers.get(name)([p], 0.1).step()
    assert torch.equal(p.detach(), torch.zeros(4))
