"""CPU: the knowledge-graph models' bfloat16 tables as the constructors build them, and the refusals that need no device:
an unknown table dtype, bf16 with fused=False, DistMult's whole-table L2 term on bf16 tables, and train_step without a
fused model or without one of optimizers.py's optimizers."""
import pytest
import torch

import graphs  # noqa: F401  (sys.path)

MODELS = ['TransE', 'TransH', 'TransR', 'TransD', 'DistMult']
TABLES = {'TransE': 2, 'TransH': 3, 'TransR': 3, 'TransD': 4, 'DistMult': 2}


def _model(cls, **kw):
    from euler_b200 import knowledge
    dims = (8, 4) if cls == 'TransR' else (8, 8)
    return getattr(knowledge, cls)(0, 0, 30, 5, *dims, num_negs=3, **kw)


@pytest.mark.parametrize("cls", MODELS)
def test_every_table_takes_the_requested_dtype(cls):
    for dt in (torch.bfloat16, torch.float32):
        torch.manual_seed(0)
        m = _model(cls, table_dtype=dt)
        tabs = m.tables()
        assert len(tabs) == TABLES[cls] == len(list(m.parameters()))
        assert {id(t) for t in tabs} == {id(p) for p in m.parameters()}
        for t in tabs:
            assert t.dtype == dt and t.requires_grad == (dt == torch.float32)
            assert float(t.float().abs().max()) <= 0.2 + 1e-3   # truncated normal, stddev 0.1, rounded once
        assert m.table_dtype == dt


@pytest.mark.parametrize("cls", MODELS)
def test_constructor_refusals(cls):
    with pytest.raises(ValueError, match="table_dtype"):
        _model(cls, table_dtype=torch.float16)
    with pytest.raises(ValueError, match="table_dtype"):
        _model(cls, table_dtype=torch.float64)
    with pytest.raises(ValueError, match="fused=True"):
        _model(cls, table_dtype=torch.bfloat16, fused=False)
    _model(cls, fused=False)   # f32 keeps the composed path


def test_distmult_l2_regular_refuses_bf16_tables():
    from euler_b200 import optimizers
    with pytest.raises(ValueError, match="l2_regular"):
        _model('DistMult', table_dtype=torch.bfloat16, l2_regular=True)
    m = _model('DistMult', l2_regular=True)
    assert m.l2_regular
    before = [t.clone() for t in m.tables()]
    with pytest.raises(ValueError, match="l2_regular"):   # a sparse step cannot carry the whole-table term
        m.train_step(torch.zeros((4, 3), dtype=torch.int64), optimizers.get('adam')(m.tables(), 0.001))
    for a, b in zip(before, m.tables()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("cls", MODELS)
def test_train_step_refusals(cls):
    from euler_b200 import optimizers
    m = _model(cls, table_dtype=torch.bfloat16)
    before = [t.clone() for t in m.tables()]
    edges = torch.zeros((4, 3), dtype=torch.int64)
    with pytest.raises(ValueError, match="optimizers"):
        m.train_step(edges, torch.optim.SGD(m.tables(), lr=0.1))   # no apply_sparse
    with pytest.raises(ValueError, match="fused"):
        optimizers.get('adam')(m.tables(), 0.001, fused=False)     # a non-fused optimizer takes no bf16 table
    f32 = _model(cls, fused=False)
    with pytest.raises(ValueError, match="fused=True"):
        f32.train_step(edges, optimizers.get('adam')(f32.tables(), 0.001))
    for a, b in zip(before, m.tables()):
        assert torch.equal(a, b)
