"""GPU: the fixed order of the id-table gradients, bit for bit.  Every entry of a table's list (node order, then the bag's
stored order) is summed per distinct row in 256-entry chunks from +0, and a row's chunk sums are added from +0 in chunk order.
The restatement below does exactly that in numpy float32 and the int32 views of the gradients must be equal: on a default row
of more than three chunks of entries, rows of exactly 256 and 257 entries, and non-integer gradients, so that any other
grouping of the adds would show."""
import numpy as np
import pytest
import torch

import embedding_reference as er

pytestmark = pytest.mark.gpu

N_NODES, N_ROWS, DEFAULT = 3000, 50, 3
EMPTY = 1000                 # nodes without values: 1000 entries of the default row, four chunks
EXACT = {7: 256, 8: 257}     # rows hit by exactly one full chunk, and by one entry more
COUNT = 10                   # the pooled op's segment length


def _slot():
    """per-node lengths and the values in storage order: EMPTY empty bags first, then 1-4 values per node, rows 7 and 8
    exactly EXACT times, every other value in [9, N_ROWS)"""
    rng = np.random.RandomState(17)
    lens = np.concatenate([np.zeros(EMPTY, np.int64), rng.randint(1, 5, size=N_NODES - EMPTY)])
    rng.shuffle(lens)
    total = int(lens.sum())
    vals = np.concatenate([np.full(n, r) for r, n in EXACT.items()] + [rng.randint(9, N_ROWS, size=total - sum(EXACT.values()))])
    rng.shuffle(vals)
    return lens, vals


@pytest.fixture(scope="module")
def env():
    import euler_b200
    lens, vals = _slot()
    it = iter(vals)
    g = er.slot_graph(23, N_NODES, [lambda rng, n: lens], [lambda rng, k: np.array([next(it) for _ in range(k)], np.int64)])
    gr = er.cuda_slot_graph(g)
    nodes = g["ids"][np.random.RandomState(5).permutation(N_NODES)].astype(np.int64)
    bags = er.bags(g["ids"], g["u64_ptr"], g["u64_val"], g["S"], nodes, 0, DEFAULT)
    hits = np.bincount([v for b in bags for v in b], minlength=N_ROWS)
    assert hits[DEFAULT] > 3 * 256 and hits[7] == 256 and hits[8] == 257
    return dict(gr=gr, nodes=nodes, bags=bags)


@pytest.fixture(autouse=True)
def _installed(env):
    import euler_b200
    euler_b200.set_graph(env["gr"], rng="minstd", seed=1)


def _restated(n_rows, keys, values):
    """the documented order in float32: keys[e] the row of entry e in list order, values [E, dim] its value"""
    out = np.zeros((n_rows, values.shape[1]), np.float32)
    for r in np.unique(keys):
        x = values[keys == r]
        total = np.zeros(values.shape[1], np.float32)
        for c0 in range(0, len(x), 256):
            acc = np.zeros(values.shape[1], np.float32)
            for row in x[c0:c0 + 256]:
                acc = acc + row
            total = total + acc
        out[r] = total
    return out


def _slot_entries(bags, node_grad, combiner):
    """the slot's entry list: keys and values, node i's gradient row divided by its combiner's divisor (one rounding)"""
    keys, vals = [], []
    for i, b in enumerate(bags):
        n = np.float32(len(b))
        den = {"sum": None, "mean": n, "sqrtn": np.sqrt(n)}[combiner]
        v = node_grad[i] if den is None else (node_grad[i] / den).astype(np.float32)
        keys += b
        vals += [v] * len(b)
    return np.asarray(keys), np.stack(vals).astype(np.float32)


def _dense(grad):
    return (grad.coalesce().to_dense() if grad.is_sparse else grad).cpu().numpy()


def _grad(seed, rows, dim):
    return torch.randn(rows, dim, generator=torch.Generator().manual_seed(seed)).cuda() * 0.37


@pytest.mark.parametrize("dim", (5, 16))
@pytest.mark.parametrize("sparse_grad", (False, True))
@pytest.mark.parametrize("combiner", er.COMBINERS)
def test_sparse_feature_embedding_order(env, dim, sparse_grad, combiner):
    import euler_b200
    nodes, bags = env["nodes"], env["bags"]
    table = torch.randn(N_ROWS, dim, generator=torch.Generator().manual_seed(1)).cuda().requires_grad_(True)
    g = _grad(2, len(nodes), dim)
    euler_b200.sparse_feature_embedding(nodes, "u64_0", table, DEFAULT, combiner, sparse_grad=sparse_grad).backward(g)
    keys, vals = _slot_entries(bags, g.cpu().numpy(), combiner)
    want = _restated(N_ROWS, keys, vals)
    assert np.array_equal(_dense(table.grad).view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("dim", (5, 16))
@pytest.mark.parametrize("sparse_grad", (False, True))
@pytest.mark.parametrize("combiner", ("sum", "mean"))
def test_shallow_encode_pool_mean_order(env, dim, sparse_grad, combiner):
    """pool='mean': node i's entries read row i / COUNT of the pooled gradient, divided by fl(COUNT) first, then by the
    slot's combiner divisor"""
    import euler_b200
    nodes, bags = env["nodes"], env["bags"]
    n_id = N_NODES + 2
    id_table = torch.randn(n_id, dim, generator=torch.Generator().manual_seed(3)).cuda().requires_grad_(True)
    table = torch.randn(N_ROWS, dim, generator=torch.Generator().manual_seed(4)).cuda().requires_grad_(True)
    out = euler_b200.shallow_encode_pool(nodes, COUNT, id_table, sparse=[("u64_0", table, DEFAULT, combiner)], pool="mean",
                                         sparse_grad=sparse_grad)
    g = _grad(6, len(nodes) // COUNT, 2 * dim)
    out.backward(g)
    gh = g.cpu().numpy()
    node_grad = (gh[np.arange(len(nodes)) // COUNT] / np.float32(COUNT)).astype(np.float32)   # [M, id | slot]
    want_id = _restated(n_id, nodes, node_grad[:, :dim])
    keys, vals = _slot_entries(bags, node_grad[:, dim:], combiner)
    want_slot = _restated(N_ROWS, keys, vals)
    assert np.array_equal(_dense(id_table.grad).view(np.int32), want_id.view(np.int32))
    assert np.array_equal(_dense(table.grad).view(np.int32), want_slot.view(np.int32))
