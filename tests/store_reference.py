"""The embedding-store updates on bfloat16 stores (store.cu's eu_store_*_dtype), restated in numpy: the exchange's
round-to-nearest write and widened read, and the accumulation's f32 sum, widened add and stochastic rounding.  Test
infrastructure."""
import numpy as np

import bf16_reference as bf
import sr_reference as sr


def distinct_sums(ids, grad, count, pool):
    """{id: S_v f32[dim]}: each id's entries e in input order, grad[e // count] (divided by fl(count) as read under 'mean'),
    summed left to right from +0 in chunks of 256, a sum of several chunks adding its chunk sums in chunk order from +0"""
    ids = np.asarray(ids).reshape(-1)
    grad = np.asarray(grad, np.float32)
    c = np.float32(count)
    order = np.argsort(ids, kind="stable")
    keys, starts = np.unique(ids[order], return_index=True)
    bounds = list(starts) + [len(order)]
    zero = np.zeros((1, grad.shape[1]), np.float32)
    out = {}
    for k, v in enumerate(keys):
        es = order[bounds[k]:bounds[k + 1]]
        x = grad[es // count]
        if pool == "mean":
            x = x / c
        sums = [np.cumsum(np.concatenate([zero, x[i:i + 256]]), axis=0, dtype=np.float32)[-1] for i in range(0, len(es), 256)]
        out[int(v)] = sums[0] if len(sums) == 1 else np.cumsum(np.concatenate([zero, np.stack(sums)]), axis=0, dtype=np.float32)[-1]
    return out


def accumulate(G, ids, grad, count, pool, seed, step, tensor, rows=None):
    """A copy of the bf16 gradient store G (uint16 bits [N, dim]) after grad_store[ids] += grad: each touched row v becomes
    sr_bits(widen(G[v]) + S_v) with word 0 of philox_bits(seed, step, tensor, row(v) * dim + f).  rows: None, or int64[N]
    the global row of each given row of G (ids then index G's rows), so rows picked from a table too large to copy draw the
    table's own random bits."""
    G = np.array(G, np.uint16)
    dim = G.shape[1]
    glob = np.arange(G.shape[0], dtype=np.int64) if rows is None else np.asarray(rows, np.int64)
    for v, s in distinct_sums(ids, grad, count, pool).items():
        x = bf.widen(G[v]) + s                            # one f32 add per element
        elem = glob[v] * dim + np.arange(dim, dtype=np.int64)
        G[v] = sr.sr_bits(x, sr.philox_bits(seed, step, tensor, elem)[0])
    return G


def exchange(S, G, ids, rows):
    """(S', G', taken) for bf16 stores S, G (uint16 bits [N, dim]), ids [M] and f32 rows [M, dim]: taken = the widened
    pre-clear rows G[ids] (f32), S[v] = the round to nearest of rows[the last i with ids[i] = v] (a NaN as
    bf16_reference's canonical NaN, which the device's need not be), G[ids] = 0"""
    S, G = np.array(S, np.uint16), np.array(G, np.uint16)
    ids = np.asarray(ids).reshape(-1)
    taken = bf.widen(G[ids]).reshape(len(ids), G.shape[1])
    last = {int(v): i for i, v in enumerate(ids)}
    for v, i in last.items():
        S[v] = bf.round_bits(np.asarray(rows, np.float32)[i])
    G[ids] = 0
    return S, G, taken
