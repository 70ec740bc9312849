"""Stochastic rounding of trained bfloat16 tables, restated in numpy: the Philox4x32-10 block each stored element draws its
random bits from, the rounding itself (common.cuh's sr_st), and one optimizer step on bf16 tables (optim.cu's *_dtype
kernels).  Test infrastructure."""
import numpy as np

import bf16_reference as bf
import optim_reference as ref

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)


def philox_bits(seed, step, tensor, element):
    """the four uint32 words of Philox4x32-10 with counter (element lo, element hi, step mod 2^32, tensor) and key seed, for
    an array of element indices"""
    e = np.asarray(element, np.uint64)
    c = [e & MASK32, e >> np.uint64(32), np.full(e.shape, step % 2 ** 32, np.uint64), np.full(e.shape, tensor, np.uint64)]
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & MASK32]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return [w.astype(np.uint32) for w in c]


def sr_bits(x, r):
    """f32 array x -> the uint16 bits of its stochastic rounding to bf16 with random words r (their low 16 bits are added to
    the low half of x's bits, which are then dropped).  +-Inf stays; a NaN keeps its sign and upper payload, made quiet."""
    x = np.ascontiguousarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    out = ((u + (np.asarray(r, np.uint64) & np.uint64(0xFFFF))) >> np.uint64(16)).astype(np.uint16)
    special = (u & np.uint64(0x7F800000)) == np.uint64(0x7F800000)
    nan_bit = np.where((u & np.uint64(0x007FFFFF)) != 0, 0x40, 0).astype(np.uint16)
    out[special] = ((u[special] >> np.uint64(16)).astype(np.uint16) | nan_bit[special])
    return out


def step(name, tables, grad, seed, step_no, tensor, lr, adam=None, momentum=0.0, rows=None):
    """One update of bf16 tables (uint16 bit arrays [N, D]: var, then its slots) in place: widen, the f32 update of
    optim_reference, then stochastic rounding of every element written -- the rows of a sparse Momentum / Adagrad gradient,
    every element otherwise -- with word w of philox_bits(seed, step_no, tensor, r D + d) for table w.  grad: a dense f32
    array or (rows, values).  adam: an optim_reference.Adam whose powers are the step's (the caller calls finish()).
    rows: None when the tables are whole, else int64[N], the row of the full table each given row is: row i then draws with
    element rows[i] D + d, so a step can be restated on picked rows of a table too large to copy."""
    N, D = tables[0].shape
    f = [bf.widen(t).reshape(N, D) for t in tables]
    if name == 'adam':
        adam.update(f[0], f[1], f[2], grad)
    elif name == 'adagrad':
        ref.adagrad(f[0], f[1], grad, lr)
    else:
        ref.momentum(f[0], f[1], grad, lr, momentum)
    written = np.unique(grad[0]) if isinstance(grad, tuple) and name != 'adam' else np.arange(N)
    glob = written if rows is None else np.asarray(rows, np.int64)[written]
    elem = (glob.astype(np.int64)[:, None] * D + np.arange(D)[None, :]).reshape(-1)
    words = philox_bits(seed, step_no, tensor, elem)
    for w, (t, v) in enumerate(zip(tables, f)):
        t[written] = sr_bits(v[written].reshape(-1), words[w]).reshape(len(written), D)
