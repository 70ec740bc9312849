"""The device hash tables' key -> slot maps, restated in numpy, and keys built to collide in them.  (Test infrastructure.)

Every table probes linearly from a home slot `hash & (cap - 1)`, with cap = table_cap(keys):
    node id -> row       mix64(id)                 graph.cu k_hash_insert, common.cuh lookup_row
    fanout dedup         mix64(id)                 common.cuh dedup_insert_one (id 2^64-1: the extra slot [cap])
    first occurrence     mix64(id)                 uq.cuh uq_insert / uq_first (id 2^64-1: the extra slot [cap])
    SAGE segment         segment_hash(ids)         mp_ops.cu k_sage_classify (a slot keeps the upper 32 bits: the tag)
    edge                 edge_hash(src, dst, type) edges.cu eu_graph_set_edges, lookup_edge

mix64 (the MurmurHash3 finalizer) is a bijection of 64-bit words: `x ^= x >> 33` is its own inverse and the two multipliers
are odd.  So a wanted hash h has exactly one key unmix64(h), and the constructors below pick keys by their hash: ids that all
home at a table's last slot (their probe chains wrap to slot 0), and segments or edges whose hash is a chosen one.

The keys they return are never 0, 2^64-1 or repeated, and are below 2^63, so they are the same numbers as int64 and uint64.
"""
import numpy as np

M64 = (1 << 64) - 1
C1, C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53          # common.cuh mix64
C1_INV, C2_INV = pow(C1, -1, 1 << 64), pow(C2, -1, 1 << 64)
EK1, EK2 = 0x9E3779B97F4A7C15, 0x632BE59BD9B4E019        # edges.cu edge_hash
TAG_MASK = 0xFFFFFFFF00000000                            # what a SAGE slot keeps of a segment's hash
TWIN_SHIFT = 24   # twin k of hash h is h ^ (k << 24), k in [1, 256): the same tag, the same home in any table of <= 2^24 slots
PAIR_TWIN = 1 << (31 - TWIN_SHIFT)                       # twin(h, PAIR_TWIN) == h ^ 2^31


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def mix64(x):
    """common.cuh mix64 over a uint64 array"""
    k = _u64(x).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(C1)
        k ^= k >> np.uint64(33)
        k *= np.uint64(C2)
        k ^= k >> np.uint64(33)
    return k


def unmix64(h):
    """the key whose mix64 is h, over a uint64 array"""
    k = _u64(h).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(C2_INV)
        k ^= k >> np.uint64(33)
        k *= np.uint64(C1_INV)
        k ^= k >> np.uint64(33)
    return k


def mix64_int(k):
    k &= M64
    k ^= k >> 33
    k = (k * C1) & M64
    k ^= k >> 33
    k = (k * C2) & M64
    return k ^ (k >> 33)


def unmix64_int(h):
    h &= M64
    h ^= h >> 33
    h = (h * C2_INV) & M64
    h ^= h >> 33
    h = (h * C1_INV) & M64
    return h ^ (h >> 33)


def table_cap(n):
    """slots of a table for n keys: the smallest power of two >= max(2n, 64) (uq_table_cap, make_geom, fanout_aggregate,
    build_hash, eu_graph_set_edges)"""
    cap = 64
    while cap < 2 * n:
        cap <<= 1
    return cap


def segment_hash(ids):
    """k_sage_classify's chain hash h = mix64(h + id + 1) over a segment, from h = 0: one segment (1-D) or each row of a
    [R, count] array"""
    ids = np.atleast_2d(_u64(np.asarray(ids).astype(np.int64).view(np.uint64)))
    h = np.zeros(ids.shape[0], np.uint64)
    with np.errstate(over="ignore"):
        for j in range(ids.shape[1]):
            h = mix64(h + ids[:, j] + np.uint64(1))
    return h


def edge_hash(s, d, t):
    """edges.cu edge_hash: mix64(s * K1 ^ mix64(d + K2 * uint32(t)))"""
    s, d = _u64(np.asarray(s).astype(np.int64).view(np.uint64)), _u64(np.asarray(d).astype(np.int64).view(np.uint64))
    t = np.asarray(t).astype(np.int64).astype(np.uint32).astype(np.uint64)
    with np.errstate(over="ignore"):
        return mix64((s * np.uint64(EK1)) ^ mix64(d + np.uint64(EK2) * t))


def twin(h, k):
    """twin k of segment hash h: same tag, same home slot in every table of <= 2^TWIN_SHIFT slots"""
    return (int(h) ^ (int(k) << TWIN_SHIFT)) & M64


def _ok(key, taken):
    return 0 < key < (1 << 63) and key not in taken


def clustered_ids(k, low_bits, rs, taken=()):
    """k ids whose mix64 has its low `low_bits` bits all set: they home at the last slot of every table of <= 2^low_bits
    slots, so their chains wrap to slot 0 (and none is in `taken`)"""
    taken, out = set(int(x) for x in taken), []
    while len(out) < k:
        h = (int(rs.randint(0, 1 << 62)) << low_bits | ((1 << low_bits) - 1)) & M64
        key = unmix64_int(h)
        if _ok(key, taken):
            taken.add(key)
            out.append(key)
    return np.asarray(out, np.uint64)


def homed_ids(k, slot, bits, rs, taken=()):
    """k ids that home at `slot` of a table of 2^bits slots"""
    taken, out = set(int(x) for x in taken), []
    while len(out) < k:
        key = unmix64_int((int(rs.randint(0, 1 << 62)) << bits) | slot)
        if _ok(key, taken):
            taken.add(key)
            out.append(key)
    return np.asarray(out, np.uint64)


def tag_twin(prefix, h_target):
    """the last id that makes segment_hash(prefix + [id]) == h_target (None when that id is 0, 2^64-1 or >= 2^63)"""
    h_prev = int(segment_hash(np.asarray(prefix, np.int64).reshape(1, -1))[0]) if len(prefix) else 0
    key = (unmix64_int(int(h_target)) - h_prev - 1) & M64
    return key if _ok(key, ()) else None


def edge_twin(s, t, h_target):
    """the dst that makes edge_hash(s, dst, t) == h_target (None when that dst is 0, 2^64-1 or >= 2^63)"""
    x = unmix64_int(int(h_target)) ^ ((int(s) * EK1) & M64)
    key = (unmix64_int(x) - EK2 * (int(t) & 0xFFFFFFFF)) & M64
    return key if _ok(key, ()) else None


# ---------------------------------------------------------------------------------------------------- probe statistics
def linear_probe(homes, cap):
    """the slot each key lands in when distinct keys with these home slots are inserted in order into a linear-probing table
    of cap slots (the occupied set does not depend on the order)"""
    occupied = np.zeros(cap, bool)
    slots = np.empty(len(homes), np.int64)
    for i, h in enumerate(np.asarray(homes, np.int64)):
        s = int(h)
        while occupied[s]:
            s = (s + 1) & (cap - 1)
        occupied[s] = True
        slots[i] = s
    return slots


def chain_stats(homes, cap):
    """what keys with these home slots make of a linear-probing table of cap slots, whatever their insertion order:
    (wrapped: occupied slots from slot 0 on that continue a run through the last slot, i.e. keys whose chain wrapped;
    longest: the longest run of occupied slots, the longest chain a lookup can walk -- an absent key homed at its start
    walks it all and one empty slot more)"""
    occ = np.zeros(cap, bool)
    occ[linear_probe(homes, cap)] = True
    wrapped = int(np.argmin(occ)) if occ[-1] else 0
    run, best = 0, 0
    for s in range(2 * cap):   # twice around: a run through the last slot continues at slot 0
        run = run + 1 if occ[s & (cap - 1)] else 0
        best = max(best, min(run, cap))
    return wrapped, best


def run_end(homes, cap, start):
    """the first empty slot at or after `start` once keys with these homes are in the table"""
    occ = np.zeros(cap, bool)
    occ[linear_probe(homes, cap)] = True
    s = start
    while occ[s]:
        s = (s + 1) & (cap - 1)
    return s


def tag_pairs(hashes, cap):
    """distinct segment hashes that share a tag and a home slot in a table of cap slots, counted as pairs"""
    key = np.unique(np.asarray(hashes, np.uint64))
    grp = (key & np.uint64(TAG_MASK)) | (key & np.uint64(cap - 1))
    _, n = np.unique(grp, return_counts=True)
    return int((n * (n - 1) // 2).sum())
