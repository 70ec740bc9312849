"""The inputs of tests/test_hash_collisions_gpu.py, built from tests/hash_reference.py's constructors so that every device
hash table meets keys that collide on purpose.  Deterministic and GPU-free: tests/test_hash_collisions_cpu.py counts the
collisions each case contains.  (Test infrastructure.)

The graph (collision_graph) has 2934 nodes, so its id table has 8192 slots, and its ids are:
    CLUSTER        1024 ids that home at the last slot of every table of <= 2^20 slots: one chain that wraps to slot 0 in
                   the id table, in every fanout dedup region and in every first-occurrence table of this file
    0              homes at slot 0 (mix64(0) == 0), inside the wrapped chain
    DUP            CLUSTER[500] listed again as the last row: the later row is the node
    twins          for each SAGE count, the last ids of segments whose hashes share a tag and a home slot (sage_pool)
    the rest       random ids below 2^63
Neighbours are cluster ids 60% of the time, so every hop of a fanout probes the wrapped chain.
"""
import functools

import numpy as np

import hash_reference as hr

CLUSTER_BITS = 20
N_BASE, N_CLUSTER, N_ABSENT_CLUSTER = 1500, 1024, 64
DUP_OF = 500
SAGE_COUNTS = (1, 2, 10, 25)
N_PAIRS, CHAIN_LENGTHS, N_LAST_SLOT = 48, (3, 4, 5, 6, 7, 8, 3, 8), 6
SAGE_ROWS = (1 << 17) + 3000          # one call past 2^17 rows: the segment table's path
SAGE_ROWS_BIG = (1 << 18) + 777       # and the two calls of the table-cleanliness case
SAGE_ROWS_SMALL = (1 << 17) + 555


@functools.lru_cache(maxsize=None)
def _ids():
    rs = np.random.RandomState(2024)
    cl = hr.clustered_ids(N_CLUSTER + N_ABSENT_CLUSTER, CLUSTER_BITS, rs)
    cluster, absent_cluster = cl[:N_CLUSTER], cl[N_CLUSTER:]
    taken = set(int(x) for x in cl)
    base = []
    while len(base) < N_BASE:
        k = int(rs.randint(1, 1 << 62)) * 2 + 1
        if k not in taken:
            taken.add(k)
            base.append(k)
    base = np.asarray(base, np.uint64)
    families = {c: _sage_family(c, np.concatenate([base, cluster]), taken, np.random.RandomState(77 + c)) for c in SAGE_COUNTS}
    twins = np.asarray([k for c in SAGE_COUNTS for k in families[c][1]], np.uint64)
    ids = np.concatenate([base, cluster, np.zeros(1, np.uint64), twins, cluster[DUP_OF:DUP_OF + 1]])
    return ids, cluster, absent_cluster, families


def _sage_family(c, pool, taken, rs):
    """segments of `count` c whose hashes collide: (segments, their new last ids, groups of segment indices that share a tag
    and a home slot).  Pairs A, B = twin(A, 2^31); chains A, twin(A, 1), .., twin(A, L - 1); and short chains whose hashes
    have their low 24 bits set (the last slot of every segment table these tests size)."""
    segs, new, groups = [], [], []

    def member(prefix, h):
        k = hr.tag_twin(prefix, h)
        return None if k is None or k in taken else k

    def chain(L, last_slot):
        while True:
            prefix = [int(x) for x in pool[rs.randint(0, len(pool), size=c - 1)]]
            if last_slot:
                hA = (int(rs.randint(0, 1 << 40)) << hr.TWIN_SHIFT) | ((1 << hr.TWIN_SHIFT) - 1)
                first = [member(prefix, hA)]
            else:
                a = int(pool[rs.randint(0, len(pool))])
                hA, first = int(hr.segment_hash(np.asarray(prefix + [a], np.uint64).view(np.int64))[0]), []
            ks = [hr.PAIR_TWIN] if L == 2 and not last_slot else list(range(1, L))
            last = first + [member(prefix, hr.twin(hA, k)) for k in ks]
            if all(k is not None for k in last) and len(set(last)) == len(last):
                break
        taken.update(last)
        new.extend(last)
        if not last_slot:
            last = [a] + last
        groups.append(list(range(len(segs), len(segs) + len(last))))
        segs.extend(prefix + [k] for k in last)

    for _ in range(N_PAIRS):
        chain(2, False)
    for L in CHAIN_LENGTHS:
        chain(L, False)
    for L in (2, 3, 4, 2, 3, 4)[:N_LAST_SLOT]:
        chain(L, True)
    return np.asarray(segs, np.uint64).view(np.int64).reshape(-1, c), new, groups


def cluster():
    return _ids()[1].view(np.int64)


def absent_cluster():
    """ids not in the graph that home where the cluster does"""
    return _ids()[2].view(np.int64)


@functools.lru_cache(maxsize=None)
def collision_graph(feat_dim=0, T=2, seed=5):
    """the graph as numpy CSR (the layout of tests/graphs.py); features over 16 binades, so sums round differently in
    different orders"""
    from graphs import po
    ids = _ids()[0]
    n = len(ids)
    rs = np.random.RandomState(seed)
    deg = rs.poisson(4, size=(n, T))
    deg[rs.rand(n, T) < 0.1] = 0
    grp_ptr = np.zeros(n * T + 1, np.int64)
    grp_ptr[1:] = np.cumsum(deg.reshape(-1))
    E = int(grp_ptr[-1])
    cl = _ids()[1]
    nbr = np.where(rs.rand(E) < 0.6, cl[rs.randint(0, len(cl), size=E)], ids[rs.randint(0, n, size=E)]).astype(np.uint64)
    w = (1 + rs.randint(0, 100, size=E)).astype(np.float32) / np.float32(10)
    cum_w, grp_cum = po.build_cum(grp_ptr, w, n, T)
    feat = None
    if feat_dim:
        feat = (rs.uniform(-1, 1, (n, feat_dim)) * np.exp2(rs.randint(-8, 8, size=(n, feat_dim)))).astype(np.float32)
    return dict(ids=ids, node_type=rs.randint(0, 3, size=n).astype(np.int32),
                node_w=(1 + rs.randint(0, 50, size=n)).astype(np.float32) / np.float32(4), T=T, grp_ptr=grp_ptr, nbr=nbr,
                w=w, cum_w=cum_w, grp_cum=grp_cum, feat=feat, n_node_types=3)


def row_of_id():
    """id -> row as a dict: a later row of a repeated id replaces the earlier one"""
    return {int(k): r for r, k in enumerate(_ids()[0])}


def node_queries():
    """every cluster id, the repeated id, 0, -1, absent ids homed at the cluster's slot and just past the end of its run, and
    random present and absent ids"""
    ids, cl, acl, _ = _ids()
    rs = np.random.RandomState(8)
    cap = hr.table_cap(len(ids))
    end = hr.run_end(hr.mix64(np.unique(ids)) & np.uint64(cap - 1), cap, cap - 1)
    taken = set(int(x) for x in ids)
    past = np.concatenate([hr.homed_ids(4, (end + d) % cap, cap.bit_length() - 1, rs, taken) for d in (-2, -1, 0, 1, 2)])
    q = np.concatenate([cl, cl[DUP_OF:DUP_OF + 1], np.asarray([0, hr.M64], np.uint64), acl, past,
                        ids[rs.randint(0, len(ids), size=300)], hr.homed_ids(50, 3, 8, rs, taken)])
    return q[rs.permutation(len(q))].view(np.int64)


def fanout_seeds(n, rs):
    """n seeds from the cluster (many repeated), with the repeated id, 0, -1 and absent cluster-homed ids among them"""
    cl = cluster()
    s = cl[rs.randint(0, len(cl), size=n)]
    s[::97] = cl[DUP_OF]
    s[1::101] = 0
    s[2::89] = -1
    s[3::83] = absent_cluster()[rs.randint(0, N_ABSENT_CLUSTER, size=len(s[3::83]))]
    return s


def unique_input(rs):
    """cluster ids in runs of 1-700 equal ids (across warp and CTA boundaries), with 0 and -1 runs among them"""
    cl = np.concatenate([cluster(), absent_cluster(), [0, -1]])
    vals = cl[rs.randint(0, len(cl), size=1500)]
    vals[::50] = 0
    vals[25::50] = -1
    reps = rs.choice([1, 2, 3, 31, 33, 64, 255, 257, 700], size=len(vals), p=[.3, .2, .1, .1, .1, .08, .06, .04, .02])
    return np.repeat(vals, reps).astype(np.int64)


def sage_pool(count):
    """the distinct segments of a SAGE call: (pool [P, count] i64, groups of pool rows that share a tag and a home slot,
    rows whose ids are all absent)"""
    _, cl, acl, fam = _ids()
    segs, _, groups = fam[count]
    rs = np.random.RandomState(300 + count)
    ids = _ids()[0].view(np.int64)
    rnd = ids[rs.randint(0, len(ids), size=(200, count))]
    clu = cl.view(np.int64)[rs.randint(0, len(cl), size=(100, count))]
    absent = np.where(rs.rand(20, count) < 0.5, -1, acl.view(np.int64)[rs.randint(0, len(acl), size=(20, count))])
    pool = np.concatenate([segs, rnd, clu, absent])
    return pool, groups, np.arange(len(pool) - len(absent), len(pool))


def sage_rows(count, rows, seed):
    """[rows] indices into sage_pool(count): every pool row once, then repeats of all of them, shuffled"""
    P = len(sage_pool(count)[0])
    rs = np.random.RandomState(seed)
    idx = np.concatenate([np.arange(P), rs.randint(0, P, size=rows - P)])
    return idx[rs.permutation(rows)]


@functools.lru_cache(maxsize=None)
def edge_case():
    """edges (src, dst, type) of types 0 and 1 on the graph's ids: random ones, a cluster of 300 whose hashes home at the last
    slot of every table of <= 2^20 slots, and the first cluster edge again as the last row (the first row is the edge).
    Returns (src, dst, type, absent cluster-homed triples [50, 3])."""
    ids = _ids()[0]
    rs = np.random.RandomState(99)
    n_rand, n_cl = 1000, 300
    src = list(ids[rs.randint(0, len(ids), size=n_rand)])
    dst = list(ids[rs.randint(0, len(ids), size=n_rand)])
    typ = list(rs.randint(0, 2, size=n_rand))
    made = []
    while len(made) < n_cl + 50:
        s, t = int(ids[rs.randint(0, len(ids))]), int(rs.randint(0, 2))
        d = hr.edge_twin(s, t, (int(rs.randint(0, 1 << 40)) << CLUSTER_BITS) | ((1 << CLUSTER_BITS) - 1))
        if d is not None:
            made.append((s, d, t))
    for s, d, t in made[:n_cl] + made[:1]:
        src.append(s), dst.append(d), typ.append(t)
    return (np.asarray(src, np.uint64).view(np.int64), np.asarray(dst, np.uint64).view(np.int64), np.asarray(typ, np.int32),
            np.asarray(made[n_cl:], np.int64))
