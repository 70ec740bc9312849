"""tests/hash_reference.py against the device code, its constructors against their conditions, and the collisions each case of
tests/test_hash_collisions_gpu.py really contains: without them those tests would pass while testing nothing."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import collision_cases as cc
import graphs
import hash_reference as hr

CSRC = os.path.join(graphs.ROOT, "euler_b200", "csrc")


def _nvcc():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if p and os.path.exists(p):
            return p
    return None


def _homes(keys, cap):
    return (hr.mix64(np.unique(np.asarray(keys, np.int64).view(np.uint64))) & np.uint64(cap - 1)).astype(np.int64)


# ------------------------------------------------------------------------------------------------ the restatement
def test_unmix64_inverts_mix64():
    rs = np.random.RandomState(1)
    x = np.concatenate([np.asarray([0, 1, hr.M64], np.uint64), rs.randint(0, 1 << 63, size=5000, dtype=np.int64).view(np.uint64) * np.uint64(2) + np.uint64(1)])
    assert (hr.unmix64(hr.mix64(x)) == x).all() and (hr.mix64(hr.unmix64(x)) == x).all()
    for k in (0, 1, hr.M64, 0x0123456789ABCDEF):
        assert hr.unmix64_int(hr.mix64_int(k)) == k
        assert hr.mix64_int(k) == int(hr.mix64(np.asarray([k], np.uint64))[0])
    assert hr.mix64_int(0) == 0


def test_mix64_equals_the_device_header(tmp_path):
    """a host program built by nvcc against common.cuh hashes the same keys"""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "probe.cu"
    src.write_text('#include <stdio.h>\n#include "common.cuh"\n'
                   'int main() { unsigned long long k;\n'
                   '  while (scanf("%llx", &k) == 1) printf("%llx\\n", eu::mix64(k));\n  return 0; }\n')
    exe = tmp_path / "probe"
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src), "-o", str(exe)])
    rs = np.random.RandomState(2)
    keys = np.concatenate([np.asarray([0, 1, hr.M64, hr.M64 - 1, 1 << 63], np.uint64), rs.randint(0, 1 << 62, size=3000).astype(np.uint64) * np.uint64(4) + np.uint64(3),
                           cc.cluster().view(np.uint64)])
    out = subprocess.run([str(exe)], input="".join("%x\n" % int(k) for k in keys), capture_output=True, text=True, check=True).stdout
    got = np.asarray([int(v, 16) for v in out.split()], np.uint64)
    assert (got == hr.mix64(keys)).all()


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return re.sub(r"\s+", " ", f.read())


def test_segment_and_edge_hashes_are_the_device_expressions():
    """edge_hash and k_sage_classify's chain hash live inside .cu files no host program can link alone: hash_reference restates
    them, and this pins the expressions it restates (mix64 itself is pinned by the probe above)"""
    edges = _source("edges.cu")
    expr = "mix64(s * 0x9E3779B97F4A7C15ull ^ mix64(d + 0x632BE59BD9B4E019ull * (unsigned long long)(uint32_t)t))"
    assert edges.count(expr) == 2, "edge_hash and edge_hash_host"
    assert "unsigned long long h = edge_hash(s, d, (int32_t)t) & e.hmask;" in edges
    assert "unsigned long long h = edge_hash_host(d->src[r], d->dst[r], d->type[r]) & (cap - 1);" in edges
    mp = _source("mp_ops.cu")
    for line in ("unsigned long long h = 0;", "h = mix64(h + id + 1);", "const unsigned long long tag = h & 0xFFFFFFFF00000000ull;",
                 "unsigned long long p = h & mask;"):
        assert line in mp, line
    assert hr.TAG_MASK == 0xFFFFFFFF00000000
    # hand-computed chain: [5, 7] -> mix64(mix64(6) + 8)
    assert int(hr.segment_hash([5, 7])[0]) == hr.mix64_int(hr.mix64_int(6) + 8)


# ------------------------------------------------------------------------------------------------ constructors
def test_table_cap():
    assert [hr.table_cap(n) for n in (0, 1, 32, 33, 64, 65, 4096, 4097)] == [64, 64, 64, 128, 128, 256, 8192, 16384]


def test_constructors_meet_their_conditions():
    rs = np.random.RandomState(5)
    ids = hr.clustered_ids(300, 20, rs)
    assert len(set(ids.tolist())) == 300 and (ids > 0).all() and (ids < np.uint64(1 << 63)).all()
    for bits in (6, 13, 19, 20):
        assert (hr.mix64(ids) & np.uint64((1 << bits) - 1) == np.uint64((1 << bits) - 1)).all()
    h = hr.homed_ids(20, 77, 13, rs)
    assert (hr.mix64(h) & np.uint64(8191) == np.uint64(77)).all()
    prefix, s, t = [11, 22, 33], 123456789, 1
    made = 0
    for target in (int(x) * 3 for x in rs.randint(0, 1 << 62, size=40)):
        for pre in (prefix, []):
            last = hr.tag_twin(pre, target)
            if last is not None:   # None: the key would be >= 2^63
                made += 1
                assert 0 < last < 1 << 63 and int(hr.segment_hash(pre + [last])[0]) == target
        d = hr.edge_twin(s, t, target)
        if d is not None:
            made += 1
            assert 0 < d < 1 << 63 and int(hr.edge_hash([s], [d], [t])[0]) == target
    assert made >= 30
    assert hr.edge_hash([s], [d], [t + (1 << 32)])[0] == hr.edge_hash([s], [d], [t])[0], "the type hashes as uint32"
    a = int(hr.segment_hash([5, 9])[0])
    for k in (1, 7, hr.PAIR_TWIN):
        b = hr.twin(a, k)
        assert b != a and (a ^ b) & hr.TAG_MASK == 0 and (a ^ b) & ((1 << 24) - 1) == 0
    assert hr.twin(a, hr.PAIR_TWIN) == a ^ (1 << 31)


def test_case_keys_are_distinct_and_in_range():
    ids = cc._ids()[0]
    assert len(np.unique(ids)) == len(ids) - 1, "one repeated id"
    assert (ids < np.uint64(1 << 63)).all() and (ids == 0).sum() == 1
    assert not np.isin(cc.absent_cluster(), ids.view(np.int64)).any()
    for c in cc.SAGE_COUNTS:
        pool, groups, absent = cc.sage_pool(c)
        h = hr.segment_hash(pool)
        for grp in groups:
            assert len(set(h[grp].tolist())) == len(grp)
            assert len({int(x) & (hr.TAG_MASK | ((1 << 24) - 1)) for x in h[grp]}) == 1, "a group shares its tag and home"
            assert np.isin(pool[grp, -1], ids.view(np.int64)).all(), "every twin's last id is a node"
        assert not np.isin(pool[absent], ids.view(np.int64)).any()
    s, d, t, absent = cc.edge_case()
    assert not np.isin(absent[:, 1], d).any()


# ------------------------------------------------------------------------------------------------ what the GPU cases contain
def test_node_table_case():
    """2934 ids in 8192 slots: the cluster's run holds the last slot and slots 0-1327 (id 0, home slot 0, and the repeated id
    sit in it), so an absent id homed there walks 1329 slots"""
    ids = cc._ids()[0]
    cap = hr.table_cap(len(ids))
    wrapped, longest = hr.chain_stats(_homes(ids.view(np.int64), cap), cap)
    assert (cap, wrapped, longest) == (8192, 1328, 1329)
    q = cc.node_queries()
    assert (_homes(q[np.isin(q, cc.absent_cluster())], cap) == cap - 1).all()


def test_fanout_and_unique_cases():
    """the seed hops of the fanout cases wrap their dedup regions (table_cap(B) slots per batch); so do the unique inputs"""
    for B, want in ((3000, (993, 994)), (50_000, (1088, 1089)), (140_000, (1088, 1089))):
        seeds = cc.fanout_seeds(B, np.random.RandomState(B))
        cap = hr.table_cap(B)
        assert hr.chain_stats(_homes(seeds[seeds != -1], cap), cap) == want, B
        assert (seeds == -1).sum() > 0 and (seeds == 0).sum() > 0
    x = cc.unique_input(np.random.RandomState(3))
    assert len(x) == 75333 and hr.table_cap(len(x)) == 1 << 18
    for n, want in ((5000, (87, 88)), (len(x), (805, 806))):
        cap = hr.table_cap(n)
        assert hr.chain_stats(_homes(x[:n][x[:n] != -1], cap), cap) == want, n


@pytest.mark.parametrize("count", cc.SAGE_COUNTS)
def test_sage_case(count):
    """tag-equal pairs, wrapped chains and the longest chain of the distinct segments in the 2^19-slot table of a call of
    2^17 + 3000 rows; and the segments of the 2^17 + 555-row call that home where the 2^18 + 777-row call put them"""
    pool, groups, absent = cc.sage_pool(count)
    h = hr.segment_hash(np.delete(pool, absent, 0))
    cap = hr.table_cap(cc.SAGE_ROWS)
    assert cap == 1 << 19
    pairs = hr.tag_pairs(h, cap)
    wrapped, longest = hr.chain_stats((np.unique(h) & np.uint64(cap - 1)).astype(np.int64), cap)
    # 48 pairs, 8 chains of 3-8 twins and 6 chains of 2-4 at the last slot: 62 groups of 158 segments, 182 tag-equal pairs
    assert (len(groups), sum(map(len, groups)), pairs, wrapped, longest) == (62, 158, 182, 17, 18)
    big, small = hr.table_cap(cc.SAGE_ROWS_BIG), hr.table_cap(cc.SAGE_ROWS_SMALL)
    assert (big, small) == (1 << 20, 1 << 19)
    tw = hr.segment_hash(pool[[i for grp in groups for i in grp]])
    same = int(((tw & np.uint64(big - 1)) == (tw & np.uint64(small - 1))).sum())
    assert same == {1: 53, 2: 62, 10: 79, 25: 58}[count]


def test_edge_case():
    s, d, t, absent = cc.edge_case()
    cap = hr.table_cap(len(s))
    keys = np.unique(np.stack([s, d, t.astype(np.int64)], 1), axis=0)
    assert len(keys) == len(s) - 1, "one repeated triple"
    homes = (hr.edge_hash(keys[:, 0], keys[:, 1], keys[:, 2]) & np.uint64(cap - 1)).astype(np.int64)
    wrapped, longest = hr.chain_stats(homes, cap)
    assert (cap, wrapped, longest) == (4096, 389, 390)
    assert (hr.edge_hash(absent[:, 0], absent[:, 1], absent[:, 2]) & np.uint64(cap - 1) == np.uint64(cap - 1)).all()
