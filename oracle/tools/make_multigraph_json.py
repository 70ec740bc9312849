#!/usr/bin/env python
"""TEST INFRASTRUCTURE.  Writes the Euler JSON of the multi-graph fixture (tests/golden/multigraph_euler, converted by
oracle/tools/make_multigraph_fixture.sh with the reference's own converter).

40 small graphs laid out as tf_euler/python/dataset/multigraph_util.py:68-100 lays out graph-classification data: every node
has a sparse `f1` (its node label, also its node type), a dense `label` (its graph's class) and a binary `graph_label` (its
graph's index as a string); edges have type 0 and weight 1.  Graph sizes are 1-120 nodes plus one of 300 (above the 256 rows
of a readout chunk); each graph is a ring (both directions) with a few chords.  Five nodes carry no `graph_label`, so the
reference's label list holds "" as well.  Deterministic: numpy RandomState(20261016).

    python oracle/tools/make_multigraph_json.py OUT.json"""
import json
import sys

import numpy as np


def main(out):
    rs = np.random.RandomState(20261016)
    sizes = [int(s) for s in rs.randint(1, 121, size=39)] + [300]
    rs.shuffle(sizes)
    n = sum(sizes)
    unlabelled = set(int(i) for i in rs.choice(n, size=5, replace=False) + 1)
    nodes, edges, nid = [], [], 1
    for k, s in enumerate(sizes):
        ids = list(range(nid, nid + s))
        nid += s
        cls = k % 2
        for v in ids:
            f1 = int(rs.randint(0, 3))
            feats = [{"name": "f1", "type": "sparse", "value": [f1]},
                     {"name": "label", "type": "dense", "value": [float(cls)]}]
            if v not in unlabelled:
                feats.append({"name": "graph_label", "type": "binary", "value": str(k)})
            nodes.append({"id": v, "type": f1, "weight": 1.0, "features": feats})
        pairs = set()
        if s > 1:
            for i in range(s):
                pairs.add((ids[i], ids[(i + 1) % s]))
                pairs.add((ids[(i + 1) % s], ids[i]))
            for _ in range(s // 5):
                a, b = rs.randint(0, s, size=2)
                if a != b:
                    pairs.add((ids[a], ids[b]))
                    pairs.add((ids[b], ids[a]))
        for a, b in sorted(pairs):
            edges.append({"src": a, "dst": b, "type": 0, "weight": 1.0, "features": []})
    with open(out, "w") as f:
        json.dump({"nodes": nodes, "edges": edges}, f)


if __name__ == "__main__":
    main(sys.argv[1])
