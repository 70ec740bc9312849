#!/usr/bin/env python
"""TEST INFRASTRUCTURE.  Writes the Euler JSON of the knowledge-graph fixture (tests/golden/kg_euler, converted by
oracle/tools/make_kg_fixture.sh with the reference's own converter).

A small FB15k-like set of named triples -- 60 entities, 7 relations, 300 triples split 240 / 30 / 30 into train, test and
valid -- laid out exactly as tf_euler/python/dataset/fb15k.py:convert2json lays out FB15k: the files are read in the order
train, test, valid; an entity gets the next id and, as its node type, the file it first appears in; a relation gets the next
id on first appearance; each triple is an edge (head, tail) of the file's type, weight 1, with the dense feature 'id' = the
relation id.  Relation frequencies are Zipf-like and some entities first appear in test or valid, so all three node types
exist.  Each (head, tail) pair occurs once: Euler keys an edge by (src, dst, type), so every edge's 'id' is unambiguous.  Deterministic: numpy RandomState(20261017).

    python oracle/tools/make_kg_json.py OUT.json"""
import json
import sys

import numpy as np


def triples():
    """{file: [(head, relation, tail)]} of entity and relation names"""
    rs = np.random.RandomState(20261017)
    ents = ["/m/e%02d" % i for i in range(60)]
    rels = ["/r/%s" % n for n in ("born_in", "works_for", "capital_of", "member_of", "located_in", "spouse", "genre")]
    p = 1.0 / np.arange(1, len(rels) + 1) ** 1.1
    seen, out = set(), {}
    for name, n, pool in (("train", 240, ents[:50]), ("test", 30, ents), ("valid", 30, ents)):
        rows = []
        while len(rows) < n:
            h, t = rs.choice(len(pool), size=2, replace=False)
            r = rels[rs.choice(len(rels), p=p / p.sum())]
            if (pool[h], pool[t]) not in seen:
                seen.add((pool[h], pool[t]))
                rows.append((pool[h], r, pool[t]))
        out[name] = rows
    return out


def main(out):
    tri = triples()
    nodes, edges, entity, relation = [], [], {}, {}
    for file_type in ("train", "test", "valid"):
        for h, r, t in tri[file_type]:
            for e in (h, t):
                if e not in entity:
                    entity[e] = len(entity)
                    nodes.append({"id": entity[e], "type": file_type, "weight": 1, "features": []})
            if r not in relation:
                relation[r] = len(relation)
            edges.append({"src": entity[h], "dst": entity[t], "type": file_type, "weight": 1,
                          "features": [{"name": "id", "type": "dense", "value": [relation[r]]}]})
    with open(out, "w") as f:
        json.dump({"nodes": nodes, "edges": edges}, f)


if __name__ == "__main__":
    main(sys.argv[1])
