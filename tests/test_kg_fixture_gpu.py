"""GPU: the knowledge-graph fixture tests/golden/kg_euler -- the JSON of oracle/tools/make_kg_json.py (laid out as
fb15k.py:convert2json lays out FB15k) converted by the reference's own converter -- loaded as FB15k users load it: the 'id'
edge feature gives the relation ids, sample_node('train') draws train-typed entities only, and a TransE step on it matches
the composition."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "kg_euler")


@pytest.fixture(scope="module")
def kg():
    """(graph, the fixture's JSON)"""
    import euler_b200
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "kg.json")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "tools", "make_kg_json.py"), out])
        with open(out) as f:
            js = json.load(f)
    g = euler_b200.Graph.load(FIXTURE)
    euler_b200.set_graph(g, rng="minstd", seed=5)
    return g, js


def test_shape_and_relation_ids(kg):
    import euler_b200
    g, js = kg
    assert g.num_nodes == len(js["nodes"]) and g.num_edge_records == len(js["edges"])
    types = {name: g.edge_type_id(name) for name in ("train", "test", "valid")}
    assert sorted(types.values()) == [0, 1, 2]
    edges = [[e["src"], e["dst"], types[e["type"]]] for e in js["edges"]]
    want = np.array([e["features"][0]["value"][0] for e in js["edges"]], np.float32)
    got = euler_b200.get_edge_dense_feature(torch.tensor(edges, dtype=torch.int64), ['id'], [1])[0]
    assert np.array_equal(got.cpu().numpy().reshape(-1), want)
    assert int(want.max()) == 6 and len(set(want.tolist())) == 7


def test_sample_node_train_draws_train_entities_only(kg):
    import euler_b200
    _, js = kg
    train = {n["id"] for n in js["nodes"] if n["type"] == "train"}
    assert len(train) < len(js["nodes"])
    drawn = set(euler_b200.sample_node(4000, 'train').cpu().tolist())
    assert drawn <= train and len(drawn) > len(train) // 2


def test_transe_step_matches_composed(kg):
    """sample_edge('train') -> 'id' -> sample_node('train') -> loss -> backward -> SGD, fused against fused=False"""
    import euler_b200
    from euler_b200 import knowledge
    _, js = kg
    node_max_id = max(n["id"] for n in js["nodes"])
    edge_max_id = int(max(e["features"][0]["value"][0] for e in js["edges"]))
    torch.manual_seed(0)
    kw = dict(num_negs=3, margin=1.0, corrupt='both', device='cuda')
    fused = knowledge.TransE('train', 'train', node_max_id, edge_max_id, 16, 16, **kw)
    composed = knowledge.TransE('train', 'train', node_max_id, edge_max_id, 16, 16, fused=False, **kw)
    composed.load_state_dict(fused.state_dict())
    edges = euler_b200.sample_edge(48, 'train')
    outs = []
    for mdl in (fused, composed):
        euler_b200.seed(11)
        opt = torch.optim.SGD(mdl.parameters(), lr=0.5)
        out = mdl(edges)
        opt.zero_grad()
        out.loss.backward()
        opt.step()
        outs.append(out)
    assert abs(float(outs[0].loss) - float(outs[1].loss)) <= 1e-5 * max(1.0, abs(float(outs[1].loss)))
    assert abs(float(outs[0].metric) - float(outs[1].metric)) <= 1e-5
    for (n, p), (_, q) in zip(fused.named_parameters(), composed.named_parameters()):
        assert float((p - q).abs().max()) <= 1e-5 * max(1.0, float(q.abs().max())), n
