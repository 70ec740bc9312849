"""CPU: the closed forms of the skip-gram step (rank, cross-entropy, metrics) against literal restatements of the reference,
the torch composition of the unfused path on CPU tensors, and the sample shapes of the model classes."""
import numpy as np
import pytest
import torch

import skipgram_reference as sr


def _tied_logits(rng, B, J):
    """small integers: many ties, the last positive among them"""
    return rng.randint(-3, 4, size=(B, J)).astype(np.float32)


@pytest.mark.parametrize("P,K", [(1, 0), (1, 1), (1, 5), (3, 0), (3, 5), (2, 20)])
def test_rank_closed_form_is_stable_top_k(P, K):
    rng = np.random.RandomState(P * 100 + K)
    x = _tied_logits(rng, 300, P + K)
    want = sr.rank_top_k_literal(x[:, :P], x[:, P:])
    assert np.array_equal(sr.rank_closed_form(x, P), want)
    assert (want > 0).any() or K == 0 and P == 1


def test_rank_of_all_ties_is_last():
    x = np.zeros((4, 6), np.float32)
    assert np.array_equal(sr.rank_closed_form(x, 1), [5] * 4)
    assert np.array_equal(sr.rank_top_k_literal(x[:, :1], x[:, 1:]), [5] * 4)


@pytest.mark.parametrize("name", ["mrr", "hit1", "hit3", "hit10", "mr"])
def test_skipgram_metric_matches_the_restatement(name):
    from euler_b200.ops import skipgram_metric
    rng = np.random.RandomState(5)
    rank = rng.randint(0, 21, size=997)
    got = skipgram_metric(torch.as_tensor(rank, dtype=torch.int32), name)
    want = sr.metric(rank, name)
    if name == 'mr':
        assert got.dtype == torch.int64 and int(got) == want
    else:
        assert abs(float(got) - float(want)) <= 1e-6 * abs(float(want))


def test_mr_is_an_integer_mean():
    """tf.reduce_mean over int64 ranks divides in integers: 1, 2 -> 1, not 1.5"""
    from euler_b200.ops import skipgram_metric
    assert int(skipgram_metric(torch.tensor([1, 2], dtype=torch.int32), 'mr')) == 1
    assert sr.metric([1, 2], 'mr') == 1
    assert sr.metric([0, 0, 2], 'mr') == 0


def test_xent_formula():
    x = np.array([-50, -3.5, -1, 0, 0.25, 2, 40], np.float64)
    for z in (0.0, 1.0):
        p = 1 / (1 + np.exp(-x))
        with np.errstate(divide='ignore', invalid='ignore'):
            direct = -(z * np.log(p) + (1 - z) * np.log1p(-p))
        ok = np.isfinite(direct)
        assert np.allclose(sr.xent64(x, z)[ok], direct[ok], rtol=1e-12, atol=1e-15)
    assert sr.xent64(np.array([-1000.0]), 1.0)[0] == 1000.0   # the stable form never overflows


@pytest.mark.parametrize("P,K", [(1, 0), (1, 5), (3, 20)])
@pytest.mark.parametrize("name", ["mrr", "hit3", "mr"])
def test_composition_on_the_cpu(P, K, name):
    """unsupervised.composed_skipgram_loss (the fused=False path) restates PosNegLogits + xent_loss + the metric"""
    from euler_b200.unsupervised import composed_skipgram_loss
    rng = np.random.RandomState(P + K)
    B, dim = 64, 8
    tb = rng.randint(-2, 3, size=(30, dim)).astype(np.float64) / 4
    src = rng.randint(0, 30, size=B)
    ctx = rng.randint(0, 30, size=(B, P + K))
    T = torch.tensor(tb, requires_grad=True)
    loss, met = composed_skipgram_loss(T[src][:, None, :], T[ctx[:, :P]], T[ctx[:, P:]], name)
    x, want = sr.forward64(tb, tb, src, ctx, P)
    assert abs(float(loss.detach()) - want) <= 1e-12 * want
    got_m = met.item()
    want_m = sr.metric(sr.rank_closed_form(x, P), name)
    assert got_m == want_m if name == 'mr' else abs(got_m - float(want_m)) <= 1e-6
    loss.backward()
    gt, gc = sr.grads64(tb, tb, src, ctx, P)
    assert np.allclose(T.grad.numpy(), gt + gc, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("walk_len,left,right", [(3, 1, 1), (80, 1, 1), (10, 2, 3), (1, 1, 1)])
def test_model_sample_shapes(walk_len, left, right):
    from euler_b200 import unsupervised as un
    ratio = sr.gen_pair_count(walk_len + 1, left, right)
    assert un.pairs_per_walk(walk_len, left, right) == ratio
    m = un.DeepWalk(0, [0], 99, 8, walk_len=walk_len, left_win_size=left, right_win_size=right, num_negs=5)
    assert m.sample_shapes(7) == ((7 * ratio, 1), (7 * ratio, 1), (7 * ratio, 5))
    line = un.Line(0, [0], 99, 8, num_negs=3, order=2)
    assert line.sample_shapes(7) == ((7, 1), (7, 1), (7, 3))


def test_model_tables_and_orders():
    from euler_b200 import unsupervised as un
    m = un.Line(0, [0], 99, 16, order=1)
    assert m.context_encoder is m.target_encoder
    assert tuple(m.target_encoder.embeddings.shape) == (101, 16)   # ShallowEncoder: Embedding(max_id + 1) -> max_id + 2 rows
    w = m.target_encoder.embeddings.detach()
    assert float(w.abs().max()) <= 0.2 and 0.05 < float(w.std()) < 0.1   # truncated normal, stddev 0.1, cut at 2 stddev
    m2 = un.Line(0, [0], 99, 16, order='second')
    assert m2.context_encoder is not m2.target_encoder
    with pytest.raises(ValueError):
        un.Line(0, [0], 99, 16, order=3)
