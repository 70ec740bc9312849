"""bfloat16 outputs of the graph-feature ops without a GPU: the Python refusals of an output dtype other than f32 / bf16
(before the library is loaded and before any device is touched), the f32 defaults, and the numpy restatement of the
output rounding on special values."""
import inspect

import numpy as np
import pytest
import torch

import bf16_reference as br


@pytest.fixture
def no_library(monkeypatch):
    """every path into the library or onto a device fails loudly"""
    from euler_b200 import _lib, ops

    def refuse(*a, **k):
        raise AssertionError("the library or a device was reached")
    monkeypatch.setattr(_lib, "load", refuse)
    monkeypatch.setattr(ops, "_call", refuse)
    monkeypatch.setattr(ops, "_t", refuse)
    monkeypatch.setattr(ops, "get_graph", refuse)
    monkeypatch.setattr(ops, "_ctx_on_stream", refuse)
    return ops


CALLS = {
    "get_dense_feature": lambda ops, dt: ops.get_dense_feature([1, 2], [0], [4], out_dtype=dt),
    "sage_mean_aggregate": lambda ops, dt: ops.sage_mean_aggregate([1, 2], 2, 4, out_dtype=dt),
    "neighbor_top_k_feature": lambda ops, dt: ops.neighbor_top_k_feature([1], [[1, 2]], 0, 4, 1, out_dtype=dt),
    "sample_fanout_with_feature": lambda ops, dt: ops.sample_fanout_with_feature([1], [[0]], [2], -1, [0], [4], [], [],
                                                                                 dense_dtype=dt),
}


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64, torch.int32, torch.int64, "bfloat16", None])
@pytest.mark.parametrize("op", sorted(CALLS))
def test_other_output_dtypes_are_refused_before_the_library(no_library, op, dtype):
    from euler_b200 import EulerError
    with pytest.raises(EulerError, match="%s: the output dtype must be torch.float32 or torch.bfloat16" % op):
        CALLS[op](no_library, dtype)


@pytest.mark.parametrize("op,kw", [("get_dense_feature", "out_dtype"), ("sage_mean_aggregate", "out_dtype"),
                                   ("neighbor_top_k_feature", "out_dtype"), ("sample_fanout_with_feature", "dense_dtype")])
def test_outputs_default_to_float32(op, kw):
    import euler_b200
    from euler_b200 import ops
    assert inspect.signature(getattr(ops, op)).parameters[kw].default is torch.float32
    assert getattr(euler_b200, op) is getattr(ops, op)


def test_output_dtypes_are_the_feature_dtype_codes():
    from euler_b200 import _lib
    assert _lib.TORCH_DTYPES == {torch.float32: 0, torch.bfloat16: 1}
    for name in ("eu_get_dense_feature", "eu_get_dense_feature_host", "eu_sage_mean_aggregate", "eu_sage_mean_aggregate_host",
                 "eu_sage_add_aggregate", "eu_neighbor_top_k_feature"):
        f32, twin = _lib.SIGNATURES[name][1], _lib.SIGNATURES[name + "_out_dtype"][1]
        assert twin[:-1] == f32[:-1] + [_lib._I32] and twin[-1] == f32[-1]   # (..., int32_t out_dtype, void* out)
    f32, twin = _lib.SIGNATURES["eu_sample_fanout_with_feature"][1], _lib.SIGNATURES["eu_sample_fanout_with_feature_out_dtype"][1]
    assert twin == f32[:15] + [_lib._I32] + f32[15:]   # dense_dtype before out_dense


def test_restated_rounding_on_special_values():
    """the output contract: round to nearest even, NaN to a canonical NaN, +-Inf kept, overflow to +-Inf only where the
    rounding says so, subnormals rounded like any other value -- the numpy restatement against torch's host conversion"""
    sp = br.special_values()
    x = np.concatenate([sp, -sp])
    got = br.round_bits(x)
    want = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    nan = np.isnan(x)          # torch's host NaN need not be the restatement's: compared as NaN-ness
    assert np.array_equal(got[~nan], want[~nan])
    assert np.isnan(br.widen(want[nan])).all() and np.isnan(br.widen(got[nan])).all()
    b = dict(zip(x.view(np.uint32).tolist(), got.tolist()))
    assert b[0x7F7FFFFF] == 0x7F80 and b[0xFF7FFFFF] == 0xFF80          # the largest normals round up to +-Inf
    assert b[0x7F7F7FFF] == 0x7F7F and b[0x7F7F8000] == 0x7F80          # below the last tie stays finite; the tie goes to even
    assert b[0x3F808000] == 0x3F80 and b[0x3F818000] == 0x3F82          # ties to even, both parities
    assert b[0x00008000] == 0x0000 and b[0x00018000] == 0x0002          # subnormal ties round like normal ones
    assert b[0x007FFFFF] == 0x0080                                       # the largest subnormal rounds to the smallest normal
    assert b[0x7F800000] == 0x7F80 and b[0xFF800000] == 0xFF80
    assert all(b[u] == br.CANONICAL_NAN for u in (0x7FC00000, 0xFFC00001, 0x7F800001, 0xFF80ABCD, 0x7FBFFFFF))
    assert np.array_equal(br.widen(got)[~np.isnan(x)], br.rounded(x)[~np.isnan(x)])
