"""Argument validation of bf16 node features (sampler feature_dtype, merge_batches, GraphSignature.feat_dtype, pad_batch);
runs without a GPU."""
import types

import numpy as np
import pytest
import torch

from pyhgt_b200 import graphed, sampler

BF16 = torch.bfloat16


def test_sampler_feature_dtype_rules():
    """bf16 batches need a bf16 graph; other dtypes are refused.  Checked before any CUDA work."""
    g32 = types.SimpleNamespace(device="cuda:0", feature_dtype=torch.float32)
    g16 = types.SimpleNamespace(device="cuda:0", feature_dtype=BF16)
    for dt in (None, torch.float32):
        assert sampler._batch_feature_dtype(g32, dt) == torch.float32
        assert sampler._batch_feature_dtype(g16, dt) == torch.float32
    assert sampler._batch_feature_dtype(g16, BF16) == BF16
    with pytest.raises(ValueError, match="DeviceGraph built with feature_dtype=torch.bfloat16"):
        sampler.sample_subgraphs_cuda(g32, None, 2, 8, [{}], feature_dtype=BF16)
    with pytest.raises(ValueError, match="DeviceGraph built with feature_dtype=torch.bfloat16"):
        sampler.sample_subgraph_cuda(g32, None, 2, 8, {}, feature_dtype=BF16)
    for dt in (torch.float16, torch.float64, "bfloat16"):
        with pytest.raises(ValueError, match="feature_dtype must be"):
            sampler.sample_subgraphs_cuda(g16, None, 2, 8, [{}], feature_dtype=dt)


def _batch(dtype, n=3):
    return (torch.zeros(n, 4, dtype=dtype), torch.zeros(n, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
            torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64))


def test_merge_batches_refuses_mixed_and_unsupported_dtypes():
    with pytest.raises(ValueError, match="same dtype"):
        sampler.merge_batches([_batch(torch.float32), _batch(BF16)], 2, 1)
    with pytest.raises(ValueError, match="same dtype"):
        sampler.merge_batches([_batch(BF16), _batch(torch.float32)], 2, 1)
    for dt in (torch.float16, torch.float64):
        with pytest.raises(ValueError, match="float32 or bfloat16"):
            sampler.merge_batches([_batch(dt)], 2, 1)


def _sig(feat_dtype=torch.float32):
    return graphed.GraphSignature([4, 3], 10, [(0, 0), (1, 0)], 1, 5, feat_dtype=feat_dtype)


def test_graph_signature_feat_dtype():
    assert _sig().feat_dtype == torch.float32
    assert _sig(BF16).feat_dtype == BF16
    for dt in (torch.float16, torch.float64, "bfloat16", None):
        with pytest.raises(ValueError, match="feat_dtype"):
            _sig(dt)


def _host_batch(dtype):
    x = torch.arange(4 * 5, dtype=torch.float32).view(4, 5) / 7 - 1
    nt = torch.tensor([0, 0, 1, 1])
    ei = torch.tensor([[0, 2, 3], [1, 0, 2]])
    et = torch.zeros(3, dtype=torch.int64)
    tm = torch.tensor([100, 110, 120])
    return x.to(dtype), nt, tm, ei, et


def test_pad_batch_bf16_holds_the_bit_patterns():
    x16, nt, tm, ei, et = _host_batch(BF16)
    sig16, sig32 = _sig(BF16), _sig()
    p16 = graphed.pad_batch(sig16, x16, nt, tm, ei, et)
    p32 = graphed.pad_batch(sig32, x16.float(), nt, tm, ei, et)
    assert p16[0].dtype == np.int16 and p16[0].shape == p32[0].shape
    assert torch.equal(torch.from_numpy(p16[0]).view(BF16).float(), torch.from_numpy(p32[0]))
    for a, b in zip(p16[1:], p32[1:]):
        assert np.array_equal(a, b)
    out = (np.full((sig16.n_nodes, 5), 77, dtype=np.int16), np.empty(10, np.int64), np.empty((2, 10), np.int64),
           np.empty(10, np.int64))
    graphed.pad_batch(sig16, x16, nt, tm, ei, et, out=out)
    assert np.array_equal(out[0], p16[0])


def test_pad_batch_refuses_a_dtype_other_than_the_signatures():
    x16, nt, tm, ei, et = _host_batch(BF16)
    with pytest.raises(ValueError, match="feat_dtype"):
        graphed.pad_batch(_sig(), x16, nt, tm, ei, et)
    with pytest.raises(ValueError, match="feat_dtype"):
        graphed.pad_batch(_sig(BF16), x16.float(), nt, tm, ei, et)
    with pytest.raises(ValueError, match="feat_dtype"):
        graphed.pad_batch(_sig(), x16.double(), nt, tm, ei, et)
