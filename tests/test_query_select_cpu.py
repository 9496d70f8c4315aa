"""The host check of the top-k override (b200.capi.check_topk_override) that Engine.forward and Engine.forward_frames run
before handing the tensor to the engine, which gathers encoder rows, class logits and proposals at its indices unchecked.
On CPU tensors with a CPU "engine device"; no engine is involved.  Also the numpy helpers of test_query_select_gpu."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "lw-detr_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from b200.capi import check_topk_override  # noqa: E402

CPU = torch.device("cpu")
B, NQ, S = 2, 100, 1600


def _ov(dtype=torch.int32):
    return (torch.arange(B * NQ) * 7 % S).reshape(B, NQ).to(dtype)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64, torch.int16])
def test_accepts_any_integer_tensor_and_returns_int32(dtype):
    ov = _ov(dtype)
    ov[0, 3] = ov[0, 4]                    # duplicates are a legal selection
    ov[0, 0], ov[1, -1] = 0, S - 1         # both ends of [0, S)
    out = check_topk_override(ov, B, NQ, S, CPU)
    assert out.dtype == torch.int32 and out.is_contiguous()
    assert torch.equal(out.long(), ov.long())


def test_accepts_non_contiguous_view():
    full = torch.zeros(B, 2 * NQ, dtype=torch.int64)
    full[:, ::2] = _ov(torch.int64)
    out = check_topk_override(full[:, ::2], B, NQ, S, CPU)
    assert out.is_contiguous() and torch.equal(out.long(), _ov(torch.int64))


@pytest.mark.parametrize("shape", [(B, NQ - 1), (B + 1, NQ), (B * NQ,), (B, NQ, 1), (1, NQ)])
def test_refuses_wrong_shape(shape):
    ov = torch.zeros(shape, dtype=torch.int32)
    with pytest.raises(RuntimeError, match=r"\[B, num_queries\] = \[%d, %d\]" % (B, NQ)):
        check_topk_override(ov, B, NQ, S, CPU)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.float64, torch.bool])
def test_refuses_non_integer(dtype):
    with pytest.raises(RuntimeError, match="integer tensor"):
        check_topk_override(_ov().to(dtype), B, NQ, S, CPU)


@pytest.mark.parametrize("engine_device", [torch.device("cuda", 0), CPU])
def test_refuses_a_device_other_than_the_host_and_the_engines(engine_device):
    """A host tensor is copied to the engine's device (the oracle's indices are host tensors); a tensor on any other device
    is refused before anything reads it.  The meta device stands in for "another device" without needing one."""
    ov = torch.zeros(B, NQ, dtype=torch.int32, device="meta")
    with pytest.raises(RuntimeError, match="engine lives on %s" % engine_device):
        check_topk_override(ov, B, NQ, S, engine_device)


@pytest.mark.parametrize("bad", [-1, S, S + 5, -(2 ** 40), 2 ** 40])
def test_refuses_index_outside_memory(bad):
    ov = _ov(torch.int64)
    ov[1, 37] = bad
    with pytest.raises(RuntimeError, match=r"\[0, %d\)" % S):
        check_topk_override(ov, B, NQ, S, CPU)


def test_limit_is_the_plans_memory_length():
    """S - 1 passes at S and fails one token shorter: the bound is the memory length handed in, not a constant."""
    ov = _ov()
    ov[0, 1] = S - 1
    check_topk_override(ov, B, NQ, S, CPU)
    with pytest.raises(RuntimeError, match=r"\[0, %d\)" % (S - 1)):
        check_topk_override(ov, B, NQ, S - 1, CPU)


def test_memory_length_per_input_size():
    """The S the forwards pass: tokens over all levels of the input size (P3 = 2x, P4 = 1x, P5 = 1/2 of the 16-px grid)."""
    from b200.config import CONFIGS
    assert CONFIGS["tiny"].memory_len_at(640, 640) == 1600
    assert CONFIGS["tiny"].memory_len_at(832, 1344) == 52 * 84
    assert CONFIGS["large"].memory_len_at(1024, 1024) == 128 * 128 + 32 * 32
    assert CONFIGS["large"].memory_len_at(1344, 1344) == 29988


# ------------------------------------------------------------------------------------- helpers of the GPU test
def test_mask_tables_ties_at_50_and_150_tokens():
    """The numpy restatement of mask_setup puts the first and last valid token of a 50- and 150-token valid extent exactly
    on 0.01 / 0.99 and drops them, as the strict (0.01, 0.99) test of the reference does."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_query_select_gpu import mask_tables
    assert np.float32(0.5) / np.float32(50) == np.float32(0.01) and np.float32(49.5) / np.float32(50) == np.float32(0.99)
    assert np.float32(1.5) / np.float32(150) == np.float32(0.01) and np.float32(148.5) / np.float32(150) == np.float32(0.99)
    H, W = 832, 1344                                    # tiny: one P4 level of 52 x 84
    mask = np.zeros((1, H, W), bool)
    mask[0, 800:, :] = True                             # 50 valid rows
    props, invalid, pad, vr = mask_tables(mask, 1, H, W, [(52, 84)])
    inv = invalid.reshape(52, 84)
    assert inv[0].all() and inv[49].all() and inv[50:].all()
    assert not inv[1:49, 1:83].any()
    assert pad.reshape(52, 84)[50:].all() and not pad.reshape(52, 84)[:50].any()
    assert vr[0, 0] == 1.0 and vr[0, 1] == np.float32(50) / np.float32(52)
    assert (props.reshape(52, 84, 4)[inv.astype(bool)] == 0).all()


def test_ulp_helpers():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_query_select_gpu import ulp16, ulp32
    x = np.array([1.0, 1.5, 0.75, 1e-30, 0.0, 3e4])
    assert np.array_equal(ulp32(x), np.spacing(x.astype(np.float32)).astype(np.float64))
    h = np.array([1.0, 0.75, 2.0 ** -20, 0.0, 1000.0])
    assert np.array_equal(ulp16(h, torch.float16), np.spacing(h.astype(np.float16)).astype(np.float64))
    assert ulp16(np.array([1.0]), torch.bfloat16)[0] == 2.0 ** -7
