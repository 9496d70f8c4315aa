"""The packed-qkv attention kernel (attn_wg.cu) against fp32 softmax attention at the last chunk of a sequence: keys
beyond the sequence's end are masked, and a tail of at most 40 keys (the second chunk of a 100-token window) computes
5 n-tiles of 8 keys instead of 8.  Every case passes one packed qkv matrix, so only the wgmma kernel runs here; the
tails of the mma.sync kernels (decoder self-attention) are tested in test_attn_mma_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
TOL = {torch.float16: 3e-3, torch.bfloat16: 2e-2}          # max-abs, relative to max|ref| (as test_kernels_gpu.py)
REL_L2 = {torch.float16: 1e-3, torch.bfloat16: 8e-3}


def _run(qkv, nseq, seqlen, heads, dh):
    from b200 import capi
    C = heads * dh
    out = torch.full((nseq * seqlen, C), float("nan"), device="cuda", dtype=qkv.dtype)
    scale = dh ** -0.5
    capi.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, nseq, seqlen, heads, dh, scale)
    q, k, v = [t.float().reshape(nseq, seqlen, heads, dh).transpose(1, 2) for t in (qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:])]
    ref = ((q * scale) @ k.transpose(-2, -1)).softmax(-1) @ v
    return out.float(), ref.transpose(1, 2).reshape(nseq * seqlen, C)


def _check(out, ref, dt):
    assert torch.isfinite(out).all()
    err = (out - ref).abs().max().item()
    assert err <= TOL[dt] * ref.abs().max().item(), err
    rel = ((out - ref).norm() / ref.norm()).item()
    assert rel <= REL_L2[dt], rel


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("dh", [16, 32, 64])
@pytest.mark.parametrize("seqlen", [100, 104, 105, 110, 129, 1153])
def test_masked_tails_ignore_the_next_sequence(dt, dh, seqlen):
    """The last chunk of each sequence reads the next sequence's rows (or zero fill) as keys beyond its end.  The first
    rows of every sequence carry dominant keys whose values alternate in sign from one sequence to the next, so a key
    the tail fails to mask moves the output by a large amount.  100 / 104 / 129 / 1153 end in the 40-key tail (100:
    keys 64..99 of a window), 105 / 110 in a masked 64-key one."""
    nseq, heads = 3, 4
    C = heads * dh
    g = torch.Generator(device="cuda").manual_seed(seqlen + dh)
    qkv = torch.randn(nseq * seqlen, 3 * C, device="cuda", generator=g)
    qkv[:, :C] = 1.0 + 0.2 * qkv[:, :C]
    row = torch.arange(nseq * seqlen, device="cuda")
    first = row % seqlen < 8
    qkv[first, C:2 * C] = 6.0
    sign = 1.0 - 2.0 * ((row // seqlen) % 2).float()
    qkv[first, 2 * C:] = (100.0 * sign[first]).unsqueeze(1)
    late = row % seqlen == seqlen - 3
    qkv[late, C:2 * C] = 6.5                                        # a key near the end raises the running maximum again
    qkv = qkv.to(dt)
    out, ref = _run(qkv, nseq, seqlen, heads, dh)
    _check(out, ref, dt)
