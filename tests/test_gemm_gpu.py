"""wgmma/TMA GEMM family vs. fp32 torch math on the same 16-bit-rounded operands (kernel-level)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _tol(dt):
    return 4e-3 if dt == torch.float16 else 2.5e-2


def _close(got, ref, dt, what):
    got = got.float()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    assert err <= _tol(dt) * scale, "%s: max err %.4g vs scale %.4g" % (what, err, scale)
    # rel-L2 (a single wrong low-magnitude row passes the max-abs / max|ref| criterion): output rounding only, the
    # accumulation is fp32 on identical 16-bit operands
    rel = ((got - ref).norm() / (ref.norm() + 1e-30)).item()
    assert rel <= (6e-4 if dt == torch.float16 else 5e-3), "%s: rel-L2 %.3g" % (what, rel)
    if got.dim() == 2 and got.shape[0] > 1:
        rows = (got - ref).norm(dim=1) / (ref.norm(dim=1) + 1e-3 * scale)
        assert rows.max().item() <= (4e-3 if dt == torch.float16 else 3e-2), "%s: worst row rel-L2 %.3g" % (what, rows.max().item())


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("M,N,K", [(300, 96, 256), (128, 64, 64), (1000, 192, 768), (51200, 576, 192),
                                   (257, 91, 256), (4800, 2048, 384), (900, 4, 256), (6400, 384, 960)])
def test_gemm_plain_bias(dt, M, N, K):
    from b200 import capi
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(dt)
    bias = torch.randn(N, device="cuda", generator=g)
    ref = A.float() @ W.float().t() + bias
    if N % 8 == 0:
        out = torch.full((M, N), float("nan"), device="cuda", dtype=dt)
        capi.gemm(A, W, out, bias=bias)
        _close(out, ref, dt, "16-bit out")
    out32 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
    capi.gemm(A, W, out32, bias=bias)
    _close(out32, ref, dt, "fp32 out")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_gemm_epilogue_act_gamma_resid(dt, act):
    from b200 import capi
    M, N, K = 3200, 192, 768
    g = torch.Generator(device="cuda").manual_seed(act)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(dt)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    big = torch.randn(M, 4 * N, device="cuda", generator=g).to(dt)
    resid = big[:, N:2 * N]                      # strided residual (row stride 4N)
    outbuf = torch.zeros(M, 3 * N, device="cuda", dtype=dt)
    out = outbuf[:, 2 * N:]                      # strided destination (concat slot)
    z = A.float() @ W.float().t() + bias
    z = [lambda v: v, F.relu, lambda v: F.gelu(v), F.silu][act](z)
    ref = resid.float() + gamma * z
    capi.gemm(A, W, out, bias=bias, gamma=gamma, resid=resid, act=act)
    _close(out, ref, dt, "act %d" % act)
    assert outbuf[:, :2 * N].abs().max().item() == 0.0


@pytest.mark.parametrize("dt", DTYPES)
def test_gemm_resid_mod_and_strided_A(dt):
    from b200 import capi
    B, T, N, K = 3, 1600, 192, 768
    g = torch.Generator(device="cuda").manual_seed(7)
    Abig = (torch.randn(B * T, K + 64, device="cuda", generator=g) * 0.5).to(dt)
    A = Abig[:, 64:]
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(dt)
    pos = torch.randn(T, N, device="cuda", generator=g).to(dt)
    out = torch.empty(B * T, N, device="cuda", dtype=dt)
    capi.gemm(A, W, out, resid=pos, resid_mod=T)
    ref = A.float() @ W.float().t() + pos.float().repeat(B, 1)
    _close(out, ref, dt, "resid_mod")


def _window_major(x_bhwc):
    B, H, W, C = x_bhwc.shape
    return x_bhwc.reshape(B, 4, H // 4, 4, W // 4, C).permute(0, 1, 3, 2, 4, 5).reshape(B * H * W, C)


@pytest.mark.parametrize("dt", DTYPES)
def test_gemm_window_major_to_spatial(dt):
    from b200 import capi
    B, H, Wd, K, N = 2, 40, 40, 192, 256
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.randn(B, H, Wd, K, device="cuda", generator=g)).to(dt)
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(dt)
    A = _window_major(x).contiguous()
    out = torch.empty(B * H * Wd, N, device="cuda", dtype=dt)
    capi.gemm(A, W, out, rows_in=1, remap_rows=1, IH=H, IW=Wd)
    ref = x.reshape(-1, K).float() @ W.float().t()
    _close(out, ref, dt, "remap")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("rows_in", [0, 1])
def test_gemm_conv_transpose_pixel_shuffle(dt, rows_in):
    from b200 import capi
    B, H, Wd, Cin, Cout = 2, 40, 40, 384, 192
    g = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(B, H, Wd, Cin, device="cuda", generator=g).to(dt)
    wt = (torch.randn(Cin, Cout, 2, 2, device="cuda", generator=g) / Cin ** 0.5).to(dt)   # ConvTranspose2d layout
    bias = torch.randn(Cout, device="cuda", generator=g)
    Wk = wt.permute(2, 3, 1, 0).reshape(4 * Cout, Cin).contiguous()    # row (dy*2+dx)*Cout+co
    A = (_window_major(x) if rows_in else x.reshape(-1, Cin)).contiguous()
    out = torch.empty(B * 2 * H * 2 * Wd, Cout, device="cuda", dtype=dt)
    capi.gemm(A, Wk, out, bias=bias.repeat(4), rows_in=rows_in, shuffle_cout=Cout, IH=H, IW=Wd)
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2).float(), wt.float(), bias, stride=2)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, Cout)
    _close(out, ref, dt, "convT")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("B,OH,OW,stride,Cin,N", [(2, 40, 40, 1, 128, 128), (2, 80, 80, 1, 192, 192),
                                                   (3, 20, 20, 1, 192, 192), (2, 20, 20, 2, 384, 384),
                                                   (1, 20, 20, 2, 768, 768)])
def test_conv3x3_implicit_gemm(dt, B, OH, OW, stride, Cin, N):
    from b200 import capi
    g = torch.Generator(device="cuda").manual_seed(B * OH + Cin + stride)
    IH, IW = OH * stride, OW * stride
    ld = Cin + 64                                   # channel slice of a wider NHWC buffer
    xbuf = torch.randn(B, IH, IW, ld, device="cuda", generator=g).to(dt)
    x = xbuf[..., :Cin]
    w = (torch.randn(N, Cin, 3, 3, device="cuda", generator=g) / (9 * Cin) ** 0.5).to(dt)
    bias = torch.randn(N, device="cuda", generator=g)
    Wk = w.permute(0, 2, 3, 1).reshape(N, 9 * Cin).contiguous()
    out = torch.full((B * OH * OW, N), float("nan"), device="cuda", dtype=dt)
    capi.conv3x3(xbuf, Wk, out, B, OH, OW, stride, Cin, bias=bias, act=capi.ACT_SILU)
    ref = F.silu(F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias, stride=stride, padding=1))
    ref = ref.permute(0, 2, 3, 1).reshape(-1, N)
    _close(out, ref, dt, "conv3x3 s%d" % stride)
