"""The kernels whose indexing depends on the input size, at every geometry the engine can plan (the enumeration of
test_geometry_cpu), element by element against float64:
  * the implicit-GEMM 3x3 convolution, stride 1 (all 1,037 output grids) and stride 2 (all 399), and at the engine's channel
    widths once per distinct tile plan;
  * the window-major -> spatial row remap and the pixel-shuffle ConvTranspose store (all 399 token grids, and the engine's
    widths on non-square grids);
  * the deformable attention over all 796 level tables (staged bands or direct gather, whichever the plan picks, and the
    test checks that this kernel ran), then its persistent (image, head) walk and query passes.

Bounds are per element.  GEMM / conv: |y - y64| <= 1/2 ulp_T(|y64|) + (K/16) 2^-22 sum|a w|, times 1.1 after SiLU (y64 the
float64 result of the same 16-bit operands, sum|a w| the float64 product / convolution of |A| and |W|).  Deformable attention:
|y - y64| <= 1/2 ulp_T(|y64|) + 2^-17 A + 2^-22 A_top, A = msda_core(|value|, loc, aw) and A_top the same with each sample
on its top row (test_geometry_cpu.msda_bound says why).  Reference boxes, offsets and valid ratios lie on a
dyadic grid, so the kernel's fp32 location arithmetic is exact and the float64 reference samples the same positions; what
is left is the __expf / __fdividef softmax, the rounding of the corner weights and the fp32 accumulation of at most 4 L P
terms.

Each sweep collects every failing geometry with its plan and asserts once, and prints its worst error / bound ratio
(pytest -s).  test_geometry_cpu.test_bounds_resolve_one_misplaced_tap_or_corner shows that one tap read from the neighbouring
pixel, or one sample read a row off, costs far more than these bounds.  The file runs in 2.2 to 3.2 minutes on one H100."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200.config import CONFIGS
from test_geometry_cpu import (conv_s1_grids, conv_s2_grids, gemm_bound, level_tables, msda_bound, tile_plans, token_grids,
                               top_row_locations)

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
NAN = float("nan")
GUARD_ROWS = 64               # NaN rows after every output: a store past the last row shows up there


class Sweep:
    """Failures and the worst error / bound ratio over the cases of one sweep."""

    def __init__(self, name):
        self.name, self.failures, self.worst, self.cases = name, [], (0.0, ""), 0

    def check(self, what, got, y64, bound, buf=None, inside=None):
        """got: the 16-bit output; buf / inside: the whole NaN-prefilled output buffer and the mask of what the call may write."""
        self.cases += 1
        ratio = ((got.double() - y64).abs() / bound).nan_to_num(nan=math.inf).flatten()
        i = int(ratio.argmax())
        r = ratio[i].item()
        if r > self.worst[0]:
            self.worst = (r, what)
        if not r <= 1.0:
            self.failures.append("%s: err/bound %.3g at flat index %d (got %r, want %r)" % (
                what, r, i, got.flatten()[i].item(), y64.flatten()[i].item()))
        if buf is not None and not torch.isnan(buf[~inside]).all():
            self.failures.append("%s: %d elements written outside the output" % (what, int((~torch.isnan(buf[~inside])).sum())))

    def finish(self):
        print("\n%s: %d cases, worst err/bound %.3f (%s)" % (self.name, self.cases, self.worst[0], self.worst[1]))
        assert not self.failures, "%d of %d cases failed:\n%s" % (len(self.failures), self.cases, "\n".join(self.failures[:20]))


def _rnd(shape, dt, g, scale=1.0):
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dt)


def _out_buffer(rows, ld, off, n, dt):
    """NaN-prefilled [rows + GUARD_ROWS, ld] buffer, its [rows, off:off+n] slice and the mask of that slice."""
    buf = torch.full((rows + GUARD_ROWS, ld), NAN, device="cuda", dtype=dt)
    inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    inside[:rows, off:off + n] = True
    return buf, buf[:rows, off:off + n], inside


# ------------------------------------------------------------------------------------------------ implicit-GEMM conv
def _conv_case(sw, dt, g, what, B, OH, OW, stride, Cin, N, off_in, ld_in, off_out, ld_out, act=0, bias=False):
    from b200 import capi
    IH, IW = OH * stride, OW * stride
    x = _rnd((B, IH, IW, Cin), dt, g)
    xbuf = torch.full((B, IH, IW, ld_in), NAN, device="cuda", dtype=dt)
    xbuf[..., off_in:off_in + Cin] = x
    w = _rnd((N, Cin, 3, 3), dt, g, (9 * Cin) ** -0.5)
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    Wk = w.permute(0, 2, 3, 1).reshape(N, 9 * Cin).contiguous()
    M = B * OH * OW
    buf, out, inside = _out_buffer(M, ld_out, off_out, N, dt)
    capi.conv3x3(xbuf[..., off_in:], Wk, out, B, OH, OW, stride, Cin, bias=b, act=act)
    xc = x.permute(0, 3, 1, 2)
    z = F.conv2d(xc.double(), w.double(), None if b is None else b.double(), stride=stride, padding=1)
    absacc = F.conv2d(xc.double().abs(), w.double().abs(), None, stride=stride, padding=1)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(M, N)
    y64 = flat({0: z, capi.ACT_RELU: F.relu(z), capi.ACT_SILU: F.silu(z)}[act])
    sw.check("%s %dx%d tile %s" % (what, OH, OW, capi.conv3x3_plan(OH, OW)), out, y64,
             gemm_bound(y64, flat(absacc), 9 * Cin, dt, act == capi.ACT_SILU), buf, inside)


@pytest.mark.parametrize("dt", DTYPES)
def test_conv3x3_stride1_every_grid(dt):
    """All 1,037 stride-1 output grids, B = 2, Cin = 128 (two 64-channel blocks) read at channel 64 of a 256-wide NHWC buffer
    whose other channels are NaN, N = 64 written into columns 64..127 of a NaN-filled 192-wide buffer.
    Worst err/bound on an NVIDIA H100 80GB HBM3 (700 W): 0.86 fp16, 0.98 bf16."""
    sw = Sweep("conv3x3 s1 %s" % dt)
    g = torch.Generator(device="cuda").manual_seed(1)
    for oh, ow in conv_s1_grids():
        _conv_case(sw, dt, g, "s1", 2, oh, ow, 1, 128, 64, 64, 256, 64, 192)
    sw.finish()


@pytest.mark.parametrize("dt", DTYPES)
def test_conv3x3_stride2_every_grid(dt):
    """All 399 stride-2 output grids (the P5 down-sampling of large / xlarge), built as the stride-1 sweep.
    Worst err/bound on an NVIDIA H100 80GB HBM3 (700 W): 0.85 fp16, 0.98 bf16."""
    sw = Sweep("conv3x3 s2 %s" % dt)
    g = torch.Generator(device="cuda").manual_seed(2)
    for oh, ow in conv_s2_grids():
        _conv_case(sw, dt, g, "s2", 2, oh, ow, 2, 128, 64, 64, 256, 64, 192)
    sw.finish()


@pytest.mark.parametrize("dt", DTYPES)
def test_conv3x3_engine_widths_every_tile_plan(dt):
    """The engine's convolutions, one grid per distinct tile plan (a ragged one, OH % TH != 0, where the plan has one):
    stride 1 with Cin = N = c2 (128, 192), bias and SiLU, reading column slice (1+j) c2 of a 5 c2-wide buffer and writing slice
    (2+j) c2 (the C2f bottlenecks); stride 2 with Cin = N = C (384, 768), bias and ReLU, slice t C of an ntap C-wide buffer.
    Worst err/bound on an NVIDIA H100 80GB HBM3 (700 W): 0.81 fp16, 0.94 bf16."""
    sw = Sweep("conv3x3 engine widths %s" % dt)
    g = torch.Generator(device="cuda").manual_seed(3)
    s1 = conv_s1_grids()
    for k, (plan, grids) in enumerate(tile_plans(s1).items()):
        oh, ow = grids[0]
        for c2 in s1[(oh, ow)]:
            j = k % 3
            _conv_case(sw, dt, g, "s1 c2=%d" % c2, 2, oh, ow, 1, c2, c2, (1 + j) * c2, 5 * c2, (2 + j) * c2, 5 * c2, act=3, bias=True)
    s2 = conv_s2_grids()
    for k, (plan, grids) in enumerate(tile_plans(s2).items()):
        oh, ow = grids[0]
        for C in s2[(oh, ow)]:
            t = k % 4
            _conv_case(sw, dt, g, "s2 C=%d" % C, 2, oh, ow, 2, C, C, t * C, 4 * C, t * C, 4 * C, act=1, bias=True)
    sw.finish()


# ------------------------------------------------------------------------------------------------ row remap / pixel shuffle
def _window_major(x_bhwc):
    B, H, W, C = x_bhwc.shape
    return x_bhwc.reshape(B, 4, H // 4, 4, W // 4, C).permute(0, 1, 3, 2, 4, 5).reshape(B * H * W, C)


def _rows_case(sw, dt, g, what, B, GH, GW, K, N, ld_out, off_out, shuffle=0, act=0, bias=True, lda=None, off_a=32):
    """Window-major rows in (columns off_a.. of a NaN-filled buffer lda wide, K + 64 by default), remapped to spatial order
    (shuffle = 0) or pixel-shuffled by ConvTranspose2d(k=2, s=2) with cout = shuffle."""
    from b200 import capi
    lda = K + 64 if lda is None else lda
    x = _rnd((B, GH, GW, K), dt, g)
    abuf = torch.full((B * GH * GW, lda), NAN, device="cuda", dtype=dt)
    abuf[:, off_a:off_a + K] = _window_major(x)
    Wt = _rnd((N, K), dt, g, K ** -0.5)
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    x64 = x.double().reshape(-1, K)
    z = x64 @ Wt.double().t() + (0 if b is None else b.double())
    absacc = x64.abs() @ Wt.double().abs().t()
    if shuffle:
        rows, n = 4 * B * GH * GW, shuffle
        sh = lambda t: t.reshape(B, GH, GW, 2, 2, n).permute(0, 1, 3, 2, 4, 5).reshape(rows, n)
        z, absacc = sh(z), sh(absacc)
    else:
        rows, n = B * GH * GW, N
    buf, out, inside = _out_buffer(rows, ld_out, off_out, n, dt)
    capi.gemm(abuf[:, off_a:off_a + K], Wt, out, bias=b, act=act, rows_in=1, remap_rows=0 if shuffle else 1, shuffle_cout=shuffle, IH=GH, IW=GW)
    y64 = F.silu(z) if act == capi.ACT_SILU else z
    sw.check("%s %dx%d" % (what, GH, GW), out, y64, gemm_bound(y64, absacc, K, dt, act == capi.ACT_SILU), buf, inside)


@pytest.mark.parametrize("dt", DTYPES)
def test_remap_and_pixel_shuffle_every_token_grid(dt):
    """All 399 token grids, B = 2, K = 64: the remap (N = 64) into columns 64..127 of a 192-wide buffer and the pixel shuffle
    (cout = 16) into columns 16..31 of a 48-wide buffer.  Then the engine's widths on non-square grids, derived from the
    configs as the engine derives them: the P4 cv1 (K = ntap C of tiny / small / medium, N = 2 c2, SiLU) and the P3
    up-sampling (K = C reading slice t C of the ntap C-wide tap buffer for C <= 512; K = C / 2 reading the contiguous output
    of the `pre` GEMM for C > 512; cout = cs = C / 2 or C / 4) into slice t cs of the ntap cs-wide sample buffer.  Worst err/bound on an NVIDIA H100 80GB HBM3 (700 W): 0.998 fp16, 1.000 bf16 (a result that
    sits on a rounding midpoint: the bound is tight by construction)."""
    sw = Sweep("remap / pixel shuffle %s" % dt)
    g = torch.Generator(device="cuda").manual_seed(4)
    for gh, gw in token_grids():
        _rows_case(sw, dt, g, "remap", 2, gh, gw, 64, 64, 192, 64)
        _rows_case(sw, dt, g, "shuffle", 2, gh, gw, 64, 64, 48, 16, shuffle=16)
    cv1 = sorted({(len(c.taps) * c.vit_dim, c.hidden_dim) for c in CONFIGS.values() if c.projector_scale == ("P4",)})
    up = sorted({(len(c.taps), c.vit_dim) for c in CONFIGS.values() if "P3" in c.projector_scale})
    for k, (gh, gw) in enumerate([(8, 84), (84, 8), (12, 44), (44, 76), (76, 28), (52, 84)]):
        for K, d in cv1:
            _rows_case(sw, dt, g, "cv1 K=%d" % K, 2, gh, gw, K, d, 5 * d // 2, 0, act=3)
        for ntap, C in up:
            cs, t = (C // 4 if C > 512 else C // 2), k % ntap
            if C > 512:     # the `pre` GEMM's contiguous [rows, C / 2] output
                _rows_case(sw, dt, g, "up C=%d" % C, 2, gh, gw, C // 2, 4 * cs, ntap * cs, t * cs, shuffle=cs, lda=C // 2, off_a=0)
            else:           # slice t C of the tap buffer
                _rows_case(sw, dt, g, "up C=%d" % C, 2, gh, gw, C, 4 * cs, ntap * cs, t * cs, shuffle=cs, lda=ntap * C, off_a=t * C)
    sw.finish()


# ------------------------------------------------------------------------------------------------ deformable attention
FAMILY = {1: (16, 2), 2: (24, 4)}          # levels -> (heads M, points P): P4 of tiny..medium, P3 + P5 of large / xlarge
VR = [(0.75, 0.625), (1.0, 1.0), (0.625, 0.75)]
Q13 = 2.0 ** -13


def _targets(shapes, bands, gen):
    """(level, y, x) pixel positions (the kernel's py, px) to aim queries at: each band's own0, own1 and own1 + 1 rows, on the
    row and at +0.25 / +0.75; y in (-1, 0) and (H-1, H); x in (-1, 0) and (W-1, W); just outside each level."""
    out = []
    u = lambda lo, hi: lo + (hi - lo) * torch.rand((), generator=gen).item()
    for lvl, _, own0, own1, _, _ in bands:
        H, W = shapes[lvl]
        for r in (own0, own1, own1 + 1):
            if 0 <= r < H:
                out += [(lvl, r + f, u(0, W - 1)) for f in (0.0, 0.25, 0.75)]
    for lvl, (H, W) in enumerate(shapes):
        out += [(lvl, -0.5, u(0, W - 1)), (lvl, -0.9, u(0, W - 1)), (lvl, H - 0.5, u(0, W - 1)), (lvl, H - 0.9, u(0, W - 1)),
                (lvl, u(0, H - 1), -0.5), (lvl, u(0, H - 1), -0.9), (lvl, u(0, H - 1), W - 0.5), (lvl, u(0, H - 1), W - 0.9),
                (lvl, -1.03, u(0, W - 1)), (lvl, H + 0.03, u(0, W - 1)), (lvl, u(0, H - 1), -1.03), (lvl, u(0, H - 1), W + 0.03)]
        if not bands:
            out += [(lvl, r + f, u(0, W - 1)) for r in (0, H // 2, H - 2) for f in (0.0, 0.25, 0.75)]
    return out


def _msda_inputs(shapes, bands, B, Lq, dt, gen):
    """Dyadic reference boxes [B*Lq, 4], valid ratios [B, L, 2] and 16-bit offsets / logits [B*Lq, 3 M L P].
    Aimed queries: the box centre sits on the target (on a 2^-13 grid before the valid ratio), w = h = 2^-10 and integer
    offsets in [-4, 4] spread the samples a few hundredths of a row around it.  The other queries: centres on the 2^-13 grid
    in [-0.05, 1.05], w, h multiples of 2^-7 up to 1/4, offsets multiples of 1/2 in [-6, 6].  Every product and sum of the
    location arithmetic then fits 24 bits: the kernel's fp32 positions are exact."""
    L = len(shapes)
    M, P = FAMILY[L]
    vr = torch.tensor([[VR[(b + l) % 3] for l in range(L)] for b in range(B)], dtype=torch.float64)
    ref = torch.zeros(B, Lq, 4, dtype=torch.float64)
    ref[..., :2] = torch.randint(-410, 8602, (B, Lq, 2), generator=gen) * Q13
    ref[..., 2:] = torch.randint(1, 33, (B, Lq, 2), generator=gen) * 2.0 ** -7
    offs = torch.randint(-12, 13, (B, Lq, M, L, P, 2), generator=gen) * 0.5
    targets = _targets(shapes, bands, gen)
    for i, (lvl, y, x) in enumerate(targets[:Lq * B]):
        b, q = i % B, (i // B) % Lq
        H, W = shapes[lvl]
        ref[b, q, 0] = round((x + 0.5) / W / vr[b, lvl, 0].item() / Q13) * Q13
        ref[b, q, 1] = round((y + 0.5) / H / vr[b, lvl, 1].item() / Q13) * Q13
        ref[b, q, 2:] = 2.0 ** -10
        offs[b, q] = torch.randint(-4, 5, (M, L, P, 2), generator=gen).double()
    logits = torch.randn(B, Lq, M, L * P, generator=gen, dtype=torch.float64) * 2
    ol = torch.cat([offs.reshape(B * Lq, -1), logits.reshape(B * Lq, -1)], 1).to(dt)
    assert torch.equal(ol[:, :M * L * P * 2].double(), offs.reshape(B * Lq, -1))      # offsets exact in dt
    return ref, vr, ol, len(targets)


def _msda_case(sw, dt, gen, what, shapes, B, Lq, kernels):
    from b200 import capi
    from oracle import lwdetr_oracle as orc
    L = len(shapes)
    M, P = FAMILY[L]
    S = sum(h * w for h, w in shapes)
    bands = capi.msda_plan(shapes)
    kernels.append("msda_fwd_kernel" if bands else "msda_gather_kernel")
    ref, vr, ol, ntarget = _msda_inputs(shapes, bands, B, Lq, dt, gen)
    hm = torch.full((B, 3, M, S, 16), NAN, device="cuda", dtype=dt)              # [B][slice][head][token][16], middle slice used
    value = torch.randn(B, M, S, 16, device="cuda", dtype=torch.float64, generator=torch.Generator(device="cuda").manual_seed(S))
    hm[:, 1] = value.to(dt)
    buf, out, inside = _out_buffer(B * Lq, M * 16 + 32, 16, M * 16, dt)
    capi.msda_forward(hm[:, 1], ol.cuda(), ref.float().cuda().reshape(B * Lq, 4), out, B, S, Lq, M, L, P, shapes,
                      valid_ratio=vr.float().cuda().contiguous(), v_image_stride=3 * M * S * 16)
    v64 = hm[:, 1].double().permute(0, 2, 1, 3).contiguous()                       # [B, S, M, 16]
    olc = ol.cuda().double()
    off = olc[:, :M * L * P * 2].reshape(B, Lq, M, L, P, 2)
    aw = olc[:, M * L * P * 2:].reshape(B, Lq, M, L * P).softmax(-1).reshape(B, Lq, M, L, P)
    rb = ref.cuda()[:, :, None, None, None, :]
    loc = (rb[..., :2] + off * rb[..., 2:] * (0.5 / P)) * vr.cuda()[:, None, None, :, None, :]
    y64 = orc.msda_core(v64, shapes, loc, aw).reshape(B * Lq, M * 16)
    A = orc.msda_core(v64.abs(), shapes, loc, aw).reshape(B * Lq, M * 16)
    A_top = orc.msda_core(v64.abs(), shapes, top_row_locations(loc, shapes), aw).reshape(B * Lq, M * 16)
    plan = "%d bands" % len(bands) if bands else "gather"
    sw.check("%s %s (%s, %d aimed)" % (what, shapes, plan, ntarget), out, y64, msda_bound(y64, A, A_top, dt), buf, inside)


def _assert_kernels(prof, want):
    """The deformable-attention kernels the profiler saw, in launch order, are the ones the plans named."""
    ev = [e for e in prof.events() if "msda_fwd_kernel" in e.name or "msda_gather_kernel" in e.name]
    ev.sort(key=lambda e: e.time_range.start)
    ran = ["msda_fwd_kernel" if "msda_fwd_kernel" in e.name else "msda_gather_kernel" for e in ev]
    first = next((i for i, (a, b) in enumerate(zip(ran, want)) if a != b), min(len(ran), len(want)))
    assert ran == want, "kernels that ran differ from the plans: %d launches seen, %d planned, first difference at %d: %s vs %s" % (
        len(ran), len(want), first, ran[first:first + 3], want[first:first + 3])


@pytest.mark.parametrize("dt", DTYPES)
def test_msda_every_level_table(dt):
    """All 796 level tables (397 P4: M = 16, L = 1, P = 2; 399 P3 + P5: M = 24, L = 2, P = 4), B = 2, Lq = 300, valid ratios
    0.75 / 0.625 / 1 per image and level.  The value is the middle slice of a three-slice head-major buffer whose other
    slices are NaN; the output is a NaN-guarded column slice.  The kernel that ran (profiler) is the one the plan names.
    Worst err/bound on an NVIDIA H100 80GB HBM3 (700 W): 1.000 fp16, 0.998 bf16."""
    from torch.profiler import ProfilerActivity, profile
    sw = Sweep("msda %s" % dt)
    gen = torch.Generator().manual_seed(5)
    want = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for shapes in level_tables():
            _msda_case(sw, dt, gen, "table", list(shapes), 2, 300, want)
        torch.cuda.synchronize()
    sw.finish()
    _assert_kernels(prof, want)
    assert want.count("msda_fwd_kernel") == 628 and want.count("msda_gather_kernel") == 168


@pytest.mark.parametrize("dt", DTYPES)
def test_msda_persistent_walk_and_passes(dt):
    """One multi-band non-square table per family (P4 64 x 76 of small at 1024 x 1216, 4 bands with a one-row last band;
    P3 56 x 136 + P5 14 x 34 of large at 448 x 1088, 7 bands) with more (image, head) items than twice the SM count and not a
    multiple of it, so that CTAs walk several items with the (image, head) carry; Lq = 300 / 321 / 700 are 1, 2 and 3 passes
    of 320 queries.  Worst err/bound on an NVIDIA H100 80GB HBM3 (700 W): 1.000 fp16, 0.998 bf16."""
    from b200 import capi
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if any(sms % FAMILY[L][0] == 0 for L in FAMILY):
        pytest.skip("%d SMs is a multiple of a family's head count: the grid stride never carries into the next image" % sms)
    sw = Sweep("msda walk %s" % dt)
    gen = torch.Generator().manual_seed(6)
    for shapes in ([(64, 76)], [(56, 136), (14, 34)]):
        M = FAMILY[len(shapes)][0]
        B = 2 * sms // M + 1
        B += (B * M) % sms == 0
        assert len(capi.msda_plan(shapes)) >= 4                                  # the staged kernel, several bands
        for Lq in (300, 321, 700):
            _msda_case(sw, dt, gen, "B=%d Lq=%d" % (B, Lq), shapes, B, Lq, [])
    sw.finish()
