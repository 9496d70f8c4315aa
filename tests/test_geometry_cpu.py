"""Every geometry the engine can plan, enumerated from the accepted input sizes, and the invariants of the plans the kernels
run for them (host queries only, no GPU): the implicit-GEMM conv tiles and the deformable-attention band tables.
tests/test_geometry_gpu.py runs the kernels over the same enumeration against float64."""
import collections

import pytest
import torch
import torch.nn.functional as F

from b200 import capi
from b200.config import CONFIGS, MAX_SIDE, MIN_SIDE, SIDE_STEP, check_input_size

MS_STAGE_TOKENS = 1680      # tokens one shared-memory stage of msda_fwd_kernel holds (msda.cu)
MS_TOKEN_FIELD = 8192       # 13-bit token field of the packed sample info (msda.cu info[k])

MANT = {torch.float16: 10, torch.bfloat16: 7}


def half_ulp(y64, dt):
    """1/2 ulp of |y64| in dt (subnormal spacing below the normal range)."""
    e = torch.floor(torch.log2(y64.abs().clamp_min(torch.finfo(dt).tiny)))
    return torch.exp2(e - MANT[dt] - 1)


def gemm_bound(y64, absacc, K, dt, silu=False):
    """Per-element bound of a 16-bit GEMM / implicit-GEMM conv: output rounding + (K/16) 2^-22 sum|a w|, x 1.1 after SiLU."""
    b = half_ulp(y64, dt) + (K / 16) * 2.0 ** -22 * absacc
    return b * 1.1 if silu else b


def msda_bound(y64, A, A_top, dt):
    """Per-element bound of the deformable attention with exact sample positions: output rounding + 2^-17 A, A the float64
    result on |value|, + 2^-22 A_top, A_top the same with every sample moved onto its top row (floor(y)) at full weight.
    The kernels form a sample's top-row weight as w - w fy with w fy rounded first, exact to 2^-24 w only: just above the
    bottom border (bottom row outside, fy -> 1) that rounding is all of the sample's weight, and A does not cover it."""
    return half_ulp(y64, dt) + 2.0 ** -17 * A + 2.0 ** -22 * A_top


def top_row_locations(loc, shapes):
    """loc [B, Q, M, L, P, 2] with each sample's y moved onto its top row floor(y * H - 0.5), x kept."""
    out = loc.clone()
    for lvl, (H, _) in enumerate(shapes):
        y0 = torch.floor(loc[..., lvl, :, 1] * H - 0.5)
        out[..., lvl, :, 1] = (y0 + 0.5 + 2.0 ** -20) / H
    return out


Geometry = collections.namedtuple("Geometry", "config H W grid levels conv_s1 conv_s2")


def geometries():
    """One Geometry per (config, H, W) that check_input_size accepts:
      grid     the (GH, GW) token grid (window-major rows of the ViT; the P4 cv1 remap and the P3 up-sampling read it);
      levels   the level table of the deformable attention, ((H, W), ...);
      conv_s1  [(OH, OW, c2)]: the C2f bottleneck 3x3 convs of every level, Cin = N = c2 = hidden_dim / 2;
      conv_s2  (OH, OW, C) of the P5 down-sampling conv (Cin = N = vit_dim) or None."""
    for name, cfg in CONFIGS.items():
        c2 = cfg.hidden_dim // 2
        for H in range(MIN_SIDE, MAX_SIDE + 1, SIDE_STEP):
            for W in range(MIN_SIDE, MAX_SIDE + 1, SIDE_STEP):
                try:
                    check_input_size(cfg, H, W)
                except RuntimeError:
                    continue
                levels = cfg.level_shapes_at(H, W)
                s2 = None
                if "P5" in cfg.projector_scale:
                    s2 = levels[cfg.projector_scale.index("P5")] + (cfg.vit_dim,)
                yield Geometry(name, H, W, (H // 16, W // 16), levels, [(h, w, c2) for h, w in levels], s2)


def conv_s1_grids():
    """{(OH, OW): sorted channel widths c2} over every stride-1 conv the engine can plan."""
    out = collections.defaultdict(set)
    for g in geometries():
        for oh, ow, c2 in g.conv_s1:
            out[(oh, ow)].add(c2)
    return {k: sorted(v) for k, v in sorted(out.items())}


def conv_s2_grids():
    """{(OH, OW): sorted channel widths C} over every stride-2 conv (P5 of large / xlarge)."""
    out = collections.defaultdict(set)
    for g in geometries():
        if g.conv_s2:
            out[g.conv_s2[:2]].add(g.conv_s2[2])
    return {k: sorted(v) for k, v in sorted(out.items())}


def token_grids():
    return sorted({g.grid for g in geometries()})


def level_tables():
    """{level table: [(config, H, W), ...]} over every table the engine can plan (one level: P4; two: P3 + P5)."""
    out = collections.defaultdict(list)
    for g in geometries():
        out[g.levels].append((g.config, g.H, g.W))
    return dict(sorted(out.items()))


def tile_plans(grids):
    """{(TW, TH): [grids with that plan]}, ragged grids (OH % TH != 0) first."""
    out = collections.defaultdict(list)
    for oh, ow in grids:
        out[capi.conv3x3_plan(oh, ow)].append((oh, ow))
    for tw, th in out:
        out[(tw, th)].sort(key=lambda s: (s[0] % th == 0, s))
    return dict(sorted(out.items()))


def band_rows(band, W):
    """(first, last) image row a band stages."""
    rows = band[5] // (32 * W)
    return band[1], band[1] + rows - 1


def test_enumeration_counts():
    """The counts the engine's size range gives (sides multiples of 64 in [128, 1344], at least num_queries tokens)."""
    assert len(conv_s1_grids()) == 1037
    assert len(conv_s2_grids()) == 399
    assert len(token_grids()) == 399
    tables = level_tables()
    assert sum(len(t) == 1 for t in tables) == 397 and sum(len(t) == 2 for t in tables) == 399
    assert set(conv_s1_grids()[(40, 40)]) == {128, 192} and conv_s2_grids()[(20, 20)] == [384, 768]
    assert all(gh % 4 == 0 and gw % 4 == 0 and 8 <= min(gh, gw) and max(gh, gw) <= 84 for gh, gw in token_grids())


def test_conv_tile_plans():
    grids = sorted(set(conv_s1_grids()) | set(conv_s2_grids()))
    ragged = 0
    for oh, ow in grids:
        tw, th = capi.conv3x3_plan(oh, ow)
        assert 1 <= tw <= ow and 1 <= th <= oh and tw * th <= 128, (oh, ow, tw, th)
        tx, ty = -(-ow // tw), -(-oh // th)
        assert (tx - 1) * tw < ow <= tx * tw and (ty - 1) * th < oh <= ty * th, (oh, ow, tw, th)
        ragged += oh % th != 0
    assert ragged > 0
    # a strip as wide as one pixel: P3 at 960 / 1024 px height
    assert capi.conv3x3_plan(120, 24) == (1, 120) and capi.conv3x3_plan(128, 40) == (1, 128)
    assert len(tile_plans(conv_s1_grids())) == 116 and len(tile_plans(conv_s2_grids())) == 107


def test_conv_tile_plans_at_640_are_unchanged():
    """The tiles of a 640 x 640 input (P5, P4, P3), as the planner chose them before it became a query."""
    assert capi.conv3x3_plan(20, 20) == (5, 20)
    assert capi.conv3x3_plan(40, 40) == (3, 40)
    assert capi.conv3x3_plan(80, 80) == (8, 16)


def test_conv_tile_plan_rejects_empty_grids():
    for oh, ow in ((0, 8), (8, 0), (-1, 4)):
        with pytest.raises(RuntimeError, match="must be positive"):
            capi.conv3x3_plan(oh, ow)


def _bands_per_level(H, W):
    rows_max = MS_STAGE_TOKENS // W
    return 1 if H <= rows_max else -(-H // (rows_max - 1))


def check_msda_plan(shapes, bands):
    """The invariants of one level table's plan; returns a list of violations."""
    fits = all(2 * w <= MS_STAGE_TOKENS and h * w <= MS_TOKEN_FIELD for h, w in shapes)
    staged = fits and sum(_bands_per_level(h, w) for h, w in shapes) <= capi.MSDA_MAX_BANDS
    if staged != bool(bands):
        return ["staged %s but %d bands" % (staged, len(bands))]
    if not bands:
        return []
    bad, start = [], 0
    for l, (H, W) in enumerate(shapes):
        mine = [b for b in bands if b[0] == l]
        if [b[2] for b in mine] != sorted(b[2] for b in mine):
            bad.append("level %d: bands out of order" % l)
        owned = [y for b in mine for y in range(b[2], b[3] + 1)]
        if owned != list(range(-1, H)):
            bad.append("level %d: own ranges do not partition [-1, %d]" % (l, H - 1))
        for b in mine:
            r0, r1 = band_rows(b, W)
            if b[5] % (32 * W) or b[5] > MS_STAGE_TOKENS * 32 or r0 < 0 or r1 > H - 1:
                bad.append("level %d band %s: staged rows / bytes" % (l, b))
            if b[4] != start + r0 * W:
                bad.append("level %d band %s: tok0 != level_start + row0 * W" % (l, b))
            for y0 in range(b[2], b[3] + 1):
                if not (r0 <= max(y0, 0) <= r1 and r0 <= min(y0 + 1, H - 1) <= r1):
                    bad.append("level %d band %s: floor(y) = %d reads a row it does not stage" % (l, b, y0))
                    break
        start += H * W
    if [b[0] for b in bands] != sorted(b[0] for b in bands):
        bad.append("levels out of order")
    return bad


def test_msda_plans_of_every_level_table():
    failures, staged = [], collections.Counter()
    for shapes, sizes in level_tables().items():
        bands = capi.msda_plan(shapes)
        staged[(len(shapes), bool(bands))] += 1
        failures += ["%s (%s %dx%d): %s" % ((shapes,) + sizes[0] + (v,)) for v in check_msda_plan(shapes, bands)]
    assert not failures, "\n".join(failures[:20])
    assert staged == {(1, True): 397, (2, True): 231, (2, False): 168}


def _edge_sizes():
    """(config, H, W) of the staged plans with a one-row final band, with seven bands, and with an 8192-token level."""
    one_row, seven, full = set(), set(), set()
    for g in geometries():
        bands = capi.msda_plan(g.levels)
        for b in bands:
            H, W = g.levels[b[0]]
            if b[1] == H - 1 and b[1] > 0 and band_rows(b, W) == (H - 1, H - 1):
                one_row.add((g.config, g.H, g.W))
        if len(bands) == 7:
            seven.add((g.config, g.H, g.W))
        if bands and any(h * w == MS_TOKEN_FIELD for h, w in g.levels):
            full.add((g.config, g.H, g.W))
    return one_row, seven, full


def test_named_edge_geometries_are_planned():
    one_row, seven, full = _edge_sizes()
    assert {("large", 320, 960), ("large", 448, 1088), ("large", 704, 448), ("small", 1024, 1216), ("small", 1216, 1024)} <= one_row
    assert {("large", 384, 1344), ("large", 448, 1088), ("large", 512, 1024), ("large", 576, 896)} <= seven
    assert {("large", 512, 1024), ("large", 1024, 512)} <= full
    assert capi.msda_plan([(64, 128), (16, 32)])[0][:4] == (0, 0, -1, 11)


def test_msda_plan_rejects_invalid_tables():
    with pytest.raises(RuntimeError, match="invalid level table"):
        capi.msda_plan([(40, 40)], S=1599)
    with pytest.raises(RuntimeError, match="invalid level table"):
        capi.msda_plan([(0, 40)])
    with pytest.raises(RuntimeError, match="1..4 levels"):
        capi.msda_plan([(4, 4)] * 5)
    assert capi.msda_plan([(40, 40)], S=3 * 1600) == [(0, 0, -1, 39, 0, 1600 * 32)]
    assert capi.msda_plan([(96, 128)]) == [] and capi.msda_plan([(8, 1024)]) == []


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_bounds_resolve_one_misplaced_tap_or_corner(dt):
    """At the magnitudes the GPU sweeps use, one conv tap read from the neighbouring pixel, or one deformable-attention sample
    read one row off, moves a typical output element by at least 10x its bound (median over the elements it touches).
    Measured medians: 525x (fp16) and 143x (bf16) for the tap, 1430x and 188x for the row."""
    from oracle import lwdetr_oracle as orc
    g = torch.Generator().manual_seed(7)
    Cin, N = 128, 64
    x = torch.randn(1, Cin, 20, 20, generator=g).to(dt).double()
    w = (torch.randn(N, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(dt).double()
    y64 = F.conv2d(x, w, padding=1)
    moved = torch.zeros_like(w)
    moved[:, :, 1, 1], moved[:, :, 0, 0] = w[:, :, 0, 0], -w[:, :, 0, 0]       # tap (0, 0) read at (1, 1)
    err = F.conv2d(x, moved, padding=1)[..., 1:, 1:].abs()
    bound = gemm_bound(y64, F.conv2d(x.abs(), w.abs(), padding=1), 9 * Cin, dt)[..., 1:, 1:]
    assert (err / bound).median().item() >= 10
    # deformable attention, P4 family: point 0 of every (query, head) read one row lower
    B, Q, M, P, H, W = 2, 300, 16, 2, 40, 40
    value = torch.randn(B, H * W, M, 16, generator=g).to(dt).double()
    loc = torch.rand(B, Q, M, 1, P, 2, generator=g, dtype=torch.float64) * 0.9 + 0.05
    aw = torch.randn(B, Q, M, P, generator=g, dtype=torch.float64).mul(2).softmax(-1).reshape(B, Q, M, 1, P)
    y64 = orc.msda_core(value, [(H, W)], loc, aw)
    off = loc.clone()
    off[:, :, :, :, 0, 1] += 1.0 / H
    err = (orc.msda_core(value, [(H, W)], off, aw) - y64).abs()
    top = orc.msda_core(value.abs(), [(H, W)], top_row_locations(loc, [(H, W)]), aw)
    bound = msda_bound(y64, orc.msda_core(value.abs(), [(H, W)], loc, aw), top, dt)
    assert (err / bound).median().item() >= 10
