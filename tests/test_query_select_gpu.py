"""The two-stage query selection between the encoder memory and the decoder, one engine op at a time (csrc/rowops.cu):
mask_setup, enc_score (rowmax), topk, gather_topk, query_init (box_ts, refpoint, sine embedding), tgt_init, tgt_plus_pos and
final_boxes.  Every op is checked on the engine's own captured inputs, so errors do not compound down the chain, against a
plain restatement of that one op.

Exact (bit for bit) wherever the op only moves, compares or selects values: the padding tables (against a numpy float32
restatement and against the oracle's encoder_proposals / level_padding_masks), the row max, the top-k order (a stable
descending sort: ties go to the lower index, also across the k-th place), the gathers, and the tgt rows.

Bounded against float64 elsewhere, with u = 2^-24 and ulp32 / ulp16 the spacing of fp32 / the 16-bit output at a value:
  reparametrisation xy = d * w + p      err <= ulp32(d * w) / 2 + ulp32(out) / 2     (a separate product and sum round
                                                                                       twice; a fused one once)
  reparametrisation wh = expf(d) * w    err <= 2^-22 |ref| + ulp32(out) / 2           (expf is within 2 ulp, and
                                                                                       2 ulp32(e^d) <= 2^-22 e^d)
  so wh is within 4.5 ulp of the output.  box_ts and refpoint (from the emitted box_ts) and every decoder layer's
  final_boxes take these bounds.
  sine, element e of a coordinate c (dim = hidden_dim / 2, k = 2 floor(e / 2), x = -log2(1e4) k / dim,
  v = 2 pi c 2^x):  err <= A + E + ulp16(|ref| + A + E) / 2, with A = (7 + 3 ln2 |x|) u |v| the fp32 error of the
  argument: 2pi rounded to fp32 (1 u), the product c * 2pi (1 u), the exponent -13.2877f * k / dim (three roundings,
  3 u |x| in x, so ln2 * 3 u |x| relative after exp2), exp2f (2 ulp = 4 u) and the product with 1/dim_t (1 u); sin and
  cos are 1-Lipschitz.  E = 2^-21.41, the absolute error of __sinf / __cosf, documented for [-pi, pi] only; their range
  reduction (the product with 1/2pi, rounded) adds an error that grows with |v| like the argument's own and has to fit in
  A.  The wide-reference cases run |v| past 500 to check that.  The worst err / bound and the largest |v| are printed per
  output and dtype.

Cases: tiny and large at several sizes, padding masks whose valid sizes put proposal components exactly on 0.01 / 0.99
(50 and 150 tokens), a 1 x 1 pixel and other regions with fewer valid tokens than queries (ties across the k-th place, on
the shared-memory bitonic top-k and on the radix top-k), an explicit all-False mask, raw frames (keep_aspect and explicit
dsts, mask made on the device), a forced selection with a duplicate index, wide reference points, and negative encoder
logits."""
import functools
import math
import os
import sys
from collections import namedtuple

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "lw-detr_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

pytestmark = pytest.mark.gpu

DTYPES = (torch.float16, torch.bfloat16)
U = 2.0 ** -24
SIN_ABS_ERR = 2.0 ** -21.41          # __sinf / __cosf (rowops.cu query_init_kernel)
SIN_ARG_ULPS = 7.0                   # roundings of the fp32 argument besides the exponent's (module docstring)

# mask: None, "zeros" (all False, passed explicitly) or a list of per-image valid (h, w) in pixels, top-left.
# frames: None, ("keep_aspect", [(h, w), ...]) or ("dsts", [(h, w), ...], [(dst_h, dst_w), ...]).
Case = namedtuple("Case", "id name B hw mask variant frames override straddle")


def _case(id, name, B, hw, mask=None, variant="base", frames=None, override=False, straddle=False):
    return Case(id, name, B, hw, mask, variant, frames, override, straddle)


CASES = [
    _case("tiny-640-b2", "tiny", 2, (640, 640)),
    _case("tiny-448x768", "tiny", 1, (448, 768)),
    _case("tiny-128x1344", "tiny", 1, (128, 1344)),
    _case("large-640", "large", 1, (640, 640)),
    _case("large-1024-radix", "large", 1, (1024, 1024)),
    _case("large-1344-radix", "large", 1, (1344, 1344)),
    # valid sizes of exactly 50 tokens: 800 px at P4 (the 800x1333 COCO image on its 832x1344 canvas), 400 px at P3
    _case("tiny-tie50-p4", "tiny", 2, (832, 1344), mask=[(800, 1333), (832, 800)]),
    _case("large-tie50-p3", "large", 2, (640, 640), mask=[(640, 400), (400, 640)]),
    # 150 tokens: 1200 px at P3 (radix top-k)
    _case("large-tie150-p3", "large", 1, (1216, 1216), mask=[(1200, 1200)]),
    # fewer valid tokens than queries: the tied invalid rows straddle the k-th place
    _case("tiny-1px", "tiny", 2, (640, 640), mask=[(1, 1), (640, 640)], straddle=True),
    _case("large-small-bitonic", "large", 1, (640, 640), mask=[(96, 96)], straddle=True),
    _case("large-small-radix", "large", 1, (1024, 1024), mask=[(64, 64)], straddle=True),
    _case("tiny-all-false", "tiny", 2, (640, 640), mask="zeros"),
    _case("tiny-frames-keep-aspect", "tiny", 2, None, frames=("keep_aspect", [(800, 1333), (832, 1100)])),
    _case("large-frames-dsts", "large", 2, (640, 640), frames=("dsts", [(480, 640), (600, 300)], [(400, 640), (640, 200)])),
    _case("tiny-forced", "tiny", 2, (640, 640), override=True),
    _case("large-forced", "large", 1, (640, 640), override=True),
    _case("tiny-wide-refpoints", "tiny", 2, (640, 640), variant="wide"),
    _case("large-wide-refpoints", "large", 1, (640, 640), mask=[(640, 400)], variant="wide"),
    _case("tiny-negative-logits", "tiny", 2, (640, 640), variant="negative"),
]


# ---------------------------------------------------------------------------------------------------------- engines
@functools.lru_cache(maxsize=None)
def _state_dict(name, variant):
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    cfg = CONFIGS[name]
    sd = synth_state_dict(cfg, 1)
    t = "transformer."
    if variant == "wide":
        # reference points to about [-2, 3] and widths of 20 and more: encoder boxes about e^3 * 0.05 * 2^l wide,
        # refpoint_embed spread 5x in xy and shifted by 3 in wh
        sd[t + "enc_out_bbox_embed.0.layers.2.bias"][2:] += 3.0
        sd["refpoint_embed.weight"][:, :2] *= 5.0
        sd["refpoint_embed.weight"][:, 2:] += 3.0
    elif variant == "negative":
        sd[t + "enc_out_class_embed.0.bias"] -= 20.0      # every encoder logit below zero
    return cfg, sd


_ENGINES = {}


def _engine(name, dt, variant):
    from b200 import capi
    key = (name, dt, variant)
    if key not in _ENGINES:
        cfg, sd = _state_dict(name, variant)
        eng = capi.Engine(cfg, dt)
        eng.load_state_dict(sd)
        _ENGINES[key] = eng
    cfg, sd = _state_dict(name, variant)
    return cfg, sd, _ENGINES[key]


# --------------------------------------------------------------------------------------------------------- helpers
def _ulp(x, mant, emin):
    """Spacing of a binary format with `mant` fraction bits and minimum normal exponent emin at |x| (x float64 array)."""
    a = np.abs(np.asarray(x, dtype=np.float64))
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    e = np.where(a > 0, np.maximum(e, emin), emin)
    return np.ldexp(1.0, (e - mant).astype(np.int32))


def ulp32(x):
    return _ulp(x, 23, -126)


def ulp16(x, dt):
    return _ulp(x, 10, -14) if dt == torch.float16 else _ulp(x, 7, -126)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_bits(got, want, what):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero(bits(got).reshape(-1) != bits(want).reshape(-1))[0]
    assert bad.size == 0, "%s: %d of %d elements differ, first at flat %d: got %r, want %r" % (
        what, bad.size, got.size, bad[0], got.reshape(-1)[bad[0]], want.reshape(-1)[bad[0]])


RATIOS = {}


def _note(what, dt, value):
    key = (what, "fp16" if dt == torch.float16 else "bf16")
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(value))


def check_bound(got, ref, bound, what, dt):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    bad = ~(err <= bound)                                   # NaN fails too
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError("%s: %d elements outside the bound, first %s: got %r, float64 %r, err %.3e, bound %.3e" % (
            what, int(bad.sum()), tuple(i), got[tuple(i)], ref[tuple(i)], err[tuple(i)], bound[tuple(i)]))
    return err / bound


def reparam_check(delta, ref_box, got, what, dt):
    """got = reparam(delta, ref_box) (fp32 inputs [n, 4]) within the module docstring's bounds."""
    d, r = delta.astype(np.float64), ref_box.astype(np.float64)
    dw = d[:, :2] * r[:, 2:]
    want = np.concatenate([dw + r[:, :2], np.exp(d[:, 2:]) * r[:, 2:]], 1)
    mag = np.maximum(np.abs(want), np.abs(got.astype(np.float64)))
    bound = np.concatenate([0.5 * ulp32(dw) + 0.5 * ulp32(mag[:, :2]),
                            2.0 ** -22 * np.abs(want[:, 2:]) + 0.5 * ulp32(mag[:, 2:])], 1)
    r = check_bound(got, want, bound, what, dt)
    _note(what + " xy", dt, r[:, :2].max())
    _note(what + " wh", dt, r[:, 2:].max())


# ----------------------------------------------------------------------------------------------- padding tables
def mask_tables(mask, B, H, W, level_shapes):
    """numpy float32 restatement of mask_setup: per image and level the nearest resize of the mask (F.interpolate's
    source index min(floor(i * (H / h)), H - 1) in fp32), valid counts of the first column / row, valid ratios (w, h),
    proposals ((j + .5) / valid_w, (i + .5) / valid_h, .05 * 2^l, .05 * 2^l), kept when every component is strictly inside
    (0.01, 0.99) and the token is not padding.  mask: bool [B, H, W] or None.  -> proposals [B*S, 4], invalid [B*S],
    pad [B*S], valid_ratio [B*L, 2]."""
    f32 = np.float32
    props, inval, pads = [], [], []
    vr = np.zeros((B, len(level_shapes), 2), f32)
    for l, (h, w) in enumerate(level_shapes):
        if mask is None:
            lm = np.zeros((B, h, w), bool)
        else:
            yi = np.minimum(np.floor(np.arange(h, dtype=f32) * (f32(H) / f32(h))).astype(np.int64), H - 1)
            xi = np.minimum(np.floor(np.arange(w, dtype=f32) * (f32(W) / f32(w))).astype(np.int64), W - 1)
            lm = mask[:, yi][:, :, xi]
        vh = (~lm[:, :, 0]).sum(1).astype(f32)
        vw = (~lm[:, 0, :]).sum(1).astype(f32)
        vr[:, l, 0], vr[:, l, 1] = vw / f32(w), vh / f32(h)
        cx = (np.arange(w, dtype=f32)[None, None, :] + f32(0.5)) / vw[:, None, None]
        cy = (np.arange(h, dtype=f32)[None, :, None] + f32(0.5)) / vh[:, None, None]
        whv = f32(0.05) * f32(2.0 ** l)
        v = np.stack(np.broadcast_arrays(cx, cy, whv, whv), -1).astype(f32)          # [B, h, w, 4]
        keep = ((v > f32(0.01)) & (v < f32(0.99))).all(-1) & ~lm
        props.append(np.where(keep[..., None], v, f32(0)).reshape(B, h * w, 4))
        inval.append((~keep).reshape(B, h * w))
        pads.append(lm.reshape(B, h * w))
    return (np.concatenate(props, 1).reshape(-1, 4), np.concatenate(inval, 1).reshape(-1).astype(f32),
            np.concatenate(pads, 1).reshape(-1).astype(f32), vr.reshape(-1, 2))


def oracle_tables(mask, cfg, B, H, W):
    """The same tables from the oracle (encoder_proposals / level_padding_masks) through oracle_hw's config view."""
    import oracle_hw
    from oracle import lwdetr_oracle as orc
    cv = oracle_hw.AtInputSize(cfg, H, W)
    if mask is None or not mask.any():
        props, valid = orc.encoder_proposals(cv, torch.float32)
        S = props.shape[0]
        props, keep = props[None].expand(B, S, 4), valid[None, :, 0].expand(B, S)
        pad = torch.zeros(B, S, dtype=torch.bool)
        vr = torch.ones(B, cfg.n_levels, 2)
    else:
        lm = orc.level_padding_masks(torch.from_numpy(mask), cv)
        props, keep = orc.encoder_proposals(cv, torch.float32, lm)
        keep = keep[..., 0]
        pad = torch.cat([m.flatten(1) for m in lm], 1)
        vr = torch.stack([torch.stack([(~m[:, 0, :]).sum(1).float() / m.shape[2], (~m[:, :, 0]).sum(1).float() / m.shape[1]], -1)
                          for m in lm], 1)
    return (props.reshape(-1, 4).numpy(), (~keep).reshape(-1).float().numpy(), pad.reshape(-1).float().numpy(),
            vr.reshape(-1, 2).numpy())


# ------------------------------------------------------------------------------------------------------- one case
def _host_mask(c, B, H, W):
    if c.mask is None:
        return None
    m = np.zeros((B, H, W), bool)
    if c.mask != "zeros":
        for b, (vh, vw) in enumerate(c.mask):
            m[b, vh:, :] = True
            m[b, :, vw:] = True
    return m


def _frames(c):
    g = torch.Generator(device="cuda").manual_seed(7)
    return [torch.randint(0, 256, (h, w, 3), device="cuda", dtype=torch.uint8, generator=g) for h, w in c.frames[1]]


def run_case(c, dt):
    cfg, sd, eng = _engine(c.name, dt, c.variant)
    B, nq, d, ncls, NL, L = c.B, cfg.num_queries, cfg.hidden_dim, cfg.num_classes, cfg.dec_layers, cfg.n_levels
    ov = None
    if c.frames is not None:
        frames = _frames(c)
        kw = dict(fit="keep_aspect", short_side=800, max_side=1333) if c.frames[0] == "keep_aspect" else dict(dsts=c.frames[2], size=c.hw)
        from b200.config import explicit_frame_sizes, frame_sizes
        if c.frames[0] == "keep_aspect":
            (H, W), dsts = frame_sizes(cfg, [f.shape[:2] for f in frames], None, **kw)
        else:
            (H, W), dsts = explicit_frame_sizes(cfg, B, c.frames[2], c.hw)
        mask = np.zeros((B, H, W), bool)
        for b, (dh, dw) in enumerate(dsts):
            mask[b, dh:, :] = True
            mask[b, :, dw:] = True
    else:
        H, W = c.hw
        mask = _host_mask(c, B, H, W)
    S = cfg.memory_len_at(H, W)
    BS, BQ = B * S, B * nq
    sizes = {"mask_setup": BS * 4, "mask_setup.invalid": BS, "mask_setup.pad": BS, "mask_setup.valid_ratio": B * L * 2,
             "enc_output_norm": BS * d, "enc_class": BS * ncls, "enc_score": BS, "topk": BQ,
             "gather_topk": BQ * d, "gather_topk.enc_logits": BQ * ncls, "enc_box2": BQ * 4,
             "query_init": BQ * 4, "query_init.box_ts": BQ * 4, "query_init.sine": BQ * 2 * d, "query_pos": BQ * d,
             "tgt_init": BQ * d, "tgt_plus_pos": BQ * d, "bbox2": NL * BQ * 4, "final_boxes": NL * BQ * 4}
    eng.clear_captures()
    for lab, n in sizes.items():
        eng.capture(lab, n)
    if c.override:
        g = torch.Generator(device="cuda").manual_seed(11)
        ov = torch.randint(0, S, (B, nq), device="cuda", generator=g, dtype=torch.int64)
        ov[0, 17] = ov[0, 5]                      # a duplicate: two queries start from the same memory row
        ov[0, 0], ov[-1, -1] = 0, S - 1           # both ends of the memory
    if c.frames is not None:
        res = eng.forward_frames(frames, topk_override=ov, **kw)
        assert [tuple(x) for x in res["frame_sizes"]] == [tuple(x) for x in dsts]
    else:
        from b200.synth import synth_images
        x = synth_images(B, 3, (H, W)).cuda()
        res = eng.forward(x, topk_override=ov, mask=None if mask is None else torch.from_numpy(mask).cuda())
    torch.cuda.synchronize()
    got = eng.capture_results()
    eng.clear_captures()
    for lab, n in sizes.items():
        assert got[lab] is not None and got[lab].numel() == n, (lab, None if got[lab] is None else got[lab].numel(), n)
    got = {k: v.numpy() for k, v in got.items()}

    # ---- mask_setup: all four tables bit for bit, against numpy and against the oracle
    want = mask_tables(mask, B, H, W, cfg.level_shapes_at(H, W))
    have = (got["mask_setup"].reshape(-1, 4), got["mask_setup.invalid"], got["mask_setup.pad"], got["mask_setup.valid_ratio"].reshape(-1, 2))
    for nm, g_, w_, o_ in zip(("proposals", "invalid", "pad", "valid_ratio"), have, want, oracle_tables(mask, cfg, B, H, W)):
        assert_bits(g_, w_, "mask_setup %s vs numpy" % nm)
        assert_bits(g_, o_, "mask_setup %s vs oracle" % nm)
    props, invalid, vr = have[0], have[1], have[3].reshape(B, L, 2)

    # ---- enc_output_norm: the rows flagged invalid are one and the same row
    omn = got["enc_output_norm"].reshape(BS, d)
    inv_rows = np.nonzero(invalid)[0]
    if inv_rows.size > 1:
        assert_bits(omn[inv_rows], np.broadcast_to(omn[inv_rows[0]], (inv_rows.size, d)), "enc_output_norm invalid rows")

    # ---- enc_score: max over the class logits, which start from -inf
    cls = got["enc_class"].reshape(BS, ncls)
    score = got["enc_score"]
    assert_bits(score, cls.max(1), "enc_score")
    if c.variant == "negative":
        assert (score < 0).all()

    # ---- topk: a stable descending sort of the captured score (ties to the lower index)
    topk = got["topk"].reshape(B, nq).astype(np.int64)
    if ov is None:
        srt = torch.sort(torch.from_numpy(score.reshape(B, S)), dim=1, descending=True, stable=True)
        assert np.array_equal(topk, srt.indices[:, :nq].numpy()), "topk differs from a stable descending sort"
        if c.straddle:
            v = srt.values.numpy()
            assert (v[:, nq - 1] == v[:, nq]).any(), "the case was meant to put a tie across the k-th place"
    else:
        assert np.array_equal(topk, ov.cpu().numpy()), "topk does not follow the override"
    assert np.array_equal(res["topk_index"].cpu().numpy(), topk), "aux topk_index differs from the captured selection"
    rows = (np.arange(B)[:, None] * S + topk).reshape(-1)

    # ---- gather_topk: rows of enc_output_norm (16-bit) and of enc_class (fp32) at the selection
    assert_bits(got["gather_topk"].reshape(BQ, d), omn[rows], "gather_topk sel")
    assert_bits(got["gather_topk.enc_logits"].reshape(BQ, ncls), cls[rows], "gather_topk enc_logits")
    assert_bits(res["enc_outputs"]["pred_logits"].cpu().numpy().reshape(BQ, ncls), cls[rows], "enc_outputs pred_logits")

    # ---- query_init: box_ts on the proposals, refpoint on the emitted box_ts, the sine embedding of the scaled refpoint
    box_ts = got["query_init.box_ts"].reshape(BQ, 4)
    reparam_check(got["enc_box2"].reshape(BQ, 4), props[rows], box_ts, "box_ts", dt)
    assert_bits(res["enc_outputs"]["pred_boxes"].cpu().numpy().reshape(BQ, 4), box_ts, "enc_outputs pred_boxes")
    rpe = sd["refpoint_embed.weight"][:nq].float().numpy()
    refpoint = got["query_init"].reshape(BQ, 4)
    reparam_check(np.tile(rpe, (B, 1)), box_ts, refpoint, "refpoint", dt)
    check_sine(refpoint, vr[:, 0, :], got["query_init.sine"].reshape(BQ, 2 * d), B, nq, d, dt)

    # ---- tgt_init / tgt_plus_pos
    qf = sd["query_feat.weight"][:nq].to(dt).float()
    assert_bits(got["tgt_init"].reshape(BQ, d), qf.repeat(B, 1).numpy(), "tgt_init")
    qpos = torch.from_numpy(got["query_pos"].reshape(BQ, d))
    assert_bits(got["tgt_plus_pos"].reshape(BQ, d), (qf.repeat(B, 1) + qpos).to(dt).float().numpy(), "tgt_plus_pos")

    # ---- final_boxes: every decoder layer's bbox delta on the refpoint
    fb = got["final_boxes"].reshape(NL * BQ, 4)
    reparam_check(got["bbox2"].reshape(NL * BQ, 4), np.tile(refpoint, (NL, 1)), fb, "final_boxes", dt)
    assert_bits(res["pred_boxes"].cpu().numpy().reshape(BQ, 4), fb[(NL - 1) * BQ:], "pred_boxes")
    for i, a in enumerate(res["aux_outputs"]):
        assert_bits(a["pred_boxes"].cpu().numpy().reshape(BQ, 4), fb[i * BQ:(i + 1) * BQ], "aux pred_boxes %d" % i)


def check_sine(refpoint, vr0, sine, B, nq, d, dt):
    """query_init.sine against float64 sin / cos of 2 pi rp / 10000^(2 floor(e/2) / dim), rp = refpoint * level-0 valid
    ratio (w, h, w, h) as the kernel forms it (one fp32 product), coordinates in the order (y, x, w, h)."""
    dim = d // 2
    rp = refpoint.reshape(B, nq, 4) * np.concatenate([vr0, vr0], 1)[:, None, :]        # fp32 product
    rp = rp.reshape(B * nq, 4).astype(np.float64)
    coord = rp[:, [1, 0, 2, 3]]                                                        # [BQ, 4] in output order
    e = np.arange(dim)
    k = 2 * (e // 2)
    x = -math.log2(10000.0) * k / dim                                                 # exponent of 1/dim_t
    v = 2 * math.pi * coord[:, :, None] * np.exp2(x)[None, None, :]                   # [BQ, 4, dim]
    ref = np.where((e % 2 == 0)[None, None, :], np.sin(v), np.cos(v)).reshape(B * nq, 2 * d)
    arg = ((SIN_ARG_ULPS + 3 * math.log(2) * np.abs(x))[None, None, :] * U * np.abs(v) * (1 + 2.0 ** -20)).reshape(B * nq, 2 * d)
    a = arg + SIN_ABS_ERR
    bound = a + 0.5 * ulp16(np.abs(ref) + a, dt)
    _note("sine", dt, check_bound(sine, ref, bound, "sine", dt).max())
    _note("|v| max", dt, np.abs(v).max())


# ---------------------------------------------------------------------------------------------------------- the tests
@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    _ENGINES.clear()
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    cm = request.config.pluginmanager.get_plugin("capturemanager")
    if tr is None or cm is None or not RATIOS:
        return
    with cm.global_and_fixture_disabled():
        tr.write_line("")
        for (what, dt), r in sorted(RATIOS.items()):
            tr.write_line("query selection %-12s %s: max %s %.4g" % (what, dt, "value" if what.startswith("|") else "err/bound", r))


@pytest.mark.parametrize("dt", DTYPES, ids=("fp16", "bf16"))
@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_query_selection_op_by_op(c, dt):
    run_case(c, dt)
