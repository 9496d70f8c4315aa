"""GPU tests of inference at input sizes other than 640x640 (lwdetr_forward_hw): the parity ladder against the oracle,
engine output against the reference's own goldens, re-planning between shapes, batch consistency, and the kernels that
change with the input size (streaming top-k, direct-gather deformable attention, non-square patch gather / unwindow,
per-resolution position table)."""
import ctypes
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))

from test_model_gpu import TOL, parity_rel  # noqa: E402



def _tol(dt, tokens):
    """TOL of test_model_gpu up to the 1600 tokens of a 640x640 input.  Above that the deviation of the final logits / boxes
    from the fp32 oracle grows with the token count (measured on an H100: large at 1024x1024 and xlarge at 768x1344 reach
    fp16 boxes 1.1e-3 and bf16 logits rel-L2 7.0e-3; tiny at 832x1344, 4368 tokens, reaches 6.03e-3 on the staged kernels
    too), so the two bars the suite already uses for larger workloads apply: the autocast-derived (AC3) logits rel-L2 and
    boxes_big."""
    tol = dict(TOL[dt])
    if tokens > 1600:
        tol["logits_rel"] = 1.8e-3 if dt == torch.float16 else 1.5e-2
        tol["boxes"] = tol["boxes_big"]
    return tol


LADDER = [("tiny", 2, (512, 512)), ("small", 1, (448, 768)), ("large", 1, (1024, 1024)), ("xlarge", 1, (768, 1344)),
          ("small", 1, (256, 1344))]


def _engine(name, dt, img_size=None, wseed=1):
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    cfg = CONFIGS[name] if img_size is None else dataclasses.replace(CONFIGS[name], img_size=img_size)
    eng = capi.Engine(cfg, dt)
    sd = synth_state_dict(cfg, wseed)
    eng.load_state_dict(sd)
    return cfg, sd, eng


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name,batch,hw", LADDER)
def test_parity_ladder_at_resolution(name, batch, hw, dt):
    import parity_report
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    rep = parity_report.ladder(name, batch, dt, hw=hw)
    tol = _tol(dt, (hw[0] // 16) * (hw[1] // 16))
    t1, t2, t3 = rep["T1"], rep["T2"], rep["T3"]
    for k, v in t1.items():
        if k.startswith("block") or k == "patch_embed":
            assert v <= tol["block"], (k, v)
        elif k.startswith("level") or k == "memory":
            assert v <= tol["memory"], (k, v)
    assert t1["enc_score_maxabs"] <= tol["score"], t1
    assert t2["topk_echo_ok"]
    for k, v in t2.items():
        if k.endswith("logits_rel_l2"):
            assert v <= tol["logits_rel"], (k, v)
        elif k.endswith("logits_maxabs"):
            assert v <= tol["logits_abs"], (k, v)
        elif k.endswith("boxes_maxabs"):
            assert v <= tol["boxes"], (k, v)
        elif k.startswith("dec") or k == "query_pos":
            assert v <= tol["dec"], (k, v)
    assert t3["finite"]
    assert t3["set_agreement_min"] >= 0.95, t3


def _check_against_golden(forced, g, dt, tokens, enc_logits=True):
    tol = _tol(dt, tokens)
    gl, gb = torch.from_numpy(g["pred_logits"]), torch.from_numpy(g["pred_boxes"])
    assert parity_rel(forced["pred_logits"].cpu(), gl) <= tol["logits_rel"]
    assert (forced["pred_logits"].cpu() - gl).abs().max().item() <= tol["logits_abs"]
    assert (forced["pred_boxes"].cpu() - gb).abs().max().item() <= tol["boxes"]
    assert (forced["enc_outputs"]["pred_boxes"].cpu() - torch.from_numpy(g["enc_boxes"])).abs().max().item() <= tol["boxes"]
    if enc_logits:
        assert (forced["enc_outputs"]["pred_logits"].cpu() - torch.from_numpy(g["enc_logits"])).abs().max().item() <= tol["logits_abs"]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name,H,W", [("tiny", 512, 512), ("small", 448, 768), ("large", 1024, 1024), ("xlarge", 768, 1344)])
def test_engine_matches_reference_golden_at_resolution(name, H, W, dt):
    """The engine against the UNMODIFIED reference's outputs (two-stage indices forced to the oracle's, which meets the
    golden to 1e-4 on the CPU), plus free-running selection agreement."""
    import oracle_hw
    from b200.synth import synth_images
    g = np.load(os.path.join(GOLD, "ref_res_%s_%dx%d.npz" % (name, H, W)))
    B, wseed, iseed, _, _, img_size = (int(v) for v in g["meta"])
    cfg, sd, eng = _engine(name, dt, img_size, wseed)
    x = synth_images(B, iseed, (H, W))
    inter = {}
    oracle_hw.forward(sd, cfg, x, inter=inter)
    forced = eng.forward(x.cuda(), topk_override=inter["topk"])
    _check_against_golden(forced, g, dt, (H // 16) * (W // 16))
    free = eng.forward(x.cuda())
    ti = free["topk_index"].cpu().long()
    for b in range(B):
        assert len(set(ti[b].tolist()) & set(inter["topk"][b].tolist())) >= 0.95 * cfg.num_queries
    eng.close()


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_padded_coco_sized_batch_matches_reference_golden(dt):
    """800x1333 and 832x1100 images: the module pads the batch to 832x1344 (each side up to a multiple of 64) with the
    NestedTensor mask, and the engine meets the reference's output on that canvas."""
    import make_goldens
    import oracle_hw
    from models.lwdetr import LWDETR
    from util.misc import nested_tensor_from_tensor_list
    g = np.load(os.path.join(GOLD, "ref_res_tiny_832x1344_padded.npz"))
    B, wseed, iseed, H, W, img_size = (int(v) for v in g["meta"])
    cfg, sd, eng = _engine("tiny", dt, img_size, wseed)
    x, mask = make_goldens.res_padded_inputs()
    inter = {}
    oracle_hw.forward(sd, cfg, x, mask=mask, inter=inter)
    forced = eng.forward(x.cuda(), mask=mask.cuda(), topk_override=inter["topk"])
    _check_against_golden(forced, g, dt, (H // 16) * (W // 16), enc_logits=False)
    free = eng.forward(x.cuda(), mask=mask.cuda())
    free = {k: v.clone() for k, v in free.items() if k.startswith("pred")}
    model = LWDETR(cfg, compute_dtype=dt).eval()
    model.load_state_dict(sd, strict=True)
    model.cuda()
    imgs = [x[b][:, :h, :w].cuda() for b, (h, w) in enumerate(make_goldens.RES_PADDED[4])]
    out = model(nested_tensor_from_tensor_list(imgs))
    assert torch.equal(out["pred_logits"], free["pred_logits"]) and torch.equal(out["pred_boxes"], free["pred_boxes"])
    eng.close()


def _forward_ex(eng, x):
    """lwdetr_forward_ex (the configured-size entry point) on an fp32 NCHW batch."""
    from b200 import capi
    B, nq, nc = x.shape[0], eng.cfg.num_queries, eng.cfg.num_classes
    logits = torch.empty(B, nq, nc, device="cuda")
    boxes = torch.empty(B, nq, 4, device="cuda")
    desc = capi.InputDesc()
    desc.images, desc.format, desc.padding_mask = x.data_ptr(), capi.IN_F32_NCHW, None
    capi.check(capi.lib().lwdetr_forward_ex(eng._h, ctypes.byref(desc), B, capi.ptr(logits), capi.ptr(boxes), None, None,
                                            capi.stream_ptr()), "lwdetr_forward_ex")
    return logits, boxes


@pytest.mark.parametrize("name", ["small", "large"])
def test_forward_hw_at_configured_size_equals_forward_ex(name):
    from b200.synth import synth_images
    cfg, sd, eng = _engine(name, torch.float16)
    x = synth_images(2, 7).cuda()
    a = eng.forward(x, want_aux=False)
    a = {k: v.clone() for k, v in a.items()}
    lb, bb = _forward_ex(eng, x)
    torch.cuda.synchronize()
    assert torch.equal(a["pred_logits"], lb) and torch.equal(a["pred_boxes"], bb)
    eng.close()


def test_shape_cycle_with_cuda_graph_matches_fresh_engines():
    """One engine cycles 640 -> 1024x1024 -> 448x768 -> 640 with CUDA graphs on (each shape re-plans and drops the graphs);
    every output equals that of a fresh engine planned only for that shape."""
    from b200.synth import synth_images
    shapes = [(640, 640), (1024, 1024), (448, 768), (640, 640)]
    xs = {hw: synth_images(1, 13, hw).cuda() for hw in set(shapes)}
    fresh = {}
    for hw in set(shapes):
        _, _, e = _engine("large", torch.float16)
        o = e.forward(xs[hw], want_aux=False)
        fresh[hw] = {k: v.clone() for k, v in o.items()}
        e.close()
    _, _, eng = _engine("large", torch.float16)
    eng.set_option("cuda_graph", 1)
    for hw in shapes:
        for rep in range(3):                       # eager first run of a plan, then graph capture, then replay
            o = eng.forward(xs[hw], want_aux=False)
            torch.cuda.synchronize()
            assert torch.equal(o["pred_logits"], fresh[hw]["pred_logits"]), (hw, rep)
            assert torch.equal(o["pred_boxes"], fresh[hw]["pred_boxes"]), (hw, rep)
    eng.close()


def test_large_batch_at_1024_is_consistent_with_small_batches():
    """large at 1024x1024 (streaming top-k, direct-gather deformable attention): B = 8 predictions agree with B = 2 slices."""
    from b200.synth import synth_images
    _, _, eng = _engine("large", torch.float16)
    batch = 8
    x = synth_images(batch, 3, (1024, 1024)).cuda()
    big = {k: v.clone() for k, v in eng.forward(x, want_aux=True).items() if k in ("pred_logits", "pred_boxes", "topk_index")}
    assert torch.isfinite(big["pred_logits"]).all() and torch.isfinite(big["pred_boxes"]).all()
    assert (big["pred_boxes"][..., 2:] > 0).all()
    for lo in (0, batch - 2):
        small = eng.forward(x[lo:lo + 2].contiguous(), want_aux=True)
        same_sel = (small["topk_index"] == big["topk_index"][lo:lo + 2])
        for i in range(2):
            a, b = set(small["topk_index"][i].tolist()), set(big["topk_index"][lo + i].tolist())
            assert len(a & b) >= 0.95 * len(a), (lo, i, len(a & b))
        rows = same_sel.all(dim=1)
        if rows.any():
            dl = (small["pred_logits"][rows] - big["pred_logits"][lo:lo + 2][rows]).abs().max().item()
            db = (small["pred_boxes"][rows] - big["pred_boxes"][lo:lo + 2][rows]).abs().max().item()
            assert dl <= 2.1e-2 and db <= 8.5e-4, (dl, db)
    eng.close()


# ------------------------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("S", [1600, 6800, 16384, 17408, 29988])
@pytest.mark.parametrize("kind", ["random", "ties"])
def test_topk_any_length(S, kind):
    from b200 import capi
    g = torch.Generator(device="cuda").manual_seed(S)
    B, k = 3, 300
    if kind == "random":
        score = torch.randn(B, S, device="cuda", generator=g)
    else:                                          # few distinct values, signed zeros: ties everywhere, also at the threshold
        score = torch.randint(-3, 4, (B, S), device="cuda", generator=g).float() * 0.5
        score[0, ::7] = -0.0
        score[1] = 1.0                             # a whole row of one value
    idx = capi.topk(score, k).long()
    vals, ref = torch.sort(score, dim=1, descending=True, stable=True)       # host order (-key, index)
    assert torch.equal(idx, ref[:, :k])
    assert torch.equal(torch.gather(score, 1, idx), vals[:, :k])


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_msda_direct_gather_path(dt):
    """A level set the staged kernel cannot hold (168x168 + 42x42, the large/xlarge levels at 1344x1344): the direct-gather
    kernel against fp32 math, with samples outside the levels and valid ratios."""
    from b200 import capi
    from oracle import lwdetr_oracle as orc
    B, Lq, M, L, P, shapes = 2, 300, 24, 2, 4, [(168, 168), (42, 42)]
    g = torch.Generator().manual_seed(17)
    d, S = M * 16, sum(h * w for h, w in shapes)
    value = torch.randn(B, S, d, generator=g).to(dt)
    ol = torch.cat([torch.randn(B * Lq, M * L * P * 2, generator=g) * 2.0, torch.randn(B * Lq, M * L * P, generator=g) * 2.0], 1).to(dt)
    ref_box = torch.rand(B * Lq, 4, generator=g) * torch.tensor([1.2, 1.2, 0.6, 0.6]) - torch.tensor([0.1, 0.1, 0.0, 0.0])
    vr = torch.tensor([[[1.0, 1.0], [1.0, 1.0]], [[0.8, 0.65], [0.8, 0.7]]])
    out = torch.full((B * Lq, d), float("nan"), dtype=dt, device="cuda")
    capi.msda_forward(capi.value_to_head_major(value.cuda().reshape(B * S, d), B, S, M), ol.cuda(), ref_box.cuda(), out, B, S, Lq,
                      M, L, P, shapes, valid_ratio=vr.cuda().contiguous())
    off = ol[:, :M * L * P * 2].float().reshape(B, Lq, M, L, P, 2)
    aw = ol[:, M * L * P * 2:].float().reshape(B, Lq, M, L * P).softmax(-1).reshape(B, Lq, M, L, P)
    rb = ref_box.reshape(B, Lq, 1, 4) * torch.cat([vr, vr], -1)[:, None]
    loc = rb[:, :, None, :, None, :2] + off / P * rb[:, :, None, :, None, 2:] * 0.5
    assert ((loc < 0) | (loc > 1)).any()                       # some samples fall outside the levels
    ref = orc.msda_core(value.float().reshape(B, S, M, 16), shapes, loc, aw).reshape(B * Lq, d)
    tol = 3e-3 if dt == torch.float16 else 2e-2
    assert (out.float().cpu() - ref).abs().max().item() <= tol * max(ref.abs().max().item(), 1.0)
    assert ((out.float().cpu() - ref).norm() / ref.norm()).item() <= (1e-3 if dt == torch.float16 else 8e-3)


def _window_major(x):
    """[B, GH, GW, C] -> [B*GH*GW, C] in window-major token order (vit.py:353-358)."""
    from oracle import lwdetr_oracle as orc
    return orc.to_window_major(x).reshape(-1, x.shape[-1])


def _patches(x):
    """[B, 3, H, W] -> [B, GH, GW, 768] with k = c*256 + py*16 + px."""
    B, _, H, W = x.shape
    return x.reshape(B, 3, H // 16, 16, W // 16, 16).permute(0, 2, 4, 1, 3, 5).reshape(B, H // 16, W // 16, 768)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_nonsquare_patch_gather_and_unwindow_are_exact_permutations(dt):
    """Patch gather (fp32, 16-bit and uint8 input) and the un-windowing copy of the P5 level at 448x768, captured from the
    engine's schedule and compared bit for bit with a torch permutation of the same values."""
    from b200 import capi
    from b200.config import CONFIGS
    cfg, _, eng = _engine("large", dt)
    B, H, W = 2, 448, 768
    GH, GW, C = H // 16, W // 16, cfg.vit_dim
    BT = B * GH * GW
    g = torch.Generator().manual_seed(5)
    u8 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    mean, std = torch.tensor(capi.IMAGENET_MEAN), torch.tensor(capi.IMAGENET_STD)
    f32 = ((u8.float() / 255.0 - mean) / std).permute(0, 3, 1, 2).contiguous()
    want = _window_major(_patches(f32.to(dt))).float()
    ntap = len(cfg.taps)
    for inp in (f32, f32.to(dt), u8):
        eng.clear_captures()
        eng.capture("patch_gather", BT * 768)
        for t in cfg.taps:
            eng.capture("block%d" % t, BT * C)
        eng.capture("level1.unwindow", BT * ntap * C)
        eng.forward(inp.cuda(), want_aux=False)
        torch.cuda.synchronize()
        got = eng.capture_results()
        assert torch.equal(got["patch_gather"].reshape(BT, 768), want), inp.dtype
        spatial = torch.cat([orc_from_window_major(got["block%d" % t].reshape(B * 16, -1, C), B, GH, GW) for t in cfg.taps], -1)
        assert torch.equal(got["level1.unwindow"].reshape(B, GH, GW, ntap * C), spatial)
    eng.clear_captures()
    eng.close()
    assert CONFIGS["large"].projector_scale[1] == "P5"


def orc_from_window_major(x, B, H, W):
    from oracle import lwdetr_oracle as orc
    return orc.from_window_major(x, B, H, W)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("hw", [(448, 768), (1344, 256), (640, 640)])
def test_position_table_per_resolution(dt, hw):
    """With the patch-embedding weights and bias zeroed, the patch-embed output IS the position table: it equals
    F.interpolate(pos_embed, (H/16, W/16), bicubic) in window-major order, rounded to the compute dtype."""
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    cfg = CONFIGS["small"]
    sd = synth_state_dict(cfg, 1)
    sd["backbone.0.encoder.patch_embed.proj.weight"] = torch.zeros_like(sd["backbone.0.encoder.patch_embed.proj.weight"])
    sd["backbone.0.encoder.patch_embed.proj.bias"] = torch.zeros_like(sd["backbone.0.encoder.patch_embed.proj.bias"])
    eng = capi.Engine(cfg, dt)
    eng.load_state_dict(sd)
    H, W = hw
    GH, GW, C = H // 16, W // 16, cfg.vit_dim
    eng.capture("patch_embed", GH * GW * C)
    eng.forward(torch.zeros(1, 3, H, W, device="cuda"), want_aux=False)
    torch.cuda.synchronize()
    got = eng.capture_results()["patch_embed"].reshape(GH * GW, C)
    pe = sd["backbone.0.encoder.pos_embed"][0, 1:].reshape(1, 14, 14, C).permute(0, 3, 1, 2)
    ref = F.interpolate(pe, size=(GH, GW), mode="bicubic", align_corners=False).permute(0, 2, 3, 1)
    want = _window_major(ref).to(dt).float()
    ulp = 2.0 ** -10 if dt == torch.float16 else 2.0 ** -7                  # one rounding step of the compute dtype
    assert ((got - want).abs() <= ulp * want.abs() + 1e-6).all()
    assert ((got == want).float().mean().item()) > 0.99
    eng.close()


def test_unsupported_shapes_raise():
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR
    cfg, sd, eng = _engine("small", torch.float16)
    for shape, msg in (((1, 3, 640, 650), "multiples of 64"), ((1, 3, 1408, 640), "1344"), ((1, 3, 64, 640), "multiples of 64"),
                       ((1, 3, 128, 256), "num_queries")):
        with pytest.raises(RuntimeError, match=msg):
            eng.forward(torch.zeros(shape, device="cuda"))
    # the C ABI checks on its own (callers that bypass the Python surface)
    desc = capi.InputDesc()
    x = torch.zeros(1, 3, 640, 704, device="cuda")
    desc.images, desc.format, desc.padding_mask = x.data_ptr(), capi.IN_F32_NCHW, None
    out = torch.empty(1, cfg.num_queries, cfg.num_classes + 4, device="cuda")
    for h, w in ((640, 650), (1408, 640), (128, 256)):
        rc = capi.lib().lwdetr_forward_hw(eng._h, ctypes.byref(desc), 1, h, w, capi.ptr(out), capi.ptr(out), None, None, capi.stream_ptr())
        assert rc != 0 and capi.lib().lwdetr_last_error().decode()
    # the engine still runs after the rejected calls
    o = eng.forward(x, want_aux=False)
    assert torch.isfinite(o["pred_logits"]).all()
    eng.close()
    model = LWDETR(CONFIGS["tiny"], compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(CONFIGS["tiny"], 1), strict=True)
    model.cuda()
    with pytest.raises(RuntimeError, match="uint8"):
        model(torch.zeros(1, 512, 640, 3, dtype=torch.uint8, device="cuda"))      # uint8 smaller than img_size
    with pytest.raises(RuntimeError, match="1344"):
        model(torch.zeros(1, 3, 640, 1400, device="cuda"))
    out = model(torch.zeros(1, 704, 896, 3, dtype=torch.uint8, device="cuda"))      # uint8 at a larger 64-multiple runs
    assert out["pred_logits"].shape == (1, 100, 91)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_broadcast_weights_position_table_follows_the_root():
    """After lwdetr_broadcast_weights, rank 1 (loaded with different weights) plans a 1024x1024 forward bit-identical to
    rank 0's: the per-resolution position table is derived from the arena, not from the rank's host copy."""
    import torch.multiprocessing as mp
    mp.spawn(_bcast_worker, nprocs=2, join=True)


def _bcast_worker(rank):
    import tempfile
    import torch.distributed as dist
    from b200.dist import broadcast_engine_weights
    from b200.synth import synth_images
    torch.cuda.set_device(rank)
    store = os.path.join(tempfile.gettempdir(), "lwdetr_res_bcast_%d" % os.getppid())
    dist.init_process_group("nccl", init_method="file://" + store, rank=rank, world_size=2)
    _, _, eng = _engine("large", torch.float16, wseed=1 if rank == 0 else 2)
    broadcast_engine_weights(eng, torch.device("cuda", rank), src=0)
    o = eng.forward(synth_images(1, 4, (1024, 1024)).cuda(), want_aux=False)
    res = torch.cat([o["pred_logits"].flatten(), o["pred_boxes"].flatten()])
    allr = [torch.empty_like(res) for _ in range(2)]
    dist.all_gather(allr, res)
    assert torch.equal(allr[0], allr[1])
    eng.close()
    dist.destroy_process_group()
