"""The e4m3 encoder mode (LWDETR_F16_E4M3) on the GPU: its two kernels against float64 restatements, the whole forward
against the mode's own CPU spec (tools/oracle_fp8.py) and the fp32 oracle, and the mode through every public path."""
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle_fp8  # noqa: E402
import oracle_hw  # noqa: E402
from test_model_gpu import TOL  # noqa: E402

FP8 = torch.float8_e4m3fn
F16_TOL = TOL[torch.float16]


def _ordinal(codes):
    """e4m3 codes -> position on the number line (+0 and -0 both 0), so neighbouring values differ by 1."""
    c = codes.to(torch.int32)
    mag = c & 0x7F
    return torch.where((c & 0x80) != 0, -mag, mag)


def _e4m3_rn(v64):
    """Round-to-nearest-even e4m3 codes of float64 values already inside +-448 (the float64 restatement's codes)."""
    return v64.float().clamp(-448, 448).to(FP8).view(torch.uint8)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("C", [192, 384, 768])
def test_layernorm_e4m3_kernel_matches_float64_spec(C):
    from b200 import capi
    g = torch.Generator().manual_seed(C)
    rows = 2053
    x = torch.randn(rows, C, generator=g) * (1 + 3 * torch.rand(rows, 1, generator=g)) + torch.randn(rows, 1, generator=g)
    x[0] = 1000 + 0.25 * torch.randn(C, generator=g)          # mean 1000, spread 0.25
    x[1] = 0.0                                                 # all equal: x^ = 0, a = 0
    x[2, :] = 0.0
    x[2, 5] = 7.0                                              # one outlier
    x16 = x.half()
    xd = torch.empty(rows, C + 64, dtype=torch.float16, device="cuda")[:, :C]      # row pitch != C
    xd.copy_(x16)
    q, s = capi.layernorm_e4m3(xd, 1e-6)
    torch.cuda.synchronize()
    xf = x16.double()
    mean = xf.mean(1, keepdim=True)
    var = ((xf - mean) ** 2).mean(1, keepdim=True)
    xh = (xf - mean) / torch.sqrt(var + 1e-6)
    a = xh.abs().amax(1, keepdim=True)
    s_ref = torch.where(a > 0, a / 448, torch.ones_like(a))[:, 0]
    inv = torch.where(a > 0, 448 / a, torch.ones_like(a))
    q_ref = _e4m3_rn(xh * inv)
    rel = ((s.cpu().double() - s_ref).abs() / s_ref).max().item()
    assert rel <= 1e-6, rel
    d = (_ordinal(q.cpu()) - _ordinal(q_ref)).abs()
    assert d.max().item() <= 1, d.max().item()
    assert (d != 0).float().mean().item() <= 1e-3, (d != 0).float().mean().item()
    assert torch.equal(q[1].cpu(), torch.zeros(C, dtype=torch.uint8)) and s[1].item() == 1.0


def _random_e4m3(shape, g):
    v = (torch.randn(shape, generator=g) * 64).clamp(-448, 448)
    return v.to(FP8).view(torch.uint8)


GEMM_SHAPES = [(576, 192), (768, 192), (1152, 384), (2304, 768), (3072, 768)]
# set loose for the tensor cores' shortened FP8 accumulation (see lwdetr_b200.h); measured on an H100 80GB HBM3 (700 W):
# at most 2.4e-4 over all 30 cases, about the fp16 rounding of the outputs
GEMM_BAR = 1e-3


@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("N,K", GEMM_SHAPES)
@pytest.mark.parametrize("M", [1, 127, 128 * 132 + 5])
def test_gemm_e4m3_kernel_matches_float64(M, N, K, gelu):
    from b200 import capi
    g = torch.Generator().manual_seed(M * 7 + N + K)
    A, W = _random_e4m3((M, K), g), _random_e4m3((N, K), g)
    sa = (0.5 + torch.rand(M, generator=g)) / 448 / math.sqrt(K)
    sw = (0.5 + torch.rand(N, generator=g)) / 448 * 8
    bias = torch.randn(N, generator=g)
    Ad = torch.zeros(M, K + 16, dtype=torch.uint8, device="cuda")[:, :K]            # row pitch != K
    Ad.copy_(A)
    out = capi.gemm_e4m3(Ad, sa.cuda(), W.cuda(), sw.cuda(), bias.cuda(), capi.ACT_GELU if gelu else capi.ACT_NONE)
    torch.cuda.synchronize()
    Ag, Wg = A.view(FP8).double().cuda(), W.view(FP8).double().cuda()
    ref = sa.double().cuda()[:, None] * sw.double().cuda()[None, :] * (Ag @ Wg.t()) + bias.double().cuda()
    if gelu:
        ref = 0.5 * ref * (1 + torch.erf(ref / math.sqrt(2)))
    rel = ((out.double() - ref).norm() / ref.norm()).item()
    print("gemm_e4m3 M=%d N=%d K=%d gelu=%d rel_l2=%.3e" % (M, N, K, gelu, rel))
    assert rel <= GEMM_BAR, rel


# ------------------------------------------------------------------------------------------------ end to end
def _stats(name, batch, hw=None):
    """Tier statistics of GPU-vs-oracle_fp8, GPU-vs-fp32 oracle and oracle_fp8-vs-fp32 oracle (two-stage indices forced to
    the fp32 oracle's for T1 / T2; T3 free-running; T3 as disagreement = 1 - smallest per-image set agreement)."""
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    cfg = CONFIGS[name]
    H, W = (cfg.img_size, cfg.img_size) if hw is None else hw
    sd = synth_state_dict(cfg, 1)
    x = synth_images(batch, 0, (H, W))
    ri, qi, qf = {}, {}, {}
    ref = oracle_hw.forward(sd, cfg, x, inter=ri)
    qref = oracle_fp8.forward(sd, cfg, x, topk_override=ri["topk"], inter=qi)
    oracle_fp8.forward(sd, cfg, x, inter=qf)
    eng = capi.Engine(cfg, FP8)
    eng.load_state_dict(sd)
    T = batch * (H // 16) * (W // 16)
    for t in cfg.taps:
        eng.capture("block%d" % t, T * cfg.vit_dim)
    forced = eng.forward(x.cuda(), topk_override=ri["topk"])
    torch.cuda.synchronize()
    caps = eng.capture_results()
    eng.clear_captures()
    free = eng.forward(x.cuda())
    torch.cuda.synchronize()
    eng.close()
    got_taps = {t: caps["block%d" % t].reshape(T, cfg.vit_dim) for t in cfg.taps}
    rel = oracle_fp8.rel_l2
    nq = cfg.num_queries

    def disagree(ta, tb):
        return 1.0 - min(len(set(ta[b].tolist()) & set(tb[b].tolist())) / float(nq) for b in range(batch))

    def tier(taps, inter_ref, out, out_ref, topk, topk_ref):
        return {"tap_rel_l2": max(rel(taps[t], inter_ref["block%d" % t].reshape(T, cfg.vit_dim)) for t in cfg.taps),
                "logits_rel_l2": rel(out["pred_logits"], out_ref["pred_logits"]),
                "boxes_maxabs": (out["pred_boxes"] - out_ref["pred_boxes"]).abs().max().item(),
                "set_disagreement": disagree(topk, topk_ref)}

    gf = {"pred_logits": forced["pred_logits"].cpu(), "pred_boxes": forced["pred_boxes"].cpu()}
    gtopk = free["topk_index"].cpu().long()
    q_taps = {t: qi["block%d" % t].reshape(T, cfg.vit_dim) for t in cfg.taps}
    assert torch.isfinite(free["pred_logits"]).all() and torch.isfinite(free["pred_boxes"]).all()
    return (tier(got_taps, qi, gf, qref, gtopk, qf["topk"]),
            tier(got_taps, ri, gf, ref, gtopk, ri["topk"]),
            tier(q_taps, ri, qref, ref, qf["topk"], ri["topk"]), nq)


# the fp16 path's own bar for each statistic (test_model_gpu.TOL; the set disagreement of test_model_gpu's >= 0.95 agreement)
F16_BAR = {"tap_rel_l2": F16_TOL["block"], "logits_rel_l2": F16_TOL["logits_rel"], "boxes_maxabs": F16_TOL["boxes"],
           "set_disagreement": 0.05}


def _check(name, stats, big=False):
    g8, g32, c, nq = stats
    print("fp8 e2e %s: gpu-vs-oracle_fp8 %s | gpu-vs-fp32 %s | oracle_fp8-vs-fp32 %s" % (name, g8, g32, c))
    for k in F16_BAR:
        bar16 = F16_TOL["boxes_big"] if (big and k == "boxes_maxabs") else F16_BAR[k]
        # the CUDA path computes THIS scheme: it sits closer to the e4m3 spec than the spec sits to fp32
        # (the set disagreement moves in steps of one query in nq: one step is allowed on top).  Boxes max-abs also keeps
        # the fp16 path's own bar: measured on an H100, small at 448x768 B = 1 gave 8.65e-4 against 0.5 x 1.69e-3 = 8.47e-4;
        # a single maximum carries the fp16 path's own deviation (its bar against fp32 is 8.5e-4 / 1.5e-3), which is as
        # large as half the scheme's cost there.  Every rel-L2 statistic stayed at or below 0.35x on all configs.
        bar8 = 0.5 * c[k] + (1.0 / nq if k == "set_disagreement" else 0.0)
        if k == "boxes_maxabs":
            bar8 = max(bar8, bar16)
        assert g8[k] <= bar8, (name, k, g8[k], c[k])
        # and against fp32 it costs what the scheme costs plus what the fp16 path costs
        assert g32[k] <= 1.25 * c[k] + bar16, (name, k, g32[k], c[k])


@pytest.mark.parametrize("name,batch", [("tiny", 2), ("small", 2), ("medium", 1), ("large", 1), ("xlarge", 1)])
def test_e2e_against_the_scheme_and_the_fp32_oracle(name, batch):
    _check(name, _stats(name, batch))


@pytest.mark.parametrize("name,hw", [("small", (448, 768)), ("large", (1024, 1024))])
def test_forward_hw_other_sizes(name, hw):
    """forward_hw at a non-square size and at 1024^2 (memory above 16384 tokens: the radix top-k) in the e4m3 mode."""
    _check(name, _stats(name, 1, hw), big=True)


# ------------------------------------------------------------------------------------------------ public paths
def _fp8_engine(name="tiny"):
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    cfg = CONFIGS[name]
    sd = synth_state_dict(cfg, 1)
    eng = capi.Engine(cfg, FP8)
    eng.load_state_dict(sd)
    return cfg, sd, eng


def test_schedule_replaces_only_the_encoder_qkv_fc1_and_counts_one_byte_operands():
    from b200 import capi
    from b200.synth import synth_images
    cfg, sd, eng = _fp8_engine("small")
    eng.forward(synth_images(2, 0).cuda())
    ref = capi.Engine(cfg, torch.float16)
    ref.set_option("fuse_layernorm", 0)
    ref.load_state_dict(sd)
    ref.forward(synth_images(2, 0).cuda())
    ops8, ops16 = eng.ops(), ref.ops()
    assert [o[0] for o in ops8] == [o[0] for o in ops16]            # same labels, same order
    for (l8, f8, b8), (l16, f16, b16) in zip(ops8, ops16):
        assert f8 == f16, l8
        if l8.endswith(".qkv") or l8.endswith(".fc1"):
            assert b8 < b16, l8                                       # 1-byte A and W
        elif l8.endswith(".ln1") or l8.endswith(".ln2"):
            pass
        else:
            assert b8 == b16, l8
    eng.close()
    ref.close()


def test_cuda_graph_replay_is_bit_identical_to_eager():
    from b200.synth import synth_images
    cfg, sd, eng = _fp8_engine()
    xs = [synth_images(2, s).cuda() for s in (0, 1)]
    eager = [{k: v.clone() for k, v in eng.forward(x).items() if k.startswith("pred")} for x in xs]
    eng.set_option("cuda_graph", 1)
    for _ in range(3):
        for x, ref in zip(xs, eager):
            out = eng.forward(x)
            torch.cuda.synchronize()
            assert torch.equal(out["pred_logits"], ref["pred_logits"]) and torch.equal(out["pred_boxes"], ref["pred_boxes"])
    eng.close()


def test_forward_frames_identity_and_keep_aspect():
    from b200.config import CONFIGS
    from b200.synth import synth_images
    cfg, sd, eng = _fp8_engine()
    g = torch.Generator().manual_seed(3)
    u8 = torch.randint(0, 256, (2, 640, 640, 3), generator=g, dtype=torch.uint8).cuda()
    a = eng.forward(u8)
    b = eng.forward_frames([u8[0], u8[1]])                             # already at the run size: the uint8 path exactly
    torch.cuda.synchronize()
    assert torch.equal(a["pred_logits"], b["pred_logits"]) and torch.equal(a["pred_boxes"], b["pred_boxes"])
    frames = [torch.randint(0, 256, (480, 640, 3), generator=g, dtype=torch.uint8).cuda(),
              torch.randint(0, 256, (720, 400, 3), generator=g, dtype=torch.uint8).cuda()]
    fit = dict(fit="keep_aspect", short_side=512, max_side=640)
    k8 = eng.forward_frames(frames, **fit)
    from b200 import capi
    e16 = capi.Engine(cfg, torch.float16)
    e16.load_state_dict(sd)
    k16 = e16.forward_frames(frames, **fit)
    f8 = eng.forward_frames(frames, topk_override=k16["topk_index"], **fit)
    torch.cuda.synchronize()
    assert k8["frame_sizes"] == k16["frame_sizes"]
    assert torch.isfinite(k8["pred_logits"]).all() and torch.isfinite(k8["pred_boxes"]).all()
    # with the same two-stage selection the e4m3 mode differs from fp16 by about what the scheme costs (CPU-measured on
    # tiny: logits rel-L2 4.6e-3), not more
    rel = oracle_fp8.rel_l2(f8["pred_logits"].float().cpu(), k16["pred_logits"].float().cpu())
    print("keep-aspect fp8 vs fp16 logits rel-L2 %.3e" % rel)
    assert rel <= 2e-2, rel
    eng.close()
    e16.close()


def test_module_and_detect_in_the_e4m3_mode(monkeypatch):
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    sd = synth_state_dict(cfg, 1)
    model = LWDETR(cfg, compute_dtype=FP8).eval()
    model.load_state_dict(sd, strict=True)
    model.cuda()
    x = synth_images(2, 0).cuda()
    out = model(x)
    assert model.engine().dtype == FP8
    assert out["pred_logits"].shape == (2, cfg.num_queries, cfg.num_classes) and out["pred_logits"].dtype == torch.float32
    direct = model.engine().forward(x)
    assert torch.equal(out["pred_logits"], direct["pred_logits"])
    frames = [torch.randint(0, 256, (360, 500, 3), dtype=torch.uint8).cuda(), torch.randint(0, 256, (640, 480, 3), dtype=torch.uint8).cuda()]
    dets = model.detect(frames, fit="keep_aspect", short_side=512, max_side=640, num_select=50)
    assert len(dets) == 2 and all(d["boxes"].shape == (50, 4) for d in dets)
    # LWDETR_B200_DTYPE=fp8 selects the mode when no compute dtype is given
    monkeypatch.setenv("LWDETR_B200_DTYPE", "fp8")
    m2 = LWDETR(cfg).eval()
    m2.load_state_dict(sd, strict=True)
    m2.cuda()
    out2 = m2(x)
    assert m2.engine().dtype == FP8 and torch.equal(out2["pred_logits"], out["pred_logits"])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_broadcast_weights_in_the_e4m3_mode():
    import torch.multiprocessing as mp
    mp.spawn(_bcast_worker, nprocs=2, join=True)


def _bcast_worker(rank):
    import tempfile
    import torch.distributed as dist
    from b200 import capi
    from b200.config import CONFIGS
    from b200.dist import broadcast_engine_weights
    from b200.synth import synth_images, synth_state_dict
    torch.cuda.set_device(rank)
    store = os.path.join(tempfile.gettempdir(), "lwdetr_fp8_bcast_%d" % os.getppid())
    dist.init_process_group("nccl", init_method="file://" + store, rank=rank, world_size=2)
    cfg = CONFIGS["small"]
    eng = capi.Engine(cfg, FP8)
    eng.load_state_dict(synth_state_dict(cfg, 1 if rank == 0 else 2))
    broadcast_engine_weights(eng, torch.device("cuda", rank), src=0)
    o = eng.forward(synth_images(1, 4).cuda(), want_aux=False)
    res = torch.cat([o["pred_logits"].flatten(), o["pred_boxes"].flatten()])
    allr = [torch.empty_like(res) for _ in range(2)]
    dist.all_gather(allr, res)
    assert torch.equal(allr[0], allr[1])
    eng.close()
    dist.destroy_process_group()
