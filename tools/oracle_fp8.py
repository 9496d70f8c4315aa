"""The CPU oracle with the e4m3 encoder mode's quantisation  --  TEST INFRASTRUCTURE ONLY.

The forward of oracle/lwdetr_oracle.py (composed as tools/oracle_hw.py composes it, so it takes any input size), except that
in every ViT block the two LayerNorm -> linear pairs in front of the tensor cores' e4m3 GEMMs, LN1 -> qkv and LN2 -> fc1,
follow the LWDETR_F16_E4M3 contract (include/lwdetr_b200.h):
  activations, per token m: x^ = (x - mean) * rstd (no affine), a_m = max|x^_m|, s_a = a_m / 448, q_a = e4m3(x^ * 448 / a_m)
  weights, per output channel n: W' = W diag(ln_w), s_w = max|W'_n| / 448, q_w = e4m3(W'_n * 448 / max|W'_n|),
  beta' = beta + W ln_b (double)
  y = s_a s_w (q_a . q_w) + beta'   (qkv: y; fc1: gelu(y))
e4m3 rounding is torch.float8_e4m3fn's (round to nearest even) after a clamp to +-448: torch turns values above the
largest finite e4m3 into NaN where the hardware saturates.  Everything else is the fp32 oracle.  quantize=False gives the
unquantised composition, i.e. oracle.forward (a self-check of the composition).
"""
import torch
import torch.nn.functional as F

from oracle import lwdetr_oracle as orc

import oracle_hw

E4M3_MAX = 448.0


def quant_rows(x):
    """Per-row e4m3 quantisation of fp32 x [..., K]: (codes as fp32 values, scale [..., 1]), scale = max|x| / 448 (0 -> 1).
    The same arithmetic as lwdetr_host_quant_e4m3_rows and the device LayerNorm -> e4m3 kernel: inv = 448 / max in fp32,
    x * inv in fp32, round to nearest even, saturate."""
    x = x.float()
    a = x.abs().amax(-1, keepdim=True)
    nz = a > 0
    inv = torch.where(nz, torch.tensor(E4M3_MAX, dtype=torch.float32) / torch.where(nz, a, torch.ones_like(a)), torch.ones_like(a))
    scale = torch.where(nz, a / E4M3_MAX, torch.ones_like(a))
    q = (x * inv).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, scale


def fold_weights(W, bias, ln_w, ln_b):
    """(e4m3 codes [N, C] as float8_e4m3fn, s_w [N], beta' [N]) of a linear behind a LayerNorm."""
    Wf = W.float() * ln_w.float()[None, :]
    qw, sw = quant_rows(Wf)
    beta = (bias.double() + W.double() @ ln_b.double()).float()
    return qw, sw[:, 0], beta


def ln_linear(x, ln_w, ln_b, W, bias, quantize=True):
    """linear(LayerNorm(x; ln_w, ln_b, eps 1e-6); W, bias), in the e4m3 mode's arithmetic when quantize."""
    C = x.shape[-1]
    if not quantize:
        return F.linear(F.layer_norm(x, (C,), ln_w, ln_b, 1e-6), W, bias)
    xh = F.layer_norm(x.float(), (C,), None, None, 1e-6)
    qa, sa = quant_rows(xh)
    qw, sw, beta = fold_weights(W, bias, ln_w, ln_b)
    acc = qa.float() @ qw.float().t()                              # products of e4m3 values are exact in fp32
    return sa * sw * acc + beta


def vit_block(x, sd, p, heads, window, quantize=True):
    """oracle.vit_block with LN1 -> qkv and LN2 -> fc1 through ln_linear."""
    Bw, N, C = x.shape
    dh = C // heads
    a = p + ".attn"
    bias = torch.cat([sd[a + ".q_bias"], torch.zeros_like(sd[a + ".v_bias"]), sd[a + ".v_bias"]])
    qkv = ln_linear(x, sd[p + ".norm1.weight"], sd[p + ".norm1.bias"], sd[a + ".qkv.weight"], bias, quantize)
    if not window:
        qkv = qkv.reshape(Bw // 16, 16 * N, 3 * C)
    Bn, L = qkv.shape[0], qkv.shape[1]
    qkv = qkv.reshape(Bn, L, 3, heads, dh).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    att = ((q * dh ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    h = F.linear((att @ v).transpose(1, 2).reshape(Bn, L, C), sd[a + ".proj.weight"], sd[a + ".proj.bias"])
    if not window:
        h = h.reshape(Bw, N, C)
    x = x + sd[p + ".gamma_1"] * h
    h = F.gelu(ln_linear(x, sd[p + ".norm2.weight"], sd[p + ".norm2.bias"], sd[p + ".mlp.fc1.weight"], sd[p + ".mlp.fc1.bias"], quantize))
    h = F.linear(h, sd[p + ".mlp.fc2.weight"], sd[p + ".mlp.fc2.bias"])
    return x + sd[p + ".gamma_2"] * h


def vit_encoder(images, sd, cfg, inter=None, quantize=True):
    """oracle_hw.vit_encoder_hw with the e4m3 blocks."""
    e = "backbone.0.encoder"
    x = F.conv2d(images, sd[e + ".patch_embed.proj.weight"], sd[e + ".patch_embed.proj.bias"], stride=cfg.patch)
    x = x.permute(0, 2, 3, 1)
    B, H, W, C = x.shape
    x = x + oracle_hw.abs_pos_embed_hw(sd[e + ".pos_embed"], H, W)
    x = orc.to_window_major(x)
    if inter is not None:
        inter["patch"] = x
    taps = []
    for i in range(cfg.vit_depth):
        x = vit_block(x, sd, "%s.blocks.%d" % (e, i), cfg.vit_heads, i in cfg.window_blocks, quantize)
        if inter is not None:
            inter["block%d" % i] = x
        if i in cfg.taps:
            taps.append(orc.from_window_major(x, B, H, W))
    return taps


def forward(sd, cfg, images, topk_override=None, inter=None, mask=None, quantize=True):
    """The e4m3 mode's forward on the CPU (fp32 outside the quantised GEMMs) at the size of `images` [B,3,H,W]; the
    arguments and outputs of oracle_hw.forward."""
    H, W = int(images.shape[-2]), int(images.shape[-1])
    if not (H == W == cfg.img_size):
        cfg = oracle_hw.AtInputSize(cfg, H, W)
    with torch.no_grad():
        sd = {k: (v.float() if v.is_floating_point() else v) for k, v in sd.items()}
        taps = vit_encoder(images.float(), sd, cfg, inter, quantize)
        levels = orc.projector(taps, sd, cfg)
        if inter is not None:
            for j, tp in enumerate(taps):
                inter["tap%d" % j] = tp
            for l, lv in enumerate(levels):
                inter["level%d" % l] = lv
        lm = orc.level_padding_masks(mask, cfg) if mask is not None and bool(mask.any()) else None
        return orc.transformer_and_heads(levels, sd, cfg, topk_override, inter, lm)


def rel_l2(a, b):
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def quant_cost(name, batch=2, wseed=1, iseed=0, hw=None):
    """What the e4m3 scheme costs against the fp32 oracle on the synthetic weights / images of a config: T1 worst tap
    rel-L2, T2 logits rel-L2 and boxes max-abs with the two-stage indices forced to the fp32 oracle's, T3 the smallest
    per-image agreement of the free-running selected sets."""
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    cfg = CONFIGS[name]
    sd = synth_state_dict(cfg, wseed)
    H, W = (cfg.img_size, cfg.img_size) if hw is None else hw
    x = synth_images(batch, iseed, (H, W))
    ri, qi = {}, {}
    ref = oracle_hw.forward(sd, cfg, x, inter=ri)
    forced = forward(sd, cfg, x, topk_override=ri["topk"], inter=qi)
    free_inter = {}
    forward(sd, cfg, x, inter=free_inter)
    nq = cfg.num_queries
    agree = min(len(set(free_inter["topk"][b].tolist()) & set(ri["topk"][b].tolist())) / float(nq) for b in range(batch))
    return {"tap_rel_l2": max(rel_l2(qi["tap%d" % j], ri["tap%d" % j]) for j in range(len(cfg.taps))),
            "logits_rel_l2": rel_l2(forced["pred_logits"], ref["pred_logits"]),
            "boxes_maxabs": (forced["pred_boxes"] - ref["pred_boxes"]).abs().max().item(),
            "set_agreement_min": agree}
