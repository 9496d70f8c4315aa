"""CPU oracle for the LW-DETR inference forward pass  --  TEST INFRASTRUCTURE ONLY.

A from-scratch fp32/fp64 torch-CPU restatement of the reference forward (eval mode, released flags
--two_stage --bbox_reparam --lite_refpoint_refine), written as plain functions over a state_dict.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this file; the product path (lw-detr_b200/) never does and has no CPU fallback.

Pinning: tests/test_oracle.py checks this oracle against golden vectors produced by the UNMODIFIED
reference (tools/make_goldens.py -> tests/golden/*.npz) for all five released configurations.  The
reference itself ships no golden vectors for this path (SURVEY.md 8c), so the goldens are outputs of
the reference code run on torch 2.11 CPU.

Every function cites the reference lines it restates (paths relative to Atten4Vis/LW-DETR).
"""
import math

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------- ViT encoder
def abs_pos_embed(pos_embed, grid):
    """vit.py:26-54 get_abs_pos: drop the cls slot, bicubic (align_corners=False) 14x14 -> grid x grid."""
    tok = pos_embed[:, 1:]
    n = int(math.isqrt(tok.shape[1]))
    img = tok.reshape(1, n, n, -1).permute(0, 3, 1, 2)
    if n != grid:
        img = F.interpolate(img, size=(grid, grid), mode="bicubic", align_corners=False)
    return img.permute(0, 2, 3, 1)                                   # [1, grid, grid, C]


def to_window_major(x):
    """vit.py:353-358: [B, H, W, C] -> [B*16, (H/4)*(W/4), C], windows enumerated (wy, wx)."""
    B, H, W, C = x.shape
    return x.reshape(B, 4, H // 4, 4, W // 4, C).permute(0, 1, 3, 2, 4, 5).reshape(B * 16, (H // 4) * (W // 4), C)


def from_window_major(x, B, H, W):
    """vit.py:362-364 (inverse reorg), returned as NHWC [B, H, W, C]."""
    C = x.shape[-1]
    return x.reshape(B, 4, 4, H // 4, W // 4, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)


def vit_attention(x, sd, p, heads):
    """vit.py:120-140 Attention.forward (use_cae): bias = [q_bias, 0, v_bias]; q scaled before QK^T."""
    Bn, N, C = x.shape
    dh = C // heads
    bias = torch.cat([sd[p + ".q_bias"], torch.zeros_like(sd[p + ".v_bias"]), sd[p + ".v_bias"]])
    qkv = F.linear(x, sd[p + ".qkv.weight"], bias).reshape(Bn, N, 3, heads, dh).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    att = ((q * dh ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    y = (att @ v).transpose(1, 2).reshape(Bn, N, C)
    return F.linear(y, sd[p + ".proj.weight"], sd[p + ".proj.bias"])


def vit_block(x, sd, p, heads, window):
    """vit.py:195-222 Block.forward (use_cae: layer-scale gamma_1/gamma_2; LN eps 1e-6 backbone.py:69)."""
    Bw, N, C = x.shape
    h = F.layer_norm(x, (C,), sd[p + ".norm1.weight"], sd[p + ".norm1.bias"], 1e-6)
    if not window:
        h = h.reshape(Bw // 16, 16 * N, C)
    h = vit_attention(h, sd, p + ".attn", heads)
    if not window:
        h = h.reshape(Bw, N, C)
    x = x + sd[p + ".gamma_1"] * h
    h = F.layer_norm(x, (C,), sd[p + ".norm2.weight"], sd[p + ".norm2.bias"], 1e-6)
    h = F.linear(h, sd[p + ".mlp.fc1.weight"], sd[p + ".mlp.fc1.bias"])
    h = F.gelu(h)                                                    # timm Mlp: exact (erf) GELU
    h = F.linear(h, sd[p + ".mlp.fc2.weight"], sd[p + ".mlp.fc2.bias"])
    return x + sd[p + ".gamma_2"] * h


def vit_encoder(images, sd, cfg, inter=None):
    """vit.py:343-365 ViT.forward.  Returns the tapped feature maps as NHWC [B, 40, 40, C]."""
    e = "backbone.0.encoder"
    x = F.conv2d(images, sd[e + ".patch_embed.proj.weight"], sd[e + ".patch_embed.proj.bias"], stride=cfg.patch)
    x = x.permute(0, 2, 3, 1)
    B, H, W, C = x.shape
    x = x + abs_pos_embed(sd[e + ".pos_embed"], H)
    x = to_window_major(x)
    if inter is not None:
        inter["patch"] = x
    taps = []
    for i in range(cfg.vit_depth):
        x = vit_block(x, sd, "%s.blocks.%d" % (e, i), cfg.vit_heads, i in cfg.window_blocks)
        if inter is not None:
            inter["block%d" % i] = x
        if i in cfg.taps:
            taps.append(from_window_major(x, B, H, W))
    return taps


# ----------------------------------------------------------------------------------------- projector
def _convx(x, sd, p, stride=1, act="silu"):
    """projector.py:85-98 ConvX: conv (no bias) -> BatchNorm (eval, eps 1e-5) -> activation.  x is NCHW."""
    w = sd[p + ".conv.weight"]
    y = F.conv2d(x, w, None, stride=stride, padding=w.shape[-1] // 2)
    y = F.batch_norm(y, sd[p + ".bn.running_mean"], sd[p + ".bn.running_var"], sd[p + ".bn.weight"],
                     sd[p + ".bn.bias"], False, 0.0, 1e-5)
    return F.silu(y) if act == "silu" else F.relu(y)


def _c2f(x, sd, p):
    """projector.py:117-132 C2f with n=3 Bottlenecks (shortcut=False, e=1.0), SiLU everywhere."""
    y = _convx(x, sd, p + ".cv1")
    c = y.shape[1] // 2
    parts = [y[:, :c], y[:, c:]]
    for j in range(3):
        t = _convx(parts[-1], sd, "%s.m.%d.cv1" % (p, j))
        parts.append(_convx(t, sd, "%s.m.%d.cv2" % (p, j)))
    return _convx(torch.cat(parts, 1), sd, p + ".cv2")


def projector(taps_nhwc, sd, cfg):
    """projector.py:214-241 MultiScaleProjector.forward.  Returns per level [B, h*w, d] (token-major)."""
    pr = "backbone.0.projector"
    C = cfg.vit_dim
    feats = [t.permute(0, 3, 1, 2) for t in taps_nhwc]
    out = []
    for lvl, scale in enumerate(cfg.projector_scale):
        fuse = []
        for t, f in enumerate(feats):
            s = "%s.stages_sampling.%d.%d" % (pr, lvl, t)
            if scale == "P3":                                       # projector.py:176-187
                if C > 512:
                    f = _convx(f, sd, s + ".0", act="relu")
                    f = F.conv_transpose2d(f, sd[s + ".1.weight"], sd[s + ".1.bias"], stride=2)
                else:
                    f = F.conv_transpose2d(f, sd[s + ".0.weight"], sd[s + ".0.bias"], stride=2)
            elif scale == "P5":                                     # projector.py:190-193
                f = _convx(f, sd, s + ".0", stride=2, act="relu")
            fuse.append(f)
        y = _c2f(torch.cat(fuse, 1), sd, "%s.stages.%d.0" % (pr, lvl))
        # projector.py:21-47 channel-first LayerNorm, eps 1e-6, biased variance
        u = y.mean(1, keepdim=True)
        s2 = (y - u).pow(2).mean(1, keepdim=True)
        y = (y - u) / torch.sqrt(s2 + 1e-6)
        y = sd["%s.stages.%d.1.weight" % (pr, lvl)][:, None, None] * y + sd["%s.stages.%d.1.bias" % (pr, lvl)][:, None, None]
        out.append(y.flatten(2).transpose(1, 2))                    # transformer.py:208 flatten
    return out


# ------------------------------------------------------------------------------- two-stage + decoder
def _mlp(x, sd, p, n):
    """transformer.py:27-39 / lwdetr.py:547-559 MLP: ReLU between layers."""
    for i in range(n):
        x = F.linear(x, sd["%s.layers.%d.weight" % (p, i)], sd["%s.layers.%d.bias" % (p, i)])
        if i < n - 1:
            x = F.relu(x)
    return x


def encoder_proposals(cfg, dtype, level_masks=None):
    """transformer.py:71-125 gen_encoder_output_proposals with unsigmoid=False:
    per token (cx, cy, w, h) = ((j+.5)/valid_W, (i+.5)/valid_H, .05*2^lvl, .05*2^lvl); padded or out-of-(0.01,0.99)
    -> zeros.  Without masks (same-size batch) valid_W/H are the level sizes and the table is batch independent
    ([S,4], [S,1]); with per-level padding masks [B,H,W] (True = padding) it is per image ([B,S,4], [B,S,1])."""
    props = []
    for lvl, (H, W) in enumerate(cfg.level_shapes):
        ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
        if level_masks is None:
            cx, cy = (xs + 0.5) / W, (ys + 0.5) / H
        else:
            m = level_masks[lvl]
            vh = (~m[:, :, 0]).sum(1).float()[:, None, None]          # transformer.py:87-89
            vw = (~m[:, 0, :]).sum(1).float()[:, None, None]
            cx, cy = (xs[None] + 0.5) / vw, (ys[None] + 0.5) / vh
        wh = torch.full_like(cx, 0.05 * (2.0 ** lvl))
        props.append(torch.stack([cx, cy, wh, wh], -1).flatten(-3, -2))
    props = torch.cat(props, -2)
    valid = ((props > 0.01) & (props < 0.99)).all(-1, keepdim=True)
    if level_masks is not None:
        pad = torch.cat([m.flatten(1) for m in level_masks], 1)[..., None]
        props = props.masked_fill(pad, 0.0)                             # transformer.py:117-118
        keep = valid & ~pad                                             # memory rows zeroed: transformer.py:121-124
        return (props * valid).to(dtype), keep
    return (props * valid).to(dtype), valid


def reparam(delta, ref):
    """transformer.py:234-240 / lwdetr.py:149-155: cxcy = d_xy*ref_wh + ref_xy ; wh = exp(d_wh)*ref_wh."""
    return torch.cat([delta[..., :2] * ref[..., 2:] + ref[..., :2], delta[..., 2:].exp() * ref[..., 2:]], -1)


def sine_embed(pos, dim):
    """transformer.py:42-68 gen_sineembed_for_position for 4-d boxes; output order (y, x, w, h)."""
    scale = 2 * math.pi
    i = torch.arange(dim, dtype=torch.float32)
    dim_t = (10000 ** (2 * (i // 2) / dim)).to(pos.dtype)

    def one(c):
        v = (pos[..., c] * scale)[..., None] / dim_t
        return torch.stack((v[..., 0::2].sin(), v[..., 1::2].cos()), dim=-1).flatten(-2)

    return torch.cat((one(1), one(0), one(2), one(3)), dim=-1)


def msda_core(value, level_shapes, loc, weight):
    """Multi-scale deformable attention core (ops/src/cuda/ms_deform_im2col_cuda.cuh:33-84, 237-299;
    same function as ops/functions/ms_deform_attn_func.py:52-75).
      value [B, S, M, D]; loc [B, Q, M, L, P, 2] normalised (x, y); weight [B, Q, M, L, P]
      out[b,q,m,:] = sum_{l,p} weight * bilinear(value_l[b,:,m,:], (x*W - .5, y*H - .5)), zero outside."""
    B, S, M, D = value.shape
    Q, P = loc.shape[1], loc.shape[4]
    out = torch.zeros(B, Q, M, D, dtype=value.dtype, device=value.device)
    start = 0
    for l, (H, W) in enumerate(level_shapes):
        v = value[:, start:start + H * W].permute(0, 2, 1, 3)                  # [B, M, HW, D]
        start += H * W
        x = loc[:, :, :, l, :, 0] * W - 0.5                                    # [B, Q, M, P]
        y = loc[:, :, :, l, :, 1] * H - 0.5
        x0, y0 = torch.floor(x), torch.floor(y)
        lx, ly = x - x0, y - y0
        for dy in (0, 1):
            for dx in (0, 1):
                xi, yi = x0 + dx, y0 + dy
                ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
                cw = (lx if dx else 1 - lx) * (ly if dy else 1 - ly) * ok * weight[:, :, :, l, :]
                idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()     # [B, Q, M, P]
                idx = idx.permute(0, 2, 1, 3).reshape(B, M, Q * P, 1).expand(-1, -1, -1, D)
                g = torch.gather(v, 2, idx).reshape(B, M, Q, P, D).permute(0, 2, 1, 3, 4)
                out = out + (cw[..., None] * g).sum(3)
    return out.reshape(B, Q, M * D)


def decoder_self_attention(tgt, query_pos, sd, p, heads):
    """attention.py:137-212,215-451,507-606 with q = k = tgt + query_pos, v = tgt (transformer.py:484-492)."""
    B, Q, d = tgt.shape
    dh = d // heads
    w, b = sd[p + ".in_proj_weight"], sd[p + ".in_proj_bias"]
    qk_in = tgt + query_pos
    q = F.linear(qk_in, w[:d], b[:d])
    k = F.linear(qk_in, w[d:2 * d], b[d:2 * d])
    v = F.linear(tgt, w[2 * d:], b[2 * d:])
    split = lambda t: t.reshape(B, Q, heads, dh).transpose(1, 2)
    att = ((split(q) / math.sqrt(dh)) @ split(k).transpose(-2, -1)).softmax(dim=-1)
    y = (att @ split(v)).transpose(1, 2).reshape(B, Q, d)
    return F.linear(y, sd[p + ".out_proj.weight"], sd[p + ".out_proj.bias"])


def deformable_cross_attention(query, ref, memory, sd, p, cfg, pad=None):
    """ops/modules/ms_deform_attn.py:96-144 with 4-d reference boxes.  ref is [B,Q,4] (same box at every level:
    valid_ratio 1) or [B,Q,L,4] (boxes scaled by each level's valid ratio, transformer.py:352-353); pad [B,S] marks
    padded memory tokens whose value rows are zeroed (ms_deform_attn.py:114-115)."""
    B, Q, d = query.shape
    M, L, P = cfg.ca_nheads, cfg.n_levels, cfg.dec_n_points
    value = F.linear(memory, sd[p + ".value_proj.weight"], sd[p + ".value_proj.bias"])
    if pad is not None:
        value = value.masked_fill(pad[..., None], 0.0)
    value = value.reshape(B, -1, M, d // M)
    off = F.linear(query, sd[p + ".sampling_offsets.weight"], sd[p + ".sampling_offsets.bias"]).reshape(B, Q, M, L, P, 2)
    aw = F.linear(query, sd[p + ".attention_weights.weight"], sd[p + ".attention_weights.bias"]).reshape(B, Q, M, L * P)
    aw = aw.softmax(-1).reshape(B, Q, M, L, P)
    if ref.dim() == 3:
        ref = ref[:, :, None, :].expand(-1, -1, L, -1)
    loc = ref[:, :, None, :, None, :2] + off / P * ref[:, :, None, :, None, 2:] * 0.5
    y = msda_core(value, cfg.level_shapes, loc, aw)
    return F.linear(y, sd[p + ".output_proj.weight"], sd[p + ".output_proj.bias"])


def decoder_layer(tgt, query_pos, ref, memory, sd, p, cfg, pad=None):
    """transformer.py:466-517 forward_post (dropout 0, LN eps 1e-5)."""
    d = tgt.shape[-1]
    ln = lambda t, n: F.layer_norm(t, (d,), sd["%s.%s.weight" % (p, n)], sd["%s.%s.bias" % (p, n)], 1e-5)
    tgt = ln(tgt + decoder_self_attention(tgt, query_pos, sd, p + ".self_attn", cfg.sa_nheads), "norm1")
    tgt = ln(tgt + deformable_cross_attention(tgt + query_pos, ref, memory, sd, p + ".cross_attn", cfg, pad), "norm2")
    ff = F.linear(F.relu(F.linear(tgt, sd[p + ".linear1.weight"], sd[p + ".linear1.bias"])),
                  sd[p + ".linear2.weight"], sd[p + ".linear2.bias"])
    return ln(tgt + ff, "norm3")


def transformer_and_heads(levels, sd, cfg, topk_override=None, inter=None, level_masks=None):
    """transformer.py:198-288 Transformer.forward (eval: group 0 only), transformer.py:328-427 decoder
    (lite_refpoint_refine: query_pos from the initial reference once), lwdetr.py:141-173 heads.
    level_masks: per-level padding masks [B,H,W] (True = padding) of a padded / mixed-size batch, or None."""
    memory = torch.cat(levels, 1)                                    # [B, S, d]
    B, S, d = memory.shape
    nq = cfg.num_queries
    proposals, valid = encoder_proposals(cfg, memory.dtype, level_masks)
    pad = vr = None
    if level_masks is not None:
        pad = torch.cat([m.flatten(1) for m in level_masks], 1)                                   # transformer.py:215-217
        vr = torch.stack([torch.stack([(~m[:, 0, :]).sum(1).float() / m.shape[2],                 # transformer.py:188-196 (w, h)
                                       (~m[:, :, 0]).sum(1).float() / m.shape[1]], -1) for m in level_masks], 1).to(memory.dtype)
    t = "transformer"
    om = F.linear(memory * valid, sd[t + ".enc_output.0.weight"], sd[t + ".enc_output.0.bias"])
    om = F.layer_norm(om, (d,), sd[t + ".enc_output_norm.0.weight"], sd[t + ".enc_output_norm.0.bias"], 1e-5)
    cls_all = F.linear(om, sd[t + ".enc_out_class_embed.0.weight"], sd[t + ".enc_out_class_embed.0.bias"])
    score = cls_all.max(-1)[0]
    topk = torch.topk(score, nq, dim=1)[1] if topk_override is None else topk_override
    sel = torch.gather(om, 1, topk[..., None].expand(-1, -1, d))     # memory_ts / hs_enc
    prop_sel = proposals[topk] if proposals.dim() == 2 else torch.gather(proposals, 1, topk[..., None].expand(-1, -1, 4))
    box_ts = reparam(_mlp(sel, sd, t + ".enc_out_bbox_embed.0", 3), prop_sel)          # per-row op: same as MLP-then-gather
    refpoint = reparam(sd["refpoint_embed.weight"][:nq][None].expand(B, -1, -1), box_ts)   # transformer.py:266-276
    tgt = sd["query_feat.weight"][:nq][None].expand(B, -1, -1)
    # transformer.py:345-356: reference boxes are scaled by each level's valid ratio; the sine embedding uses level 0's
    ref_in = refpoint if vr is None else refpoint[:, :, None, :] * torch.cat([vr, vr], -1)[:, None]
    query_pos = _mlp(sine_embed(refpoint if vr is None else ref_in[:, :, 0, :], d // 2), sd, t + ".decoder.ref_point_head", 2)
    if inter is not None:
        inter.update(memory=memory, enc_score=score, topk=topk, enc_sel=sel, box_ts=box_ts, refpoint=refpoint,
                     query_pos=query_pos)
    hs = []
    for i in range(cfg.dec_layers):
        tgt = decoder_layer(tgt, query_pos, ref_in, memory, sd, "%s.decoder.layers.%d" % (t, i), cfg, pad)
        hs.append(F.layer_norm(tgt, (d,), sd[t + ".decoder.norm.weight"], sd[t + ".decoder.norm.bias"], 1e-5))
        if inter is not None:
            inter["dec%d" % i] = tgt
    hs = torch.stack(hs)                                              # [layers, B, nq, d]
    boxes = reparam(_mlp(hs, sd, "bbox_embed", 3), refpoint[None])
    logits = F.linear(hs, sd["class_embed.weight"], sd["class_embed.bias"])
    out = {"pred_logits": logits[-1], "pred_boxes": boxes[-1],
           "aux_outputs": [{"pred_logits": a, "pred_boxes": b} for a, b in zip(logits[:-1], boxes[:-1])],
           "enc_outputs": {"pred_logits": torch.gather(cls_all, 1, topk[..., None].expand(-1, -1, cls_all.shape[-1])),
                           "pred_boxes": box_ts}}
    return out


def level_padding_masks(mask, cfg):
    """backbone.py:150-158: the image padding mask [B,H,W] (True = padding) resized to every feature level with
    F.interpolate's default nearest mode."""
    return [F.interpolate(mask[None].float(), size=(H, W)).to(torch.bool)[0] for (H, W) in cfg.level_shapes]


def forward(sd, cfg, images, topk_override=None, inter=None, dtype=torch.float32, mask=None):
    """Full LWDETR.forward (lwdetr.py:111-174).  mask: NestedTensor.mask [B,H,W] of a padded / mixed-size batch
    (True = padding, misc.py:317-339) or None for same-size batches."""
    with torch.no_grad():
        sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
        taps = vit_encoder(images.to(dtype), sd, cfg, inter)
        levels = projector(taps, sd, cfg)
        if inter is not None:
            for j, tp in enumerate(taps):
                inter["tap%d" % j] = tp
            for l, lv in enumerate(levels):
                inter["level%d" % l] = lv
        lm = level_padding_masks(mask, cfg) if mask is not None and bool(mask.any()) else None
        return transformer_and_heads(levels, sd, cfg, topk_override, inter, lm)


def postprocess(out, target_sizes, num_select):
    """lwdetr.py:515-544 PostProcess.forward."""
    logits, boxes = out["pred_logits"], out["pred_boxes"]
    prob = logits.sigmoid()
    vals, idx = torch.topk(prob.reshape(logits.shape[0], -1), num_select, dim=1)
    qi, labels = idx // logits.shape[2], idx % logits.shape[2]
    cx, cy, w, h = boxes.unbind(-1)
    xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)
    xyxy = torch.gather(xyxy, 1, qi[..., None].expand(-1, -1, 4))
    ih, iw = target_sizes.unbind(1)
    xyxy = xyxy * torch.stack([iw, ih, iw, ih], 1)[:, None, :]
    return [{"scores": s, "labels": l, "boxes": b} for s, l, b in zip(vals, labels, xyxy)]
