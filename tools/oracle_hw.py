"""The CPU oracle (oracle/lwdetr_oracle.py) at any input size  --  TEST INFRASTRUCTURE ONLY.

oracle/lwdetr_oracle.py restates the reference forward at the configured square size: its ViT resizes the position
embedding to a square grid and its level shapes come from cfg.img_size.  The reference itself takes both from the
image (vit.py:26-54 get_abs_pos with hw = (H/16, W/16), vit.py:343-358 windows of (H/64) x (W/64) tokens; the projector
and transformer take their level shapes from the feature maps).  This module composes the oracle's own functions with
exactly that: a ViT whose position table is resized to (H/16, W/16), and a config view whose level_shapes are those of
the image.  At the configured size it IS oracle.forward.  tests/test_resolution_cpu.py pins it to goldens of the
unmodified reference at 512x512, 448x768, 1024x1024, 768x1344 and a padded 832x1344 batch.
"""
import math

import torch
import torch.nn.functional as F

from oracle import lwdetr_oracle as orc


class AtInputSize:
    """The config seen through one input size: level_shapes / memory_len of an H x W image (projector.py:165-193
    scales of the (H/16, W/16) grid); every other field is the config's."""

    def __init__(self, cfg, height, width):
        self._cfg = cfg
        self.level_shapes = cfg.level_shapes_at(height, width)
        self.memory_len = sum(h * w for h, w in self.level_shapes)

    def __getattr__(self, name):
        return getattr(self._cfg, name)


def abs_pos_embed_hw(pos_embed, gh, gw):
    """vit.py:26-54 get_abs_pos with hw = (gh, gw): drop the cls slot, bicubic (align_corners=False) 14x14 -> gh x gw."""
    tok = pos_embed[:, 1:]
    n = int(math.isqrt(tok.shape[1]))
    img = tok.reshape(1, n, n, -1).permute(0, 3, 1, 2)
    if n != gh or n != gw:
        img = F.interpolate(img, size=(gh, gw), mode="bicubic", align_corners=False)
    return img.permute(0, 2, 3, 1)                                   # [1, gh, gw, C]


def vit_encoder_hw(images, sd, cfg, inter=None):
    """vit.py:343-365 ViT.forward at the image's own token grid; the blocks are the oracle's."""
    e = "backbone.0.encoder"
    x = F.conv2d(images, sd[e + ".patch_embed.proj.weight"], sd[e + ".patch_embed.proj.bias"], stride=cfg.patch)
    x = x.permute(0, 2, 3, 1)
    B, H, W, C = x.shape
    x = x + abs_pos_embed_hw(sd[e + ".pos_embed"], H, W)
    x = orc.to_window_major(x)
    if inter is not None:
        inter["patch"] = x
    taps = []
    for i in range(cfg.vit_depth):
        x = orc.vit_block(x, sd, "%s.blocks.%d" % (e, i), cfg.vit_heads, i in cfg.window_blocks)
        if inter is not None:
            inter["block%d" % i] = x
        if i in cfg.taps:
            taps.append(orc.from_window_major(x, B, H, W))
    return taps


def forward(sd, cfg, images, topk_override=None, inter=None, dtype=torch.float32, mask=None):
    """oracle.forward (lwdetr.py:111-174) at the size of `images` [B,3,H,W] (H, W multiples of 64); mask as there."""
    H, W = int(images.shape[-2]), int(images.shape[-1])
    if H == W == cfg.img_size:
        return orc.forward(sd, cfg, images, topk_override=topk_override, inter=inter, dtype=dtype, mask=mask)
    cfg = AtInputSize(cfg, H, W)
    with torch.no_grad():
        sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
        taps = vit_encoder_hw(images.to(dtype), sd, cfg, inter)
        levels = orc.projector(taps, sd, cfg)
        if inter is not None:
            for j, tp in enumerate(taps):
                inter["tap%d" % j] = tp
            for l, lv in enumerate(levels):
                inter["level%d" % l] = lv
        lm = orc.level_padding_masks(mask, cfg) if mask is not None and bool(mask.any()) else None
        return orc.transformer_and_heads(levels, sd, cfg, topk_override, inter, lm)
