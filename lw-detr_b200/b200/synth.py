"""Deterministic synthetic weights and inputs for parity tests and benchmarks.

The reference initialises many tensors to exactly zero (refpoint_embed lwdetr.py:69, the last
bbox_embed layer lwdetr.py:90-91, MSDeformAttn sampling_offsets.weight / attention_weights.*
ms_deform_attn.py:80-94, attention biases); zeros would hide bugs, so every tensor here is random
with a scale that keeps activations O(1) through the whole network (checked in
tests/test_oracle.py).  Values depend only on (config, seed) and the installed torch CPU RNG, so the
same call reproduces the same weights on every machine.
"""
import math

import torch

from .spec import param_spec


def _fan_in(shape):
    n = 1
    for s in shape[1:]:
        n *= s
    return max(n, 1)


def synth_state_dict(cfg, seed=1):
    g = torch.Generator().manual_seed(int(seed))
    sd = {}

    def randn(shape, std=1.0, mean=0.0):
        return torch.randn(shape, generator=g) * std + mean

    def uniform(shape, lo, hi):
        return torch.rand(shape, generator=g) * (hi - lo) + lo

    for e in param_spec(cfg):
        r, sh = e.role, e.shape
        if r in ("linear", "conv", "class"):
            t = randn(sh, 1.0 / math.sqrt(_fan_in(sh)))
        elif r == "convT":                       # ConvTranspose2d weight [Cin, Cout, 2, 2]: fan-in is Cin
            t = randn(sh, 1.0 / math.sqrt(sh[0]))
        elif r in ("linear_bias", "sampling_offsets_bias"):
            t = randn(sh, 0.1)
        elif r == "class_bias":
            t = randn(sh, 0.5, -2.0)
        elif r == "bbox_last":
            t = randn(sh, 0.5 / math.sqrt(_fan_in(sh)))
        elif r == "bbox_last_bias":
            t = randn(sh, 0.1)
        elif r == "sampling_offsets":
            t = randn(sh, 0.5 / math.sqrt(_fan_in(sh)))
        elif r == "attention_weights":
            t = randn(sh, 1.0 / math.sqrt(_fan_in(sh)))
        elif r == "attention_weights_bias":
            t = randn(sh, 0.5)
        elif r == "norm_weight":
            t = randn(sh, 0.1, 1.0)
        elif r == "norm_bias":
            t = randn(sh, 0.1)
        elif r == "layer_scale":
            t = uniform(sh, 0.05, 0.3)
        elif r == "pos_embed":
            t = randn(sh, 0.2)
        elif r == "refpoint":
            t = randn(sh, 0.3)
        elif r == "query_feat":
            t = randn(sh, 1.0)
        elif r == "bn_weight":
            t = uniform(sh, 0.5, 1.5)
        elif r == "bn_bias":
            t = randn(sh, 0.1)
        elif r == "bn_mean":
            t = randn(sh, 0.1)
        elif r == "bn_var":
            t = uniform(sh, 0.5, 1.5)
        elif r == "bn_count":
            t = torch.zeros((), dtype=torch.int64)
        else:
            raise KeyError("no synthetic rule for role %r (%s)" % (r, e.name))
        if e.name.endswith("sampling_offsets.bias"):
            t = randn(sh, 1.0)                   # sampling points spread over the reference box
        sd[e.name] = t
    return sd


def synth_images(batch, seed=0, size=640):
    """ImageNet-normalised-looking input: N(0, 1) pixels, [B, 3, size, size] fp32 (demo.py:146-159); size may also be a
    (height, width) pair."""
    g = torch.Generator().manual_seed(int(seed))
    h, w = (size, size) if isinstance(size, int) else (int(size[0]), int(size[1]))
    return torch.randn((batch, 3, h, w), generator=g)
