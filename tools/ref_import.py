"""Import the UNMODIFIED reference (Atten4Vis/LW-DETR): the checkout named by $LWDETR_REFERENCE_SRC, else the byte-identical
copy staged under oracle/_ref/ by oracle/vendor_reference.py (git-ignored).

Used by the golden-vector generator (tools/make_goldens.py), by tests that are skipped when no reference tree is
available, and by bench.py's reference arm / cpu_baseline leg.  Three third-party modules the
reference imports are missing offline and are shimmed (SURVEY.md section 8c):
  * timm.models.layers: DropPath (identity at eval), Mlp (fc1 -> GELU(erf) -> fc2), trunc_normal_
  * fairscale.nn.checkpoint.checkpoint_wrapper (never invoked: use_act_checkpoint=False)
  * MultiScaleDeformableAttention (the compiled CUDA op; the CPU path goes through
    ms_deform_attn_core_pytorch after MSDeformAttn.export())
"""
import argparse
import os
import sys
import types

_VENDORED = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
REF = os.environ.get("LWDETR_REFERENCE_SRC") or _VENDORED


def available():
    return os.path.isdir(os.path.join(REF, "models"))


def _install_shims():
    import torch.nn as nn
    if "timm" not in sys.modules:
        timm = types.ModuleType("timm")
        tm = types.ModuleType("timm.models")
        tl = types.ModuleType("timm.models.layers")

        class DropPath(nn.Module):
            def __init__(self, drop_prob=0.0):
                super().__init__()
                self.drop_prob = drop_prob

            def forward(self, x):
                return x

        class Mlp(nn.Module):
            def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0):
                super().__init__()
                out_features = out_features or in_features
                hidden_features = hidden_features or in_features
                self.fc1 = nn.Linear(in_features, hidden_features)
                self.act = act_layer()
                self.fc2 = nn.Linear(hidden_features, out_features)

            def forward(self, x):
                return self.fc2(self.act(self.fc1(x)))

        tl.DropPath, tl.Mlp, tl.trunc_normal_ = DropPath, Mlp, nn.init.trunc_normal_
        timm.models, tm.layers = tm, tl
        sys.modules.update({"timm": timm, "timm.models": tm, "timm.models.layers": tl})
    if "fairscale" not in sys.modules:
        fs = types.ModuleType("fairscale")
        fn = types.ModuleType("fairscale.nn")
        fc = types.ModuleType("fairscale.nn.checkpoint")
        fc.checkpoint_wrapper = lambda m, *a, **k: m
        fs.nn, fn.checkpoint = fn, fc
        sys.modules.update({"fairscale": fs, "fairscale.nn": fn, "fairscale.nn.checkpoint": fc})
    sys.modules.setdefault("MultiScaleDeformableAttention", types.ModuleType("MultiScaleDeformableAttention"))


def reference_args(cfg):
    """argparse.Namespace with exactly the fields the reference build() reads (lwdetr.py:562-619)."""
    return argparse.Namespace(
        encoder=cfg.encoder, vit_encoder_num_layers=cfg.vit_depth, pretrained_encoder=None,
        window_block_indexes=list(cfg.window_blocks), drop_path=0.0, hidden_dim=cfg.hidden_dim,
        out_feature_indexes=list(cfg.out_feature_indexes), projector_scale=list(cfg.projector_scale),
        position_embedding="sine", sa_nheads=cfg.sa_nheads, ca_nheads=cfg.ca_nheads, num_queries=cfg.num_queries,
        dropout=0.0, dim_feedforward=cfg.dim_feedforward, dec_layers=cfg.dec_layers, group_detr=cfg.group_detr,
        two_stage=True, dec_n_points=cfg.dec_n_points, lite_refpoint_refine=True, decoder_norm="LN",
        bbox_reparam=True, aux_loss=True, dataset_file="coco", device="cpu", num_select=cfg.num_queries,
        focal_alpha=0.25, cls_loss_coef=2, bbox_loss_coef=5, giou_loss_coef=2, set_cost_class=2, set_cost_bbox=5,
        set_cost_giou=2, sum_group_losses=False, use_varifocal_loss=False, use_position_supervised_loss=False,
        ia_bce_loss=False)


def build_reference(cfg):
    """Reference (model, criterion, postprocessors), eval mode, cross-attention on the grid_sample path."""
    _install_shims()
    for m in [k for k in sys.modules if k == "models" or k.startswith("models.") or k == "util" or k.startswith("util.")]:
        del sys.modules[m]
    sys.path.insert(0, REF)
    try:
        from models import build_model
        from models.ops.modules import MSDeformAttn
        model, criterion, post = build_model(reference_args(cfg))
    finally:
        sys.path.remove(REF)
        for m in [k for k in sys.modules if k == "models" or k.startswith("models.") or k == "util" or k.startswith("util.")]:
            # keep them importable by the objects already created, but free the names for our drop-in
            sys.modules["_ref_" + m] = sys.modules.pop(m)
    model.eval()
    for mod in model.modules():
        if isinstance(mod, MSDeformAttn):
            mod.export()
    return model, criterion, post
