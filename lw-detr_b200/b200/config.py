"""The five released LW-DETR configurations (reference: scripts/lwdetr_{tiny,small,medium,large,xlarge}
_coco_eval.sh:9-25, models/backbone/backbone.py:46-53) and the mapping from the reference's argparse
namespace (main.py:39-183) to them."""
from dataclasses import dataclass, field
from typing import Tuple

_ENCODER_DIM = {"vit_tiny": 192, "vit_small": 384, "vit_base": 768}


@dataclass(frozen=True)
class LWDETRConfig:
    name: str
    encoder: str
    vit_depth: int
    window_blocks: Tuple[int, ...]
    out_feature_indexes: Tuple[int, ...]
    projector_scale: Tuple[str, ...]
    hidden_dim: int
    sa_nheads: int
    ca_nheads: int
    dec_n_points: int
    num_queries: int
    dec_layers: int = 3
    dim_feedforward: int = 2048
    group_detr: int = 13
    num_classes: int = 91
    vit_heads: int = 12
    img_size: int = 640
    patch: int = 16

    @property
    def vit_dim(self):
        return _ENCODER_DIM[self.encoder]

    @property
    def grid(self):
        return self.img_size // self.patch

    @property
    def tokens(self):
        return self.grid * self.grid

    @property
    def n_levels(self):
        return len(self.projector_scale)

    @property
    def level_shapes(self):
        f = {"P3": 2.0, "P4": 1.0, "P5": 0.5}
        return tuple((int(self.grid * f[p]), int(self.grid * f[p])) for p in self.projector_scale)

    @property
    def memory_len(self):
        return sum(h * w for h, w in self.level_shapes)

    @property
    def taps(self):
        return tuple(sorted(i if i >= 0 else i + self.vit_depth for i in self.out_feature_indexes))

    def level_shapes_at(self, height, width):
        """Feature-level shapes of an input of height x width pixels: P3 = 2x, P4 = 1x, P5 = 1/2 of the (H/16, W/16) token grid."""
        gh, gw = height // self.patch, width // self.patch
        f = {"P3": 2.0, "P4": 1.0, "P5": 0.5}
        return tuple((int(gh * f[p]), int(gw * f[p])) for p in self.projector_scale)

    def memory_len_at(self, height, width):
        return sum(h * w for h, w in self.level_shapes_at(height, width))


# Input sizes the CUDA path runs: both sides multiples of 64 (4x4 windows of 16-pixel patches, vit.py:353-358) in
# [MIN_SIDE, MAX_SIDE], and at least num_queries memory tokens (torch.topk over the memory, transformer.py:246).
SIDE_STEP, MIN_SIDE, MAX_SIDE = 64, 128, 1344


def check_input_size(cfg, height, width):
    """Raise RuntimeError unless a height x width input is one the CUDA path runs."""
    if height % SIDE_STEP or width % SIDE_STEP or not (MIN_SIDE <= height <= MAX_SIDE and MIN_SIDE <= width <= MAX_SIDE):
        raise RuntimeError("lwdetr_b200: input %dx%d is not supported: height and width must be multiples of %d in [%d, %d]"
                           % (height, width, SIDE_STEP, MIN_SIDE, MAX_SIDE))
    if cfg.memory_len_at(height, width) < cfg.num_queries:
        raise RuntimeError("lwdetr_b200: a %dx%d input has %d memory tokens, fewer than num_queries = %d"
                           % (height, width, cfg.memory_len_at(height, width), cfg.num_queries))


def run_size(cfg, height, width):
    """The (H, W) a batch whose largest image is height x width runs at: each side rounded up to a multiple of 64 and never
    below img_size (smaller batches are padded to the configured size, as before), bottom / right padding carried by the
    NestedTensor mask.  800x1333 -> 832x1344.  RuntimeError when the result is not a supported input size."""
    up = lambda v: -(-int(v) // SIDE_STEP) * SIDE_STEP
    H, W = max(cfg.img_size, up(height)), max(cfg.img_size, up(width))
    check_input_size(cfg, H, W)
    return H, W


def keep_aspect_size(height, width, short_side, max_side=None):
    """(dst_h, dst_w) of the reference's resize(image, target, size, max_size) for a height x width image
    (datasets/transforms.py:97-115, the same int() / round() calls): the shorter side goes to short_side, unless the longer
    side would then exceed max_side, in which case the longer side goes to (about) max_side."""
    w, h, size = int(width), int(height), int(short_side)
    if max_side is not None:
        mn, mx = float(min(w, h)), float(max(w, h))
        if mx / mn * size > max_side:
            size = int(round(max_side * mn / mx))
    if (w <= h and w == size) or (h <= w and h == size):
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def frame_sizes(cfg, shapes, size=None, fit="stretch", short_side=None, max_side=None):
    """Run size (H, W) and per-frame (dst_h, dst_w) of a batch of raw frames with the given (h, w) shapes.
    fit="stretch": every frame fills `size` (default img_size x img_size): transforms.Resize([H, W]), what demo.py and the
    square-resize evaluation do.  fit="keep_aspect": each frame takes keep_aspect_size(h, w, short_side, max_side); without
    `size` the batch runs at run_size(cfg, max dst_h, max dst_w), frames top-left, the rest padded."""
    if fit == "stretch":
        if short_side is not None or max_side is not None:
            raise RuntimeError("lwdetr_b200: short_side / max_side belong to fit='keep_aspect'")
        H, W = (cfg.img_size, cfg.img_size) if size is None else (int(size[0]), int(size[1]))
        check_input_size(cfg, H, W)
        return (H, W), [(H, W)] * len(shapes)
    if fit != "keep_aspect":
        raise RuntimeError("lwdetr_b200: fit must be 'stretch' or 'keep_aspect', got %r" % (fit,))
    if short_side is None:
        raise RuntimeError("lwdetr_b200: fit='keep_aspect' needs short_side")
    dsts = [keep_aspect_size(h, w, short_side, max_side) for h, w in shapes]
    mh, mw = max(d[0] for d in dsts), max(d[1] for d in dsts)
    if size is None:
        H, W = run_size(cfg, mh, mw)
    else:
        H, W = int(size[0]), int(size[1])
        check_input_size(cfg, H, W)
        if mh > H or mw > W:
            raise RuntimeError("lwdetr_b200: a frame resized to %dx%d does not fit the run size %dx%d" % (mh, mw, H, W))
    return (H, W), dsts


def explicit_frame_sizes(cfg, count, dsts, size=None):
    """Run size (H, W) (`size`, default img_size x img_size) and the given per-frame (dst_h, dst_w), checked: one per frame,
    each side in [1, run side]."""
    H, W = (cfg.img_size, cfg.img_size) if size is None else (int(size[0]), int(size[1]))
    check_input_size(cfg, H, W)
    dsts = [(int(dh), int(dw)) for dh, dw in dsts]
    if len(dsts) != count:
        raise RuntimeError("lwdetr_b200: %d dsts for %d frames" % (len(dsts), count))
    for dh, dw in dsts:
        if not (1 <= dh <= H and 1 <= dw <= W):
            raise RuntimeError("lwdetr_b200: dst %dx%d does not fit the run size %dx%d" % (dh, dw, H, W))
    return (H, W), dsts


# Limits of tiled detection: the resize's downscale factor per axis (include/lwdetr_b200.h, lwdetr_frame) and what
# lwdetr_tile_merge takes per frame.
RESIZE_MAX_DOWNSCALE = 16
TILE_MAX_CANDIDATES, TILE_MAX_VIEWS = 16384, 2048


def _tile_starts(n, t, s):
    if n <= t:
        return [0]
    starts, p = [], 0
    while p + t < n:
        starts.append(p)
        p += s
    starts.append(n - t)
    out = []
    for p in starts:
        p -= p % 2
        if not out or out[-1] != p:
            out.append(p)
    return out


def _tile_dst(c, t, run):
    return run if c == t else min(max((2 * c * run + t) // (2 * t), 1), run)


def tile_views(cfg, shapes, tile=None, overlap=0.2, full_frame=True, size=None, per_view=100):
    """Views of tiled (sliced) detection for frames of the given (h, w) shapes -> ((H, W), views), every view a tuple
    (frame, y0, x0, ch, cw, dst_h, dst_w): the crop rows [y0, y0 + ch) and columns [x0, x0 + cw) of frame `frame`, resized to
    dst_h x dst_w top-left on the run size (H, W) = `size` (default img_size x img_size).  The rule, per axis of length n with
    tile side t (`tile` = (th, tw) or one int, in source pixels, default the run size) and run side R:
      stride s = t - int(overlap * t + 0.5), overlap in [0, 0.5];
      starts [0] if n <= t, else p = 0, s, 2s, ... while p + t < n, then n - t; each rounded down to even (one rule for RGB
        and NV12, whose chroma covers 2x2 pixels: an NV12 crop at even offsets is exact), duplicates dropped.  When n - t is
        odd, the last tile therefore ends one pixel short of the frame's edge; the full-frame view still sees that strip.
        Every other pixel is covered whenever the overlap is at least one pixel (s < t);
      crop side min(t, n); destination R for a full tile (a 1:1 copy when t == R), else the crop scaled as the full tiles
        are, c * R / t rounded half up and clamped to [1, R] (a partial tile, top-left on the padded, masked canvas).
    Views come per frame, tiles in row-major order, then (full_frame) the whole frame stretched to (H, W), which is what
    detect() runs; frames in input order.  RuntimeError for an overlap outside [0, 0.5], a tile more than 16x the run size
    on an axis, any view whose crop side is more than 16x its destination side (a partial tile, whose rounded destination
    may be as small as 1; with full_frame, a frame more than 16x the run size), or a frame with more views than
    lwdetr_tile_merge takes (2048, and views * per_view <= 16384)."""
    H, W = (cfg.img_size, cfg.img_size) if size is None else (int(size[0]), int(size[1]))
    check_input_size(cfg, H, W)
    th, tw = (H, W) if tile is None else ((int(tile), int(tile)) if isinstance(tile, int) else (int(tile[0]), int(tile[1])))
    if th < 1 or tw < 1:
        raise RuntimeError("lwdetr_b200: tile %dx%d must have positive sides" % (th, tw))
    if not (0.0 <= overlap <= 0.5):
        raise RuntimeError("lwdetr_b200: overlap must be in [0, 0.5], got %r" % (overlap,))
    if th > RESIZE_MAX_DOWNSCALE * H or tw > RESIZE_MAX_DOWNSCALE * W:
        raise RuntimeError("lwdetr_b200: tile %dx%d on the run size %dx%d is a downscale factor above %d"
                           % (th, tw, H, W, RESIZE_MAX_DOWNSCALE))
    sh, sw = th - int(overlap * th + 0.5), tw - int(overlap * tw + 0.5)
    views = []
    for f, (h, w) in enumerate(shapes):
        h, w = int(h), int(w)
        ch, cw = min(th, h), min(tw, w)
        dh, dw = _tile_dst(ch, th, H), _tile_dst(cw, tw, W)
        if ch > RESIZE_MAX_DOWNSCALE * dh or cw > RESIZE_MAX_DOWNSCALE * dw:
            # a partial tile's destination is rounded and clamped to >= 1, so its factor can exceed the tile's own
            raise RuntimeError("lwdetr_b200: frame %d (%dx%d): its %dx%d crop goes to %dx%d, a downscale factor above %d"
                               % (f, h, w, ch, cw, dh, dw, RESIZE_MAX_DOWNSCALE))
        mine = [(f, y0, x0, ch, cw, dh, dw) for y0 in _tile_starts(h, th, sh) for x0 in _tile_starts(w, tw, sw)]
        if full_frame:
            if h > RESIZE_MAX_DOWNSCALE * H or w > RESIZE_MAX_DOWNSCALE * W:
                raise RuntimeError("lwdetr_b200: frame %d (%dx%d) on the run size %dx%d is a downscale factor above %d"
                                   % (f, h, w, H, W, RESIZE_MAX_DOWNSCALE))
            mine.append((f, 0, 0, h, w, H, W))
        if len(mine) > TILE_MAX_VIEWS or len(mine) * per_view > TILE_MAX_CANDIDATES:
            raise RuntimeError("lwdetr_b200: frame %d (%dx%d) makes %d views of %d detections; the merge takes at most %d views "
                               "and %d candidates per frame (use a larger tile or a smaller per_view)"
                               % (f, h, w, len(mine), per_view, TILE_MAX_VIEWS, TILE_MAX_CANDIDATES))
        views += mine
    return (H, W), views


_W10 = (0, 1, 3, 6, 7, 9)
_T10 = (2, 4, 5, 9)
CONFIGS = {
    "tiny": LWDETRConfig("tiny", "vit_tiny", 6, (0, 2, 4), (1, 3, 5), ("P4",), 256, 8, 16, 2, 100),
    "small": LWDETRConfig("small", "vit_tiny", 10, _W10, _T10, ("P4",), 256, 8, 16, 2, 300),
    "medium": LWDETRConfig("medium", "vit_small", 10, _W10, _T10, ("P4",), 256, 8, 16, 2, 300),
    "large": LWDETRConfig("large", "vit_small", 10, _W10, _T10, ("P3", "P5"), 384, 12, 24, 4, 300),
    "xlarge": LWDETRConfig("xlarge", "vit_base", 10, _W10, _T10, ("P3", "P5"), 384, 12, 24, 4, 300),
}
PARAMS_M = {"tiny": 12.1, "small": 14.6, "medium": 28.2, "large": 46.8, "xlarge": 118.0}   # README.md:352-356


def config_from_args(args):
    """Build a config from the reference's argparse namespace (the fields lwdetr.py:562-619 reads)."""
    if args.encoder not in _ENCODER_DIM:
        raise NotImplementedError("lwdetr_b200 supports the ViT encoders only, got %r" % (args.encoder,))
    for flag in ("two_stage", "bbox_reparam", "lite_refpoint_refine"):
        if not getattr(args, flag, False):
            raise NotImplementedError("lwdetr_b200 implements the released configuration (--%s)" % flag)
    scales = tuple(args.projector_scale)
    if scales not in (("P4",), ("P3", "P5")):
        raise NotImplementedError("projector_scale %r is not one of the released configurations" % (scales,))
    num_classes = 91 if args.dataset_file == "coco" else (366 if args.dataset_file == "o365" else 20)
    return LWDETRConfig(
        name="custom", encoder=args.encoder, vit_depth=int(args.vit_encoder_num_layers),
        window_blocks=tuple(args.window_block_indexes), out_feature_indexes=tuple(args.out_feature_indexes),
        projector_scale=scales, hidden_dim=int(args.hidden_dim), sa_nheads=int(args.sa_nheads),
        ca_nheads=int(args.ca_nheads), dec_n_points=int(args.dec_n_points), num_queries=int(args.num_queries),
        dec_layers=int(args.dec_layers), dim_feedforward=int(args.dim_feedforward),
        group_detr=int(args.group_detr), num_classes=num_classes)
