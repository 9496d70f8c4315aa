"""CUDA-native (H100, sm_90a) LW-DETR module with the reference's `models.lwdetr` surface (lwdetr.py:36-216, 509-619):
LWDETR (an nn.Module whose parameters carry the reference's state_dict names), PostProcess, build().

The forward pass is NOT PyTorch: LWDETR.forward hands the image batch to the C-ABI engine
(include/lwdetr_b200.h, lwdetr_forward), which runs the hand-written sm_90a kernel schedule.  There is
no CPU / eager fallback: without the built library or without a CUDA device, forward raises."""
import os

import torch
from torch import nn

from b200 import capi
from b200.config import config_from_args, run_size
from b200.spec import param_spec
from util.misc import NestedTensor, nested_tensor_from_tensor_list

from ._tree import Holder, attach_entries
from .backbone import build_backbone


def _default_dtype():
    return {"bf16": torch.bfloat16, "fp16": torch.float16, "fp8": torch.float8_e4m3fn}[os.environ.get("LWDETR_B200_DTYPE", "fp16")]


class LWDETR(nn.Module):
    def __init__(self, cfg, backbone=None, aux_loss=True, compute_dtype=None):
        super().__init__()
        self.cfg = cfg
        self.num_queries = cfg.num_queries
        self.group_detr = cfg.group_detr
        self.aux_loss = aux_loss
        self.two_stage = True
        self.bbox_reparam = True
        self.lite_refpoint_refine = True
        # None: parameters' 16-bit dtype, else LWDETR_B200_DTYPE / fp16; torch.float8_e4m3fn: the fp16 engine with the
        # encoder's qkv / fc1 GEMMs in e4m3 (capi.Engine)
        self.compute_dtype = compute_dtype
        self.assume_frozen = False               # True: skip the per-forward weight-change check
        entries = [e for e in param_spec(cfg) if not e.name.startswith("backbone.0.")]
        attach_entries(self, entries)
        self.transformer.d_model = cfg.hidden_dim
        self.backbone = backbone if backbone is not None else build_backbone(None, cfg)
        self._export = False
        self._engine = None
        self._engine_sig = None

    # ------------------------------------------------------------------ engine management
    def _weights_signature(self):
        sig = []
        for t in list(self.parameters()) + list(self.buffers()):
            sig.append((t.data_ptr(), t._version, t.dtype, t.device))
        return hash(tuple(sig))

    def _resolve_dtype(self):
        if self.compute_dtype is not None:
            return self.compute_dtype
        p = self.class_embed.weight
        return p.dtype if p.dtype in (torch.float16, torch.bfloat16) else _default_dtype()

    def engine(self):
        """The packed CUDA engine for the current weights (re-packed when parameters change)."""
        dt = self._resolve_dtype()
        if self._engine is not None and self._engine.dtype == dt and (self.assume_frozen and self._engine_sig is not None):
            return self._engine
        sig = (self._weights_signature(), dt)
        pdev = next(self.parameters()).device
        if self._engine is None or self._engine.dtype != dt or (pdev.type == "cuda" and self._engine.device != pdev):
            if self._engine is not None:
                self._engine.close()
            self._engine = capi.Engine(self.cfg, dt, device=next(self.parameters()).device)
            self._engine_sig = None
        if self._engine_sig != sig:
            self._engine.load_state_dict(self.state_dict())
            self._engine_sig = sig
        return self._engine

    def __deepcopy__(self, memo):
        import copy
        new = LWDETR(self.cfg, aux_loss=self.aux_loss, compute_dtype=self.compute_dtype)
        new.load_state_dict(copy.deepcopy(self.state_dict(), memo))
        p = next(self.parameters())
        new.to(device=p.device, dtype=p.dtype)
        new.train(self.training)
        return new

    # ------------------------------------------------------------------ reference surface
    def export(self):
        self._export = True
        self.backbone.export()
        self.backbone[0].export()

    def update_drop_path(self, drop_path_rate, vit_encoder_num_layers):
        """Stochastic depth only acts in training (lwdetr.py:205-210); inference ignores it."""
        return None

    def update_dropout(self, drop_rate):
        return None

    @torch.no_grad()
    def forward(self, samples, targets=None):
        """samples: NestedTensor | list of [3,H,W] tensors | [B,3,H,W] tensor (lwdetr.py:111-127).
        Returns {'pred_logits' [B,nq,C], 'pred_boxes' [B,nq,4] (cxcywh, normalised), 'aux_outputs',
        'enc_outputs'} as fp32 CUDA tensors (lwdetr.py:161-174)."""
        if self.training:
            raise RuntimeError("lwdetr_b200 implements the inference forward only; call model.eval()")
        if isinstance(samples, torch.Tensor) and samples.dtype == torch.uint8:
            # raw camera / decoder frames [B, H, W, 3] (HWC, RGB, 0..255): the reference's host-side pre-processing
            # (demo.py:146-159: /255, Normalize(mean, std), HWC -> CHW) is fused into the patch-embed load on the device.
            # H and W are multiples of 64, not smaller than img_size (frames are not padded)
            dev = next(self.parameters()).device
            if dev.type != "cuda":
                raise RuntimeError("lwdetr_b200: move the model to a CUDA device (no CPU fallback)")
            S = self.cfg.img_size
            if samples.dim() != 4 or samples.shape[3] != 3 or samples.shape[1] < S or samples.shape[2] < S:
                raise RuntimeError("lwdetr_b200: uint8 frames must be [B, H, W, 3] (HWC) with H, W >= %d, got %s" % (S, tuple(samples.shape)))
            out = self.engine().forward(samples.to(dev), want_aux=True)
            return self._pack_outputs(out)
        if isinstance(samples, (list, torch.Tensor)):
            samples = nested_tensor_from_tensor_list(samples)
        x, mask = samples.tensors, samples.mask
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("lwdetr_b200: move the model to a CUDA device (no CPU fallback)")
        if x.dim() != 4:
            raise RuntimeError("lwdetr_b200: expected a [B, 3, H, W] batch, got %s" % (tuple(x.shape),))
        # the batch runs at (max(img_size, ceil64(H)), max(img_size, ceil64(W))): sides of at most img_size keep the
        # configured input size, larger or non-square batches run at their own 64-aligned size (b200.config.run_size)
        H, W = run_size(self.cfg, x.shape[-2], x.shape[-1])
        if x.shape[-2] != H or x.shape[-1] != W:
            # pad to the run size (bottom / right, exactly what nested_tensor_from_tensor_list does between the images of a
            # batch) and extend the mask
            xp = x.new_zeros((x.shape[0], x.shape[1], H, W))
            xp[:, :, : x.shape[-2], : x.shape[-1]] = x
            mp = torch.ones((x.shape[0], H, W), dtype=torch.bool, device=x.device)
            mp[:, : x.shape[-2], : x.shape[-1]] = mask if mask is not None else False
            x, mask = xp, mp
        x = x.to(dev)
        # the padding mask only matters when something IS padded (misc.py:317-339); an all-False mask takes the constant tables
        mask = mask.to(dev) if (mask is not None and bool(mask.any())) else None
        out = self.engine().forward(x, want_aux=True, mask=mask)
        return self._pack_outputs(out)

    @torch.no_grad()
    def forward_frames(self, frames, size=None, fit="stretch", short_side=None, max_side=None, colorspace=None):
        """Raw camera / decoder frames of ANY size: a list of CUDA uint8 [h, w, 3] tensors (RGB, each its own size) or one
        [B, h, w, 3] tensor; or NV12 frames, the output of video decoders, as (luma, chroma) pairs or packed [3h/2, w]
        tensors, with colorspace= "bt601" / "bt709" / "bt601_full" / "bt709_full" (capi.Engine.forward_frames).  The
        reference's host-side transforms.Resize (demo.py:146-159; datasets/transforms.py:97-134 for fit="keep_aspect" with
        short_side / max_side) runs on the device, fused into the patch-embed load together with the colour conversion, /255
        and Normalize.  Returns the output dict of forward()."""
        if self.training:
            raise RuntimeError("lwdetr_b200 implements the inference forward only; call model.eval()")
        if next(self.parameters()).device.type != "cuda":
            raise RuntimeError("lwdetr_b200: move the model to a CUDA device (no CPU fallback)")
        out = self.engine().forward_frames(frames, size=size, fit=fit, short_side=short_side, max_side=max_side, want_aux=True,
                                           colorspace=colorspace)
        return self._pack_outputs(out)

    @torch.no_grad()
    def detect(self, frames, size=None, fit="stretch", short_side=None, max_side=None, num_select=None, colorspace=None):
        """forward_frames + PostProcess: per frame {"scores", "labels", "boxes"} with xyxy boxes in the frame's ORIGINAL
        pixel coordinates (NV12: those of the luma plane; for fit="keep_aspect" the predicted boxes are relative to the frame's
        valid region, which the valid ratios of the padded batch already provide).  num_select defaults to num_queries."""
        frames = capi.Frames(frames, next(self.parameters()).device, colorspace)
        export, self._export = self._export, False
        try:
            out = self.forward_frames(frames, size=size, fit=fit, short_side=short_side, max_side=max_side)
        finally:
            self._export = export
        sizes = torch.tensor(frames.sizes, dtype=torch.float32, device=out["pred_logits"].device)
        return PostProcess(self.num_queries if num_select is None else num_select)(out, sizes)

    @torch.no_grad()
    def detect_tiled(self, frames, tile=None, overlap=0.2, full_frame=True, size=None, per_view=100, score_threshold=0.0,
                     iou_threshold=0.5, metric="ios", max_det=300, colorspace=None):
        """Tiled (sliced) detection for high-resolution frames: the detector runs on overlapping full-resolution crops of
        every frame (plus, with full_frame, the whole frame stretched to the run size as detect() does), all views of the
        call in one batch on the run size `size` (default img_size x img_size), and the detections of each frame's views
        are merged on the device.  Frames are RGB or NV12, taken exactly as detect() takes them; NV12 crops sit at even
        offsets, so they are exact.  Steps, all on the current stream:
          b200.config.tile_views (the views: tile = (th, tw) in source pixels, default the run size, and overlap);
          Engine.forward_frames on the crop views with their dsts (partial tiles top-left on the padded, masked canvas);
          the fused PostProcess per view (top `per_view`, boxes in crop pixels);
          capi.tile_merge (boxes moved to frame pixels, score >= score_threshold, class-aware greedy NMS by "ios" or "iou"
            beyond iou_threshold, the first max_det survivors).
        Returns detect()'s list: per frame {"scores", "labels", "boxes"} (xyxy in the frame's own pixels, score order), cut to
        the frame's survivor count; that cut copies the F counts to the host, the call's only synchronisation.  All views of
        a call share one run size, so a stream of equally sized frames keeps one plan (and its CUDA graphs).  What tiling
        does to small-object recall depends on the checkpoint and the data and is not measured here."""
        from b200.config import tile_views
        if self.training:
            raise RuntimeError("lwdetr_b200 implements the inference forward only; call model.eval()")
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("lwdetr_b200: move the model to a CUDA device (no CPU fallback)")
        fb = capi.Frames(frames, dev, colorspace)
        (H, W), views = tile_views(self.cfg, fb.sizes, tile, overlap, full_frame, size, per_view)
        crops = tile_crops(fb, views)
        out = self.engine().forward_frames(crops, size=(H, W), dsts=[(v[5], v[6]) for v in views], want_aux=False)
        sizes = torch.tensor([(v[3], v[4]) for v in views], dtype=torch.float32, device=dev)
        scores, labels, boxes = capi.postprocess(out["pred_logits"], out["pred_boxes"], sizes, per_view)
        s, l, b, counts = capi.tile_merge(scores, labels, boxes, [(v[0], v[2], v[1]) for v in views], len(fb.items),
                                          score_threshold, iou_threshold, metric, max_det)
        counts = counts.cpu().tolist()
        return [{"scores": s[f, :n], "labels": l[f, :n].long(), "boxes": b[f, :n]} for f, n in enumerate(counts)]

    @torch.no_grad()
    def track(self, frames, tracker, streams=None, size=None, fit="stretch", short_side=None, max_side=None, colorspace=None,
              max_out=None, motion=None, appearance=False, reid=None, reid_size=(256, 128), reid_filter="bilinear", reid_mean=None,
              reid_std=None, reid_normalize=True, zones=None, detect_every=1, flow=None, annotate=None, speed=None, timestamps=None):
        """Multi-object tracking of video streams: frames (RGB or NV12, taken exactly as detect() takes them) run as one
        forward; each query gives one detection, its best class (capi.query_best, boxes in the frame's original pixels);
        then capi.Tracker `tracker` (ByteTrack on the device, include/lwdetr_b200.h) updates each frame's stream.
        streams: the stream of each frame, default range(len(frames)).  Several frames of one stream in a call (one video
        batched offline) are tracked in list order: tracker launch r takes the r-th frame of every stream.
        Returns per frame {"ids", "scores", "labels", "boxes", "queries"}: the activated tracks in ByteTrack's list order,
        cut to the frame's count (one read-back for the call), "queries" the query each track took its detection from.
        max_out (default num_queries) bounds the tracks returned per frame.  motion: a capi.MotionEstimator for moving
        cameras; each frame round then estimates every frame's camera motion from the same frame descriptors (nothing
        copied) and warps the stream's tracks by it before the association (Tracker.update(motion=...)).
        appearance (a tracker made with embedding_dim): True feeds each frame's final decoder hidden state (one row per
        query, Engine.forward_frames(want_hidden=True)) to Tracker.update(embeddings=...), BoT-SORT's appearance cost with
        the detector's own features; the tracker's embedding_dim must be hidden_dim.  A CUDA tensor [len(frames),
        num_queries, D] passes the caller's own embeddings instead (any ReID model's).  With motion= as well this is
        BoT-SORT with both compensations.
        reid (a tracker made with embedding_dim D): a crop-based ReID network, any callable taking crops [N, 3, h, w] and
        returning [N, D] (BoT-SORT's FastReID configuration); not combined with appearance=.  The entries the appearance cost
        looks at (score > the tracker's track_thresh) with a valid crop are selected on the device (capi.crop_select), cut out
        of the frames and resized to reid_size = (h, w) by reid_filter ("bilinear": cv2 INTER_LINEAR, as FastReID; or
        "antialias"), with (v / 255 - reid_mean) / reid_std (default ImageNet's), or the levels 0..255 with
        reid_normalize=False (capi.crops, float32); reid runs once on all of them under no_grad, and its rows are scattered
        back to their entries (zeros elsewhere: no appearance).  Zero crops: reid is not called.  This costs one extra
        synchronisation per call, the read-back of the crop count that sizes reid's batch.
        zones: a capi.Zones over the same streams; after each round's tracker update it takes the tracker's outputs as they
        are (Zones.update), and each frame's dict gains "inside" (int64 [c], each track's zone bit mask), "occupancy" (int32
        [32], present tracks per zone) and "events" (int32 [e, 5] rows (id, kind, index, label, dwell), the frame's first
        Zones.update max_events).  The event counts come back in the read-back of the track counts: no extra
        synchronisation.  With motion= the zones stay fixed in frame pixels: they are image regions, not world regions.
        detect_every N > 1 runs the detector on every N-th frame of each stream only and tracks the frames between by
        per-object optical flow (flow: a capi.BoxFlow, required; with motion= it must be the flow's own estimator, the one
        that holds each stream's chain of pyramids).  A stream's first frame after a tracker reset is a keyframe; after that
        stream s detects on its t-th frame (t from 0, counted by the tracker) when (t + s) % N == 0, which staggers the
        streams so that the forward's batch keeps its size from call to call.  Keyframes take the path above; the other
        frames go MotionEstimator.estimate (with motion=) or observe, then BoxFlow.propagate.  zones= follows both kinds of
        frame, appearance= and reid= the keyframes only; on a flow frame "queries" is -1.  detect_every=1 is the path above.
        annotate: a capi.Annotator; after each round's tracker (and zones) update it draws that round's tracks into the
        round's frames in place, from the device outputs as they are (Annotator.annotate: ids, labels and scores, and with
        zones= the lines, polygons, line totals and occupancy).  It adds no synchronisation; on flow frames it draws the
        flow's tracks.  The returned lists are the same with and without it.
        speed: a capi.SpeedEstimator over the same streams; after each round's tracker (and zones) update it takes the
        tracker's outputs as they are (SpeedEstimator.update) with that round's timestamps (timestamps: one per frame in
        seconds, a host list or a CUDA float64 tensor; None: each stream's frame count / frame_rate), and each frame's dict
        gains "position" (fp32 [c, 2], the ground point of each track's anchor, NaN beyond the horizon), "velocity" (fp32
        [c, 2]) and "speed" (fp32 [c]; NaN before the track has min_samples samples).  No extra synchronisation; keyframes
        and flow frames alike.  Not with motion=: a fixed image-to-ground homography has no meaning for a moving camera.
        How ByteTrack's thresholds (tuned on YOLOX scores) suit LW-DETR's score distribution, and whether the decoder's features tell identities apart on real footage, in MOTA / IDF1 / HOTA, is
        not measured here."""
        if self.training:
            raise RuntimeError("lwdetr_b200 implements the inference forward only; call model.eval()")
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("lwdetr_b200: move the model to a CUDA device (no CPU fallback)")
        fb = capi.Frames(frames, dev, colorspace)
        n = len(fb.items)
        streams = list(range(n)) if streams is None else [int(s) for s in streams]
        if len(streams) != n:
            raise RuntimeError("lwdetr_b200: %d streams for %d frames" % (len(streams), n))
        emb = None
        if reid is not None:
            if not (appearance is False or appearance is None):
                raise RuntimeError("lwdetr_b200: pass reid= or appearance=, not both")
            if tracker.embedding_dim is None:
                raise RuntimeError("lwdetr_b200: reid= needs a tracker made with embedding_dim")
        if isinstance(appearance, torch.Tensor):
            if tuple(appearance.shape[:2]) != (n, self.num_queries) or appearance.dim() != 3:
                raise RuntimeError("lwdetr_b200: appearance must be [%d, %d, D], got %s" % (n, self.num_queries, tuple(appearance.shape)))
            emb = appearance
        else:
            appearance = bool(appearance)
        if appearance is True and tracker.embedding_dim != self.cfg.hidden_dim:
            raise RuntimeError("lwdetr_b200: appearance=True feeds the decoder's %d-wide features, but the tracker's embedding_dim is %s"
                               % (self.cfg.hidden_dim, tracker.embedding_dim))
        detect_every = int(detect_every)
        if detect_every < 1:
            raise RuntimeError("lwdetr_b200: detect_every must be >= 1")
        if detect_every > 1 and flow is None:
            raise RuntimeError("lwdetr_b200: detect_every > 1 needs flow= (a capi.BoxFlow)")
        if flow is not None and motion is not None and motion is not flow.estimator:
            raise RuntimeError("lwdetr_b200: motion= must be the flow's own estimator (only one estimator can hold a stream's pyramids)")
        if speed is not None and motion is not None:
            raise RuntimeError("lwdetr_b200: speed= needs a still camera (a fixed homography); it cannot go with motion=")
        if timestamps is not None:
            if speed is None:
                raise RuntimeError("lwdetr_b200: timestamps= is for speed=")
            timestamps = torch.as_tensor(timestamps, dtype=torch.float64).to(dev)
            if tuple(timestamps.shape) != (n,):
                raise RuntimeError("lwdetr_b200: %d timestamps for %d frames" % (timestamps.numel(), n))
        rounds, seen = [], {}
        key = [True] * n
        for i, s in enumerate(streams):
            r = seen.get(s, 0)
            seen[s] = r + 1
            if r == len(rounds):
                rounds.append([])
            rounds[r].append(i)
            if detect_every > 1:
                t = tracker.frames[s] + r
                key[i] = t == 0 or (t + s) % detect_every == 0
        krows = [i for i in range(n) if key[i]]
        pos = {i: p for p, i in enumerate(krows)}        # a keyframe's row in the forward's batch
        if krows:
            fk = fb if len(krows) == n else fb.select(krows)
            out = self.engine().forward_frames(fk, size=size, fit=fit, short_side=short_side, max_side=max_side, want_aux=False,
                                               want_hidden=appearance is True)
            if appearance is True:
                emb = out["hidden"]
            elif emb is not None and len(krows) < n:
                emb = emb[torch.tensor(krows, device=emb.device)]
            sizes = torch.tensor(fk.sizes, dtype=torch.float32, device=dev)
            scores, labels, boxes = capi.query_best(out["pred_logits"], out["pred_boxes"], sizes)
            if reid is not None:
                emb = self._reid_embeddings(fk, scores, boxes, tracker, reid, reid_size, reid_filter, reid_mean, reid_std, reid_normalize)
        mout = self.num_queries if max_out is None else max_out
        res, counts, ev_counts = [None] * n, [], []
        for round_rows in rounds:
            parts = [[i for i in round_rows if key[i]], [i for i in round_rows if not key[i]]]
            for kind, rows in enumerate(parts):
                if not rows:
                    continue
                ids = [streams[i] for i in rows]
                if kind == 0:
                    kp = [pos[i] for i in rows]
                    idx = torch.tensor(kp, device=dev)
                    mo = None
                    if motion is not None:
                        mo = motion.estimate(fb.select(rows), ids)[0]
                    elif flow is not None:
                        flow.estimator.observe(fb.select(rows), ids)
                    em = None
                    if emb is not None:     # consecutive frames (one round, the usual case) as a view: no copy
                        em = emb[kp[0]:kp[-1] + 1] if kp == list(range(kp[0], kp[-1] + 1)) else emb[idx]
                    got = tracker.update(scores[idx], labels[idx], boxes[idx], ids, mout, motion=mo, embeddings=em)
                else:
                    mo = motion.estimate(fb.select(rows), ids)[0] if motion is not None else None
                    if mo is None:
                        flow.estimator.observe(fb.select(rows), ids)
                    got = flow.propagate(tracker, ids, motion=mo, max_out=mout)
                counts.append(got[5])
                zo = None
                if zones is not None:
                    inside, occupancy, events, n_ev = zones.update(got[0], got[2], got[3], got[5], ids)
                    zo = (inside.long() & 0xFFFFFFFF, occupancy, events)      # the uint32 masks widened once per round
                    ev_counts.append(n_ev)
                sp = None
                if speed is not None:
                    ts_rows = None
                    if timestamps is not None:    # consecutive frames as a view: no copy
                        ts_rows = timestamps[rows[0]:rows[-1] + 1] if rows == list(range(rows[0], rows[-1] + 1)) \
                            else timestamps[torch.tensor(rows, device=dev)]
                    sp = speed.update(got[0], got[3], got[5], ids, ts_rows)[0]
                if annotate is not None:
                    annotate.annotate(fb.select(rows), got[1], got[2], got[3], ids=got[0], counts=got[5], streams=ids, zones=zones,
                                      occupancy=None if zones is None else occupancy)
                for j, i in enumerate(rows):
                    res[i] = (got, zo, sp, j)
        both = torch.cat(counts + ev_counts).cpu().tolist()     # track and event counts in one read-back
        order = [i for rows in rounds for part in ([i for i in rows if key[i]], [i for i in rows if not key[i]]) for i in part]
        cnt = {i: c for i, c in zip(order, both[:n])}
        ecnt = {i: c for i, c in zip(order, both[n:])}
        dets = []
        for i in range(n):
            (ids, sc, lab, bx, q, _), zo, sp, j = res[i]
            c = cnt[i]
            d = {"ids": ids[j, :c], "scores": sc[j, :c], "labels": lab[j, :c].long(), "boxes": bx[j, :c], "queries": q[j, :c].long()}
            if zo is not None:
                inside, occupancy, events = zo
                d.update(inside=inside[j, :c], occupancy=occupancy[j], events=events[j, :min(ecnt[i], events.shape[1])])
            if sp is not None:
                d.update(position=sp[j, :c, 0:2], velocity=sp[j, :c, 2:4], speed=sp[j, :c, 4])
            dets.append(d)
        return dets

    def _reid_embeddings(self, fb, scores, boxes, tracker, reid, size, filter, mean, std, normalize):
        """[frames, num_queries, D] embeddings of the high entries by the crop-based network `reid`, zeros elsewhere; None when
        no entry has a crop."""
        frame, entry, sel, count = capi.crop_select(scores, boxes, fb.sizes, float(tracker.params.track_thresh))
        c = int(count.item())                     # sizes reid's batch: the call's one extra synchronisation
        if c == 0:
            return None
        crops, _ = capi.crops(fb, sel[:c], frame[:c], size, filter, mean, std, normalize)
        with torch.no_grad():
            rows = reid(crops)
        D = tracker.embedding_dim
        if not isinstance(rows, torch.Tensor) or tuple(rows.shape) != (c, D):
            raise RuntimeError("lwdetr_b200: reid must return [%d, %d] (crops, the tracker's embedding_dim), got %s"
                               % (c, D, tuple(rows.shape) if isinstance(rows, torch.Tensor) else type(rows)))
        return capi.scatter_rows(rows, entry[:c], scores.numel()).view(scores.shape[0], scores.shape[1], D)

    @torch.no_grad()
    def crops(self, frames, dets, size=(256, 128), filter="bilinear", mean=None, std=None, normalize=True, dtype=None, colorspace=None):
        """The input of a second-stage network (ReID, attributes, vehicle type, plates) from detect()'s per-frame result
        list: every box of every frame cut out of its frame on the device and resized to size = (h, w) (capi.crops: filter,
        mean / std / normalize and dtype as there).  Returns (crops [N, 3, h, w], frame_of_each int64 [N]), boxes in frame
        order, then the order of each frame's list; a box with an empty or non-finite crop gives zeros."""
        fb = capi.Frames(frames, next(self.parameters()).device, colorspace)
        if len(dets) != len(fb.items):
            raise RuntimeError("lwdetr_b200: %d detection lists for %d frames" % (len(dets), len(fb.items)))
        dev = fb.device
        boxes = [d["boxes"].to(device=dev, dtype=torch.float32).reshape(-1, 4) for d in dets]
        frame = torch.cat([torch.full((b.shape[0],), f, dtype=torch.int64, device=dev) for f, b in enumerate(boxes)])
        out, _ = capi.crops(fb, torch.cat(boxes), frame, size, filter, mean, std, normalize, dtype)
        return out, frame

    def _pack_outputs(self, out):
        if self._export:
            return out["pred_boxes"], out["pred_logits"]      # forward_export tuple (lwdetr.py:176-195)
        res = {"pred_logits": out["pred_logits"], "pred_boxes": out["pred_boxes"]}
        if self.aux_loss:
            res["aux_outputs"] = out["aux_outputs"]
        res["enc_outputs"] = out["enc_outputs"]
        return res


def tile_crops(frames, views):
    """capi.Frames of the crop views (frame, y0, x0, ch, cw, ...) of `frames` (capi.Frames): strided views of the frames'
    memory, nothing copied.  NV12: the luma rows / columns of the crop and the chroma rows y0/2 .. and bytes x0 .. of its
    (U, V) pairs, exact because y0 and x0 are even."""
    if not frames.nv12:
        return capi.Frames([frames.items[f][y0:y0 + ch, x0:x0 + cw] for f, y0, x0, ch, cw, _, _ in views])
    if any(y0 % 2 or x0 % 2 for _, y0, x0, _, _, _, _ in views):
        raise RuntimeError("lwdetr_b200: NV12 crops need even offsets")
    names = {c: n for n, c in capi.COLORSPACES.items()}
    pairs = [(frames.items[f][0][y0:y0 + ch, x0:x0 + cw], frames.items[f][1][y0 // 2:y0 // 2 + (ch + 1) // 2, x0:x0 + 2 * ((cw + 1) // 2)])
             for f, y0, x0, ch, cw, _, _ in views]
    return capi.Frames(pairs, colorspace=[names[frames.codes[v[0]]] for v in views])


class PostProcess(nn.Module):
    """lwdetr.py:509-544: sigmoid -> top `num_select` over (query, class) -> boxes to absolute xyxy."""

    def __init__(self, num_select=300):
        super().__init__()
        self.num_select = num_select

    @torch.no_grad()
    def forward(self, outputs, target_sizes):
        logits, boxes = outputs["pred_logits"], outputs["pred_boxes"]
        if len(logits) != len(target_sizes) or target_sizes.shape[1] != 2:
            raise ValueError("target_sizes must be [batch, 2]")
        ncls = logits.shape[2]
        if logits.is_cuda:
            # fused on the device (lwdetr_postprocess): only [B, num_select, 6] numbers are produced / leave the GPU
            scores, labels, xyxy = capi.postprocess(logits, boxes, target_sizes, self.num_select)
            labels = labels.long()
        else:
            # host tensors (e.g. outputs already copied to the CPU): plain torch, same arithmetic as the reference
            scores, flat = torch.topk(logits.sigmoid().flatten(1), self.num_select, dim=1)
            query, labels = flat // ncls, flat % ncls
            cx, cy, w, h = boxes.unbind(-1)
            xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], dim=-1)
            xyxy = torch.gather(xyxy, 1, query.unsqueeze(-1).expand(-1, -1, 4))
            img_h, img_w = target_sizes.unbind(1)
            xyxy = xyxy * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :].to(xyxy.dtype)
        return [{"scores": s, "labels": l, "boxes": b} for s, l, b in zip(scores, labels, xyxy)]


class InferenceOnlyCriterion(nn.Module):
    """build() returns a criterion for API compatibility (lwdetr.py:596-619).  Losses / Hungarian matching
    are training-side and out of scope of the inference path (SURVEY.md section 2)."""

    def __init__(self, weight_dict):
        super().__init__()
        self.weight_dict = weight_dict

    def forward(self, outputs, targets):
        raise NotImplementedError("lwdetr_b200 is an inference path: SetCriterion is not implemented")


def build(args):
    """(model, criterion, postprocessors) from the reference's argparse namespace (lwdetr.py:562-619)."""
    cfg = config_from_args(args)
    args.num_feature_levels = len(args.projector_scale)
    backbone = build_backbone(args, cfg)
    model = LWDETR(cfg, backbone=backbone, aux_loss=getattr(args, "aux_loss", True))
    weight_dict = {"loss_ce": getattr(args, "cls_loss_coef", 2), "loss_bbox": getattr(args, "bbox_loss_coef", 5),
                   "loss_giou": getattr(args, "giou_loss_coef", 2)}
    criterion = InferenceOnlyCriterion(weight_dict)
    postprocessors = {"bbox": PostProcess(num_select=getattr(args, "num_select", cfg.num_queries))}
    return model, criterion, postprocessors
