// The per-entry expressions of PostProcess (lwdetr.py:515-544), shared by lwdetr_postprocess (rowops.cu) and
// lwdetr_query_best (track.cu) so that both produce the same bits for one (query, class) pair.
#pragma once
#include <cuda_runtime.h>

namespace lwb {

__device__ __forceinline__ float sigmoid_f32(float x) { return 1.f / (1.f + expf(-x)); }

// pred_boxes (cx, cy, w, h), normalised -> absolute xyxy for an image of img_h x img_w
__device__ __forceinline__ float4 box_cxcywh_to_xyxy(float4 bx, float img_h, float img_w) {
  float4 r;
  r.x = (bx.x - 0.5f * bx.z) * img_w;
  r.y = (bx.y - 0.5f * bx.w) * img_h;
  r.z = (bx.x + 0.5f * bx.z) * img_w;
  r.w = (bx.y + 0.5f * bx.w) * img_h;
  return r;
}

}  // namespace lwb
